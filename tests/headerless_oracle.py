"""TEST INFRASTRUCTURE ONLY. kanzi's headerless streams (NewWriter(..., headerless) and NewHeaderlessReader, io/CompressedStream.go:216,
:1060) restated on top of the CPU oracle (oracle/pyoracle.py), for the headerless tests.

Writer.writeHeader returns at once when headerless is set (:430), so a headerless stream is the block records and the end marker: the bits
the oracle's compress_stream writes behind the header (oracle/kzo_block.cpp:352). compress() takes the oracle's stream and drops its header
bits; records() builds the same bits block by block from the oracle's encode_block and the record framing of Writer.processBlock
(:951-976) and Close (:593-594), which the CPU tests hold against it.
The headerless reader skips readHeader (:1317), takes its parameters from NewHeaderlessReader's arguments once validateHeaderless
(:1178-1280, restated in validate()) accepts them, and walks the records from bit 0: decompress() is range_oracle's walk and block decode
from there.
"""
import numpy as np

import range_oracle as ro

E_STREAM_VERSION, E_INVALID_PARAM = 16, 18
BS_VERSION = 6
ENTROPY_IDS = {0, 1, 2, 4, 5, 6, 7, 8, 9}              # entropy.GetType's names (EntropyCodecFactory.go:170-206): no PAQ (3)
TRANSFORM_IDS = set(range(20)) - {4}                    # transform.GetType's names (Factory.go:330-395): no SNAPPY (4)


def end_bit(s, start):
    """The first bit behind the end marker of the records that start at bit `start`."""
    a = np.frombuffer(bytes(s), np.uint8)
    recs = ro.walk(s, start)
    pos = recs[-1][0] + recs[-1][1] if recs else start
    return pos + 5 + ro._bits(a, pos, 5) + 3


def drop_bits(s, n, total):
    """Bits n .. total - 1 of s, MSB first, zero padded to whole bytes."""
    bits = np.unpackbits(np.frombuffer(bytes(s), np.uint8))[n:total]
    return np.packbits(bits)


def compress(oracle, data, transform, entropy, block_size, checksum_bits=0, input_size=0):
    """The oracle's stream without its header: what compress_stream writes with StreamParams::headerless."""
    s = oracle.compress(data, transform, entropy, block_size, checksum_bits, input_size=input_size)
    hb = ro.header_bits(s)
    return drop_bits(s, hb, end_bit(s, hb))


def _uint_bits(v, n):
    return np.array([(v >> (n - 1 - i)) & 1 for i in range(n)], np.uint8)


def records(oracle, data, transform, entropy, block_size, checksum_bits=0):
    """The headerless stream built block by block: for every block the 5-bit length width, the length and the block's bit string
    (encode_block), then the 8-bit end marker. encode_block sizes TEXT's hash map from the block's own length, so chains with TEXT may
    differ from compress() on a short last block."""
    a = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data
    t48 = oracle.parse_transform(transform) if isinstance(transform, str) else transform
    et = oracle.parse_entropy(entropy) if isinstance(entropy, str) else entropy
    parts = []
    for off in range(0, a.size, block_size):
        payload, written = oracle.encode_block(a[off: off + block_size], t48, et, checksum_bits)
        lw = 3 if written < 8 else (written >> 3).bit_length() - 1 + 4
        parts += [_uint_bits(lw - 3, 5), _uint_bits(written, lw), np.unpackbits(payload)[:written]]
    parts.append(np.zeros(8, np.uint8))
    return np.packbits(np.concatenate(parts))


def validate(transform48, entropy, block_size, checksum_bits, bs_version=BS_VERSION):
    """0, or the code Reader.validateHeaderless gives, over ids instead of names. A bitstream version below 6 is -STREAM_VERSION: the GPU
    decoders read version 6 only."""
    if bs_version > BS_VERSION:
        return E_INVALID_PARAM
    if bs_version < BS_VERSION:
        return E_STREAM_VERSION
    if entropy not in ENTROPY_IDS:
        return E_INVALID_PARAM
    if transform48 >> 48 or any(((transform48 >> (42 - 6 * i)) & 63) not in TRANSFORM_IDS for i in range(8)):
        return E_INVALID_PARAM
    if not 1024 <= block_size <= 1 << 30:
        return E_INVALID_PARAM
    if checksum_bits not in (0, 32, 64):
        return E_INVALID_PARAM
    return 0


def decompress(oracle, s, transform, entropy, block_size, checksum_bits=0, from_block=-1, to_block=-1):
    """The headerless reader: the records walked from bit 0, the blocks of ids in [from_block, to_block) decoded with the given
    parameters and concatenated. Raises range_oracle.RangeError or the oracle's OracleError (both carry .code)."""
    t48 = oracle.parse_transform(transform) if isinstance(transform, str) else transform
    et = oracle.parse_entropy(entropy) if isinstance(entropy, str) else entropy
    recs = ro.walk(s, 0)
    out = [oracle.decode_block(ro.payload(s, p, n), n, t48, et, checksum_bits, block_size) for i, (p, n) in enumerate(recs)
           if ro.in_range(i + 1, from_block, to_block)]
    return np.concatenate(out) if out else np.zeros(0, np.uint8)
