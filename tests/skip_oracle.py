"""TEST INFRASTRUCTURE ONLY. kanzi's skipBlocks option (kanzi c --skip, ctx["skipBlocks"]) restated for the skip tests, on top of the CPU
oracle (oracle/pyoracle.py).

stored() is an independent statement of encodingTask.encode's decision (io/CompressedStream.go:773-800): a block of at most 15 bytes is
always stored; a longer one is stored when IsDataCompressed(GetMagicType(block)) (internal/Magic.go:73-153) or when
ComputeFirstOrderEntropy1024 (internal/Global.go:174-214) of its order-0 histogram reaches INCOMPRESSIBLE_THRESHOLD (973,
entropy/EntropyUtils.go:26). The integer arithmetic uses the reference's LOG2_4096 table from tests/golden/reference_tables.json.

compress() builds the stream kanzi writes with the option on. A block that is not stored gets the record the oracle's stream has without
the option (the option changes nothing else), and a stored block gets the record of the oracle's encode_block with skip_blocks, which
the CPU tests check carries COPY_BLOCK_MASK exactly when stored() says so. The records are framed as Writer.processBlock (:951-976) and
Close (:593-594) frame them.
"""
import json
import os

import numpy as np

import headerless_oracle as hlo
import range_oracle as ro

LOG2_4096 = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_tables.json")))["log2_4096"]
SMALL_BLOCK = 15
INCOMPRESSIBLE_THRESHOLD = 973

# internal/Magic.go:24-52
JPG, GIF, PDF, ZIP, LZMA, PNG, ELF = 0xFFD8FFE0, 0x47494638, 0x25504446, 0x504B0304, 0x377ABCAF, 0x89504E47, 0x7F454C46
MAC32, CIGAM32, MAC64, CIGAM64 = 0xFEEDFACE, 0xCEFAEDFE, 0xFEEDFACF, 0xCFFAEDFE
ZSTD, BROTLI, RIFF, CAB, FLAC, XZ, RAR, KNZ = 0x28B52FFD, 0x81CFB2CE, 0x52494646, 0x4D534346, 0x664C6143, 0xFD377A58, 0x52617221, 0x4B414E5A
BZIP2, ID3 = 0x425A68, 0x494433
GZIP, BMP, WIN, PBM, PGM, PPM = 0x1F8B, 0x424D, 0x4D5A, 0x5034, 0x5035, 0x5036
KEYS32 = [GIF, PDF, ZIP, LZMA, PNG, ELF, MAC32, CIGAM32, MAC64, CIGAM64, ZSTD, BROTLI, CAB, RIFF, FLAC, XZ, KNZ, RAR]  # _KEYS32 :61-66
KEYS16 = [GZIP, BMP, WIN]                                                                                          # _KEYS16 :68-70
COMPRESSED = {JPG, GIF, PNG, LZMA, ZSTD, BROTLI, CAB, ZIP, GZIP, BZIP2, FLAC, ID3, XZ, KNZ, RAR}                    # IsDataCompressed :116-153


def magic_type(block):
    """GetMagicType (:74-112); 0 = NO_MAGIC"""
    b = bytes(block[:4])
    if len(b) < 4:
        return 0
    key = int.from_bytes(b, "big")
    if key & ~0x0F == JPG:
        return key
    if key >> 8 in (BZIP2, ID3):
        return key >> 8
    if key in KEYS32:
        return key
    if key >> 16 in KEYS16:
        return key >> 16
    if key >> 16 in (PBM, PGM, PPM) and (key >> 8) & 0xFF in (0x07, 0x0A, 0x0D, 0x20):
        return key >> 16
    return 0


def log2_scaled_1024(x):
    """Log2ScaledBy1024 (internal/Global.go:174-191), x >= 1"""
    if x < 256:
        return (LOG2_4096[x] + 2) >> 2
    lg = x.bit_length() - 1
    if x & (x - 1) == 0:
        return lg << 10
    return (lg - 7) * 1024 + ((LOG2_4096[x >> (lg - 7)] + 2) >> 2)


def entropy_1024(n, histo):
    """ComputeFirstOrderEntropy1024 (:196-214): the uint32 difference wraps like the reference's"""
    if n == 0:
        return 0
    ll = log2_scaled_1024(n)
    s = sum((int(h) * ((ll - log2_scaled_1024(int(h))) & 0xFFFFFFFF)) >> 3 for h in histo if h)
    return s // n


def block_entropy(block):
    return entropy_1024(len(block), np.bincount(np.frombuffer(bytes(block), np.uint8), minlength=256))


def reason(block):
    """Why encodingTask.encode with skipBlocks stores the block: "small", "magic", "entropy", or None when it does not"""
    if len(block) <= SMALL_BLOCK:
        return "small"
    if magic_type(block) in COMPRESSED:  # len(block) >= 8 holds here (:782)
        return "magic"
    if block_entropy(block) >= INCOMPRESSIBLE_THRESHOLD:
        return "entropy"
    return None


def stored(block):
    return reason(block) is not None


def _record(payload, written):
    lw = 3 if written < 8 else (written >> 3).bit_length() - 1 + 4
    return [hlo._uint_bits(lw - 3, 5), hlo._uint_bits(written, lw), np.unpackbits(np.asarray(payload, np.uint8))[:written]]


def compress(oracle, data, transform, entropy, block_size, checksum_bits=0, input_size=0, headerless=False, skip=True):
    """The stream kanzi writes with skipBlocks = skip (and the headerless writer setting)."""
    a = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, np.uint8)
    t48 = oracle.parse_transform(transform) if isinstance(transform, str) else transform
    et = oracle.parse_entropy(entropy) if isinstance(entropy, str) else entropy
    s = oracle.compress(a, t48, et, block_size, checksum_bits, input_size=input_size)
    hb = ro.header_bits(s)
    bits = np.unpackbits(np.frombuffer(bytes(s), np.uint8))
    parts = [] if headerless else [bits[:hb]]
    for i, (p, n) in enumerate(ro.walk(s, hb)):
        block = a[i * block_size: (i + 1) * block_size]
        if skip and stored(block):
            parts += _record(*oracle.encode_block(block, t48, et, checksum_bits, skip_blocks=True))
        else:
            parts += _record(ro.payload(s, p, n), n)
    parts.append(np.zeros(8, np.uint8))
    return np.packbits(np.concatenate(parts))


def entropy_block(target, n=1 << 16, seed=0):
    """n shuffled bytes whose order-0 entropy is exactly `target` (1024 scale, found near 973): symbol 0 takes c bytes and the other 255
    share the rest evenly; the first c (searched upwards) that gives the target wins."""
    for c in range(n // 256, n):
        h = np.full(256, (n - c) // 255, np.int64)
        h[1: 1 + (n - c) % 255] += 1
        h[0] = c
        e = entropy_1024(n, h)
        if e == target:
            x = np.repeat(np.arange(256, dtype=np.uint8), h)
            np.random.default_rng(seed).shuffle(x)
            assert magic_type(x) not in COMPRESSED
            return x
        if e < target:
            break
    raise ValueError("no histogram of this family gives entropy %d at n = %d" % (target, n))
