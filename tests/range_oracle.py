"""TEST INFRASTRUCTURE ONLY. The reference's range decode (kanzi d --from / --to, ctx["from"] / ctx["to"]) restated on top of the CPU
oracle's stream header check and per-block decode (oracle/pyoracle.py), for the block range tests.

CompressedInputStream.processBlock (io/CompressedStream.go) reads every record of the stream in its serial section (:1815-1856), the
records of skipped blocks included, up to the end marker. Block ids start at 1 with the stream's first record (:1684), and decodingTask
skips block id iff `from >= 0 && id < from` or `to >= 0 && id >= to` (:1858-1871): a skipped block is not parsed, entropy decoded,
inverse transformed or checksummed. BlockDecompressor passes a bound only when it is >= 0 (app/BlockDecompressor.go:411-417), so a
negative value is "not given". The output is the decoded blocks, in order. Like the oracle's decompress_stream, the walk over all records
ends before any block is decoded, so a walk error (a length over 2^34 bits, a record or prefix past the end) wins over a block failure.
"""
import numpy as np

E_BLOCK_SIZE, E_PROCESS_BLOCK = 2, 13
COPY_MASK, TRANSFORMS_MASK = 0x80, 0x10  # io/CompressedStream.go:47-48


class RangeError(RuntimeError):
    def __init__(self, code, msg):
        self.code = code
        super().__init__("error %d: %s" % (code, msg))


def header_bits(s):
    """Bit length of the stream header (Writer.writeHeader :429-519): 121 bits of fields, 0/16/32/48 size bits, 15 + 24 bits."""
    v = int.from_bytes(bytes(s[:16]).ljust(16, b"\0"), "big")
    return 121 + (0, 16, 32, 48)[(v >> 7) & 3] + 39


def _bits(a, pos, n):
    chunk = a[pos // 8: (pos + n + 7) // 8 + 1].tobytes()
    v = int.from_bytes(chunk, "big")
    return (v >> (8 * len(chunk) - (pos % 8) - n)) & ((1 << n) - 1)


def header(oracle, s):
    """(transform48, entropy, block_size, checksum_bits, header bits); a bad header raises the oracle's code for it."""
    a = np.frombuffer(bytes(s), np.uint8)
    hb = header_bits(s)
    if 8 * a.size < hb:
        oracle.decompress(a, 1 << 20)  # raises the code of the truncated header
    # the header followed by an end marker: the oracle's readHeader checks every field and the header checksum
    bits = np.unpackbits(a)[:hb]
    probe = np.packbits(np.concatenate([bits, np.zeros(8 + (-(hb + 8)) % 8, np.uint8)]))
    oracle.decompress(probe, 1)
    ck = (0, 32, 64)[_bits(a, 36, 2)]
    return _bits(a, 43, 48), _bits(a, 38, 5), _bits(a, 91, 28) << 4, ck, hb


def walk(s, start):
    """The serial section :1815-1856 over every record: [(payload bit, payload bits)]."""
    a = np.frombuffer(bytes(s), np.uint8)
    nbits, pos, recs = 8 * a.size, start, []
    while True:
        if pos + 5 > nbits:
            raise RangeError(E_PROCESS_BLOCK, "No more data to read in the bitstream")
        lw = _bits(a, pos, 5) + 3
        if pos + 5 + lw > nbits:
            raise RangeError(E_PROCESS_BLOCK, "No more data to read in the bitstream")
        ln = _bits(a, pos + 5, lw)
        pos += 5 + lw
        if ln == 0:
            return recs
        if ln > (1 << 34):
            raise RangeError(E_BLOCK_SIZE, "Invalid block size")
        if pos + ln > nbits:
            raise RangeError(E_PROCESS_BLOCK, "No more data to read in the bitstream")
        recs.append((pos, ln))
        pos += ln


def in_range(block_id, from_block, to_block):
    """:1858-1871"""
    return not (from_block >= 0 and block_id < from_block) and not (to_block >= 0 and block_id >= to_block)


def payload(s, pos, n):
    """the record's bits, MSB first, zero padded to whole bytes (the block-local buffer :1875)"""
    a = np.frombuffer(bytes(s), np.uint8)
    bits = np.unpackbits(a[pos // 8: (pos + n + 7) // 8 + 1])[pos % 8: pos % 8 + n]
    return np.packbits(bits)


def decompress_range(oracle, s, from_block=-1, to_block=-1):
    """The decoded blocks of ids in [from_block, to_block) (negative = not given), concatenated. Raises RangeError or the oracle's
    OracleError (both carry .code)."""
    t48, et, bs, ck, hb = header(oracle, s)
    recs = walk(s, hb)
    out = [oracle.decode_block(payload(s, p, n), n, t48, et, ck, bs) for i, (p, n) in enumerate(recs) if in_range(i + 1, from_block, to_block)]
    return np.concatenate(out) if out else np.zeros(0, np.uint8)


def outcome(fn, *args, **kw):
    """("ok", bytes) or ("err", code) of a decode"""
    try:
        return "ok", bytes(np.asarray(fn(*args, **kw), np.uint8))
    except Exception as e:  # noqa: BLE001 - every decoder's error carries .code
        if not hasattr(e, "code"):
            raise
        return "err", e.code


def flip(s, bit_pos, nbits=1):
    a = np.array(s, np.uint8)
    for b in range(bit_pos, bit_pos + nbits):
        a[b // 8] ^= 0x80 >> (b % 8)
    return a


def corrupt(s, rec, kind):
    """The stream with one defect in record rec = (payload bit, payload bits): "header" (mode byte 0xFF: a COPY block whose 4-byte length
    0xFFFFFFFF is over any block size), "payload" (8 bits of its entropy data) or "checksum" (one bit of its checksum field)."""
    pos, n = rec
    if kind == "header":
        b = np.array(s, np.uint8)
        for i in range(pos, pos + 40):
            b[i // 8] |= 0x80 >> (i % 8)
        return b
    if kind == "payload":
        return flip(s, pos + n - n // 3, 8)
    mode = _bits(np.frombuffer(bytes(s), np.uint8), pos, 8)
    at = pos + 8 + (8 if (not mode & COPY_MASK and mode & TRANSFORMS_MASK) else 0) + 8 * (1 + ((mode >> 5) & 3))
    return flip(s, at + 3)
