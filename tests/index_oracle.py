"""TEST INFRASTRUCTURE ONLY. A model of the stream index and the batched range reads (kz_index_*, kz_read_ranges) on top of the CPU oracle,
whose sources stay as they are.

Record positions come from range_oracle.walk. Blocks are independent and every block but the last decodes to block_size bytes, so the
bytes of a request are a slice of the decoded blocks it touches, and a request on a damaged block fails with the outcome of decoding that
block alone: range_oracle.decompress_range(oracle, s, k + 1, k + 2) (headerless_oracle.decompress for a headerless stream). A decoded
block that is not the last and not block_size long makes the requests on it and on every later block fail with INVALID_FILE.
The blob layout of kz_index_save is stated here independently of the library (blob()), XXH64 included.
"""
import struct

import numpy as np

import headerless_oracle as ho
import range_oracle as ro

E_INVALID_FILE = 15
MAGIC, VERSION = 0x58495A4B, 1
M64 = (1 << 64) - 1


def xxh64(data, seed=0):
    """XXH64 (the public algorithm) of bytes."""
    P1, P2, P3, P4, P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261
    rotl = lambda v, r: ((v << r) | (v >> (64 - r))) & M64  # noqa: E731
    rnd = lambda acc, v: (rotl((acc + v * P2) & M64, 31) * P1) & M64  # noqa: E731
    merge = lambda h, v: ((h ^ rnd(0, v)) * P1 + P4) & M64  # noqa: E731
    n, p = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & M64, (seed + P2) & M64, seed, (seed - P1) & M64]
        while n - p >= 32:
            for i in range(4):
                v[i] = rnd(v[i], int.from_bytes(data[p + 8 * i: p + 8 * i + 8], "little"))
            p += 32
        h = (rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18)) & M64
        for x in v:
            h = merge(h, x)
    else:
        h = (seed + P5) & M64
    h = (h + n) & M64
    while n - p >= 8:
        h = (rotl(h ^ rnd(0, int.from_bytes(data[p: p + 8], "little")), 27) * P1 + P4) & M64
        p += 8
    if n - p >= 4:
        h = (rotl(h ^ (int.from_bytes(data[p: p + 4], "little") * P1) & M64, 23) * P2 + P3) & M64
        p += 4
    while p < n:
        h = (rotl(h ^ (data[p] * P5) & M64, 11) * P1) & M64
        p += 1
    h ^= h >> 33
    h = (h * P2) & M64
    h ^= h >> 29
    h = (h * P3) & M64
    return h ^ (h >> 32)


def build(oracle, s, headerless=None):
    """The model index of stream s. headerless: a dict (transform48, entropy, block_size, checksum_bits, output_size) for a stream without
    a header. A bad header or record raises with the decoders' code (.code)."""
    s = bytes(np.asarray(s, np.uint8))
    if headerless is None:
        t48, et, bs, ck, hb = ro.header(oracle, s)
        v = int.from_bytes(s[:32].ljust(32, b"\0"), "big")
        mask = (v >> (256 - 121)) & 3  # Writer.writeHeader :429-519: 119 bits of fields, the 2-bit size mask, then the size
        isz = (v >> (256 - 121 - 16 * mask)) & ((1 << (16 * mask)) - 1) if mask else 0
    else:
        t48, et, bs, ck = (headerless[k] for k in ("transform48", "entropy", "block_size", "checksum_bits"))
        isz = headerless.get("output_size", 0)
        isz = 0 if isz < 0 or isz >= 1 << 48 else isz
        hb = 0
    recs = ro.walk(s, hb)
    return {"transform48": t48, "entropy": et, "block_size": bs, "checksum_bits": ck, "input_size": isz, "header_bits": hb, "nblocks": len(recs),
            "stream_bytes": len(s), "size": 0 if not recs else -1, "head": s[:32].ljust(32, b"\0"), "recs": recs, "headerless": headerless is not None}


def info(m):
    return {k: m[k] for k in ("transform48", "entropy", "block_size", "checksum_bits", "input_size", "nblocks", "stream_bytes", "size")}


def blob(m):
    """kz_index_save's bytes for the model index."""
    b = struct.pack("<IIQIIIIqQQq", MAGIC, VERSION, m["transform48"], m["entropy"], m["block_size"], m["checksum_bits"], m["header_bits"],
                    m["input_size"], m["stream_bytes"], m["nblocks"], m["size"]) + m["head"]
    b += b"".join(struct.pack("<Q", p) for p, _ in m["recs"]) + b"".join(struct.pack("<Q", n) for _, n in m["recs"])
    return b + struct.pack("<Q", xxh64(b))


def decode_block(oracle, s, m, k):
    """("ok", bytes) or ("err", code) of block k (0-based) decoded alone"""
    if m["headerless"]:
        return ro.outcome(ho.decompress, oracle, s, m["transform48"], m["entropy"], m["block_size"], m["checksum_bits"], k + 1, k + 2)
    return ro.outcome(ro.decompress_range, oracle, s, k + 1, k + 2)


def read(oracle, s, m, requests):
    """[("ok", bytes) or ("err", code)] for requests [(off, length)]; updates m["size"] as the reads do."""
    bs, nb = m["block_size"], m["nblocks"]
    total = m["size"] if m["size"] >= 0 else nb * bs
    touched = set()
    for off, ln in requests:
        ln = min(ln, total - off) if off < total else 0
        if ln:
            touched.update(range(off // bs, (off + ln - 1) // bs + 1))
    dec = {k: decode_block(oracle, s, m, k) for k in sorted(touched)}
    bad_len = [k for k, (st, b) in dec.items() if st == "ok" and ((len(b) != bs and k != nb - 1) or len(b) > bs or not b)]
    unseekable = min(bad_len) if bad_len else None
    if nb - 1 in dec and dec[nb - 1][0] == "ok" and unseekable is None:
        m["size"] = (nb - 1) * bs + len(dec[nb - 1][1])
    out = []
    for off, ln in requests:
        ln = min(ln, total - off) if off < total else 0
        got, err = b"", None
        for k in (range(off // bs, (off + ln - 1) // bs + 1) if ln else ()):
            if unseekable is not None and k >= unseekable:
                err = E_INVALID_FILE
            elif dec[k][0] == "err":
                err = dec[k][1]
            if err is not None:
                break
            lo, hi = max(off, k * bs) - k * bs, min(off + ln, (k + 1) * bs) - k * bs
            got += dec[k][1][lo:hi]
        out.append(("err", err) if err is not None else ("ok", got))
    return out
