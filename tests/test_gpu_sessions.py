"""GPU tests of the streaming sessions (kz_writer_* / kz_reader_*): the writer's output equals the oracle's stream and kz_compress_stream's
whatever the piece sizes, batch_blocks and output caps, with batch boundaries inside a byte (the carry); the reader decodes oracle streams fed
in any pieces and ignores bytes behind the end marker; a defective stream gets kz_decompress_stream's code; errors are sticky; a session can
be freed mid-stream; memory does not grow with the stream; sessions on two contexts run side by side."""
import ctypes as C
import hashlib
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BS = 1024
LEVELS = {"l0": ("NONE", "NONE"), "l1": ("LZX", "NONE"), "l2": ("DNA+LZ", "HUFFMAN"), "l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"),
          "l4": ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")}
CHAINS = [(tr, en, 0) for tr, en in LEVELS.values()] + [
    ("BWTS+MTFT+ZRLT", "ANS0", 0), ("BWT+RANK+ZRLT", "ANS1", 0), ("LZ", "RANGE", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 32), ("NONE", "ANS0", 64)]
SIZES = [0, 1, 15, 16, 17, BS - 1, BS, BS + 1, 12 * BS + 100]


def pieces(n, mode, rng):
    if mode == "byte":
        return [1] * n
    if mode == "block":
        return [BS] * (n // BS) + ([n % BS] if n % BS else [])
    if mode == "whole":
        return [n]
    out = []
    while sum(out) < n:
        out.append(min(int(rng.integers(1, 3 * BS)), n - sum(out)))
    return out


def pump(gpu, step, fin, h, x, sizes, cap):
    """drives one session through the C ABI: sizes = piece sizes of x -> (bytes handed out, error code or 0)"""
    out = np.empty(max(cap, 1), np.uint8)
    used, made = C.c_size_t(0), C.c_size_t(0)
    parts, pos, base = [], 0, x.ctypes.data if x.size else None
    for p in sizes:
        end = pos + p
        while pos < end:
            rc = step(h, base + pos, end - pos, C.byref(used), out.ctypes.data, cap, C.byref(made))
            if rc < 0:
                return np.concatenate(parts + [np.zeros(0, np.uint8)]), -rc
            assert used.value or made.value, "a call neither consumed nor produced"
            pos += used.value
            parts.append(out[: made.value].copy())
    while True:
        rc = fin(h, out.ctypes.data, cap, C.byref(made))
        if rc < 0:
            return np.concatenate(parts + [np.zeros(0, np.uint8)]), -rc
        parts.append(out[: made.value].copy())
        if rc == 0:
            return np.concatenate(parts + [np.zeros(0, np.uint8)]), 0


def write_stream(kz, gpu, x, tr, en, ck, bb, sizes, cap, hint, bs=BS):
    h = C.c_void_p()
    gpu._check(gpu.lib.kz_writer_open(gpu.h, kz.transform_type(tr), kz.entropy_type(en), bs, ck, bb, hint, C.byref(h)))
    try:
        return pump(gpu, gpu.lib.kz_writer_write, gpu.lib.kz_writer_finish, h, x, sizes, cap)
    finally:
        gpu.lib.kz_writer_free(h)


def read_stream(gpu, s, bb, sizes, cap):
    h = C.c_void_p()
    gpu._check(gpu.lib.kz_reader_open(gpu.h, bb, C.byref(h)))
    try:
        return pump(gpu, gpu.lib.kz_reader_read, gpu.lib.kz_reader_finish, h, s, sizes, cap)
    finally:
        gpu.lib.kz_reader_free(h)


def header_bits(s):
    v = int.from_bytes(bytes(s[:16]), "big")
    return 121 + (0, 16, 32, 48)[(v >> 7) & 3] + 39


def records(s):
    """(prefix bit, payload bit, payload bits) of every block record of a complete stream"""
    v, nbits = int.from_bytes(bytes(s), "big"), 8 * len(s)
    bit = lambda p, n: (v >> (nbits - p - n)) & ((1 << n) - 1)  # noqa: E731
    pos, out = header_bits(s), []
    while True:
        lw = bit(pos, 5) + 3
        ln = bit(pos + 5, lw)
        if ln == 0:
            return out
        out.append((pos, pos + 5 + lw, ln))
        pos += 5 + lw + ln


def code_of(gpu, kz, s, cap):
    try:
        gpu.decompress(s, cap)
    except kz.KanziError as e:
        return e.code
    return 0


@pytest.mark.parametrize("chain", CHAINS, ids=["%s-%s-x%d" % c for c in CHAINS])
def test_writer_matches_oracle_and_compress(kz, gpu, oracle, synth, chain):
    tr, en, ck = chain
    rng = np.random.default_rng(len(tr) * 7 + ck)
    unaligned = 0
    case = 0
    for i, n in enumerate(SIZES):
        x = synth.markov_text(n, seed=100 + i)[:n] if n else np.zeros(0, np.uint8)
        x = np.ascontiguousarray(x, np.uint8)
        for hint in (0, n):
            want = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=hint)
            assert np.array_equal(gpu.compress(x, tr, en, BS, ck, hint), want)
            recs = records(want)
            for bb in ((1, 2, 5) if n > 4 * BS else ((1, 2, 5)[case % 3],)):
                mode = ("byte", "random", "block", "whole")[case % 4] if n <= 2 * BS or case % 4 else "random"
                cap = (1, 7, 1 << 20)[case % 3] if n <= 2 * BS else (7, 1 << 20)[case % 2]
                case += 1
                got, err = write_stream(kz, gpu, x, tr, en, ck, bb, pieces(n, mode, rng), cap, hint)
                assert err == 0 and np.array_equal(got, want), (chain, n, hint, bb, mode, cap, err)
                unaligned += sum(1 for k in range(bb, len(recs), bb) if recs[k][0] % 8)
    assert unaligned > 0, "no batch boundary inside a byte: the carry was not exercised"


def test_reader_decodes_oracle_streams(kz, gpu, oracle, synth):
    rng = np.random.default_rng(11)
    for i, (tr, en, ck) in enumerate(CHAINS):
        n = [12 * BS + 100, 3 * BS, 17, 0][i % 4]
        x = np.ascontiguousarray(synth.markov_text(max(n, 1), seed=200 + i)[:n], np.uint8)
        s = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=n)
        trailing = np.concatenate([s, rng.integers(0, 256, 100).astype(np.uint8)])
        for j, mode in enumerate(("1", "13", "random", "whole")):
            src = trailing if j % 2 else s
            sizes = {"1": [1] * src.size, "13": [13] * (src.size // 13) + [src.size % 13], "whole": [src.size]}.get(mode)
            if sizes is None:
                sizes = pieces(src.size, "random", rng)
            got, err = read_stream(gpu, src, (1, 2, 5, 1024)[(i + j) % 4], [p for p in sizes if p], (3, 1 << 20)[j % 2])
            assert err == 0 and np.array_equal(got, x), (tr, en, ck, mode, err)


def test_reader_errors_match_decompress(kz, gpu, oracle, synth):
    x = np.ascontiguousarray(synth.markov_text(10 * BS + 5, seed=3), np.uint8)
    cases = []
    for tr, en, ck in [("NONE", "NONE", 32), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0), ("LZ", "HUFFMAN", 64)]:
        s = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=len(x))
        recs = records(s)
        hb = header_bits(s)
        cases += [("header", s[: hb // 8 - 2]), ("prefix", s[: recs[3][0] // 8 + 1]), ("record", s[: (recs[4][1] + recs[4][2] // 2) // 8]),
                  ("before end", s[:-1])]
        bad = s.copy()
        p = recs[2][1] // 8 + 1
        bad[p: p + 4] = 0  # the block header of record 2: mode byte and length
        cases.append(("block header", bad))
        ver = s.copy()
        ver[4] ^= 0x30
        cases.append(("version", ver))
    s = oracle.compress(x, "NONE", "NONE", block_size=BS, checksum_bits=32, input_size=len(x))
    recs = records(s)
    bad = s.copy()
    bad[(recs[6][1] + recs[6][2]) // 8 - 20] ^= 0x5A  # data of block 6: checksum mismatch
    cases.append(("checksum", bad))
    for name, c in cases:
        want = code_of(gpu, kz, c, len(x) + 64)
        assert want != 0, name
        for bb in (1, 4):
            got, err = read_stream(gpu, np.ascontiguousarray(c), bb, [c.size], 1 << 20)
            assert err == want, (name, bb, err, want)
            if name == "checksum":
                assert got.size <= 6 * BS and np.array_equal(got, x[: got.size])


def test_writer_errors_and_sticky_codes(kz, gpu):
    h = C.c_void_p()
    L = gpu.lib
    t, e = kz.transform_type("LZ"), kz.entropy_type("HUFFMAN")
    for args, code in [((t, e, 1000, 0, 4), 18), ((t, e, BS, 16, 4), 18), ((t, e, BS, 0, 0), 18), ((t, e, BS, 0, 1025), 18),
                       ((kz.transform_type("SRT"), e, BS, 0, 4), 14), ((t, kz.entropy_type("CM"), BS, 0, 4), 14)]:
        assert L.kz_writer_open(gpu.h, *args, 0, C.byref(h)) == -code, args
        if args[4] in (0, 1025):
            continue  # batch_blocks has no counterpart in kz_compress_stream
        with pytest.raises(kz.KanziError) as ei:
            gpu.compress(np.zeros(10, np.uint8), args[0], args[1], args[2], args[3])
        assert ei.value.code == code, args
    x = np.arange(5000, dtype=np.uint8)
    gpu._check(L.kz_writer_open(gpu.h, t, e, BS, 0, 2, 0, C.byref(h)))
    out = np.empty(1 << 16, np.uint8)
    used, made = C.c_size_t(0), C.c_size_t(0)
    while True:
        if L.kz_writer_finish(h, out.ctypes.data, out.size, C.byref(made)) == 0:
            break
    rc = L.kz_writer_write(h, x.ctypes.data, x.size, C.byref(used), out.ctypes.data, out.size, C.byref(made))
    assert rc == -18
    for _ in range(2):
        assert L.kz_writer_write(h, x.ctypes.data, x.size, C.byref(used), out.ctypes.data, out.size, C.byref(made)) == rc
        assert L.kz_writer_finish(h, out.ctypes.data, out.size, C.byref(made)) == rc
    L.kz_writer_free(h)
    # a reader error is sticky too
    r = C.c_void_p()
    gpu._check(L.kz_reader_open(gpu.h, 2, C.byref(r)))
    junk = np.full(100, 7, np.uint8)
    rc = L.kz_reader_read(r, junk.ctypes.data, junk.size, C.byref(used), out.ctypes.data, out.size, C.byref(made))
    assert rc == -15
    assert L.kz_reader_read(r, junk.ctypes.data, junk.size, C.byref(used), out.ctypes.data, out.size, C.byref(made)) == rc
    assert L.kz_reader_finish(r, out.ctypes.data, out.size, C.byref(made)) == rc
    L.kz_reader_free(r)


def test_free_mid_stream(kz, gpu, oracle, synth):
    x = np.ascontiguousarray(synth.silesia_shaped(24 << 20, seed=9), np.uint8)
    tr, en = LEVELS["l3"]
    w = gpu.stream_writer(tr, en, 1 << 20, batch_blocks=4)
    w.write(x[: 18 << 20])  # several batches handed over, one in flight
    w.close()
    s = gpu.compress(x, tr, en, 1 << 20)
    r = gpu.stream_reader(batch_blocks=2)
    r.write(s[: s.size // 2])
    r.close()
    want = oracle.compress(x, tr, en, block_size=1 << 20)
    with gpu.stream_writer(tr, en, 1 << 20, batch_blocks=4) as w:
        got = np.concatenate([w.write(x[: 10 << 20]), w.write(x[10 << 20:]), w.finish()])
    assert np.array_equal(got, want)
    assert np.array_equal(gpu.decompress(want, x.size + 64), x)
    with gpu.stream_reader(batch_blocks=3) as r:
        y = np.concatenate([r.write(want[:1000]), r.write(want[1000:]), r.finish()])
    assert np.array_equal(y, x)


def test_bounded_memory_2gib(kz, gpu, synth):
    tr, en, bs, bb = "TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 4 << 20, 8
    base = np.ascontiguousarray(synth.silesia_shaped(64 << 20, seed=21), np.uint8)
    npieces = 32  # 2 GiB, generated piecewise
    piece = lambda i: np.roll(base, 7919 * i)  # noqa: E731
    ctx = kz.Context(0)
    h_in, h_out = hashlib.sha256(), hashlib.sha256()
    stream_parts = []
    after3 = None
    with ctx.stream_writer(tr, en, bs, batch_blocks=bb, input_size=npieces * base.size) as w:
        for i in range(npieces):
            p = piece(i)
            h_in.update(p)
            stream_parts.append(w.write(p))
            if i == 7:  # 512 MiB handed over: at least three batches of 32 MiB are done
                after3 = ctx.device_bytes()
        stream_parts.append(w.finish())
        at_end = ctx.device_bytes()
    assert after3 == at_end, (after3, at_end)
    stream = np.concatenate(stream_parts)
    h_out.update(stream)
    with ctx.stream_reader(batch_blocks=bb) as r:
        h_back = hashlib.sha256()
        for o in range(0, stream.size, 1 << 20):
            h_back.update(r.write(stream[o: o + (1 << 20)]))
        h_back.update(r.finish())
    assert h_back.digest() == h_in.digest()
    ctx.close()
    # the whole-stream call on the shared context (a second context beside it would hold a second set of scratch)
    x = np.concatenate([piece(i) for i in range(npieces)])
    s = gpu.compress(x, tr, en, bs, 0, x.size)
    assert hashlib.sha256(s).digest() == h_out.digest()
    assert at_end * 4 < gpu.device_bytes(), (at_end, gpu.device_bytes())


def test_sessions_on_two_contexts_side_by_side(kz, synth):
    x = np.ascontiguousarray(synth.silesia_shaped(6 << 20, seed=13), np.uint8)
    jobs = [("TEXT+UTF+BWT+RANK+ZRLT", "ANS0"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN")]
    ctxs = [kz.Context(0) for _ in jobs]

    def run(i):
        tr, en = jobs[i]
        with ctxs[i].stream_writer(tr, en, 1 << 20, batch_blocks=2) as w:
            s = np.concatenate([w.write(x[o: o + (1 << 19)]) for o in range(0, x.size, 1 << 19)] + [w.finish()])
        with ctxs[i].stream_reader(batch_blocks=3) as r:
            y = np.concatenate([r.write(s), r.finish()])
        return s, y

    alone = [run(i) for i in range(len(jobs))]
    got, errors = [None] * len(jobs), []
    gate = threading.Barrier(len(jobs))

    def worker(i):
        try:
            gate.wait()
            got[i] = run(i)
        except BaseException as e:  # noqa: B902 - re-raised below
            errors.append((i, e))

    th = [threading.Thread(target=worker, args=(i,)) for i in range(len(jobs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    for i in range(len(jobs)):
        assert np.array_equal(got[i][0], alone[i][0]) and np.array_equal(got[i][1], x)
        assert np.array_equal(alone[i][0], ctxs[i].compress(x, jobs[i][0], jobs[i][1], 1 << 20))
    for c in ctxs:
        c.close()


def set_length(s, rec, value):
    """s with the length field of the record whose prefix starts at bit rec[0] set to value (same lw)"""
    v, nbits = int.from_bytes(bytes(s), "big"), 8 * len(s)
    pos = rec[0]
    lw = ((v >> (nbits - pos - 5)) & 31) + 3
    shift = nbits - pos - 5 - lw
    v = (v & ~(((1 << lw) - 1) << shift)) | ((value & ((1 << lw) - 1)) << shift)
    return np.frombuffer(v.to_bytes(len(s), "big"), np.uint8).copy(), lw


def test_corrupt_record_length_matches_decompress(kz, gpu, oracle, synth):
    """one record's length raised or lowered: the walk runs into the payload, and the reader must report what kz_decompress_stream reports
    (a walk error found late beats every block-level failure found earlier)"""
    x = np.ascontiguousarray(synth.markov_text(14 * BS + 9, seed=41), np.uint8)
    big_cap = 1 << 26  # kz_decompress_stream's record count limit (cap / 1024 + 16) stays out of the way
    checked = 0
    for tr, en, ck in [("NONE", "NONE", 0), ("NONE", "NONE", 32), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0), ("LZ", "HUFFMAN", 64),
                       ("BWT+RANK+ZRLT", "ANS1", 0)]:
        s = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=len(x))
        recs = records(s)
        for k in (1, 6, len(recs) - 1):
            ln = recs[k][2]
            for value in (ln + 1, ln + 8, ln + 777, ln * 2, (1 << 40) - 1, ln - 1, ln - 9, ln // 2, 1):
                bad, lw = set_length(s, recs[k], value)
                if value >= 1 << lw and value != (1 << 40) - 1:
                    continue
                want = code_of(gpu, kz, bad, big_cap)
                for bb in (1, 3):
                    got, err = read_stream(gpu, bad, bb, [bad.size], 1 << 20)
                    assert err == want, (tr, en, ck, k, ln, value, bb, err, want)
                    if want == 0:
                        assert np.array_equal(got, gpu.decompress(bad, big_cap))
                checked += 1
    assert checked > 60


def test_reader_default_batch_follows_block_size(kz, synth):
    x = np.ascontiguousarray(synth.silesia_shaped(80 << 20, seed=17), np.uint8)
    ctx = kz.Context(0)
    s = ctx.compress(x, "NONE", "ANS0", 64 << 20, 0, x.size)
    with ctx.stream_reader() as r:  # about 256 MiB per batch: 4 blocks of 64 MiB, not 64
        y = np.concatenate([r.write(s[o: o + (1 << 20)]) for o in range(0, s.size, 1 << 20)] + [r.finish()])
        held = ctx.device_bytes()
    assert np.array_equal(y, x)
    assert held < 6 << 30, held
    ctx.close()


def test_context_closed_with_open_sessions(kz, synth):
    x = np.ascontiguousarray(synth.markov_text(300000, seed=5), np.uint8)
    ctx = kz.Context(0)
    w = ctx.stream_writer("LZ", "HUFFMAN", 1 << 16, batch_blocks=2)
    w.write(x)
    ctx.close()  # kz_destroy closes the session first
    with pytest.raises(kz.KanziError):
        w.write(x)
    w.close()
    ctx = kz.Context(0)
    s = ctx.compress(x, "LZ", "HUFFMAN", 1 << 16)
    r = ctx.stream_reader(batch_blocks=1)
    r.write(s[: s.size // 2])
    ctx.close()
    with pytest.raises(kz.KanziError):
        r.finish()
    r.close()
    h = C.c_void_p()  # a destroyed context's session handle answers -KZ_ERR_INVALID_PARAM until it is freed
    ctx = kz.Context(0)
    ctx._check(ctx.lib.kz_writer_open(ctx.h, kz.transform_type("LZ"), kz.entropy_type("HUFFMAN"), 1 << 16, 0, 2, 0, C.byref(h)))
    ctx.lib.kz_destroy(ctx.h)
    ctx.h = None
    made = C.c_size_t(0)
    out = np.empty(64, np.uint8)
    assert ctx.lib.kz_writer_finish(h, out.ctypes.data, out.size, C.byref(made)) == -18
    ctx.lib.kz_writer_free(h)
