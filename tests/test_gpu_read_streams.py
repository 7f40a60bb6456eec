"""GPU tests of the many-stream index build and range reads (kz_index_build_streams[_device], kz_read_ranges_streams[_device]) through
the C ABI and the Python wrappers. The yardstick is the one-stream call: every request gets what kz_read_ranges[_cached][_device] gives it
on its own stream, and the index of every stream is the one kz_index_build makes. Covered: equivalence over ~60 mixed streams on both
variants with guard bytes, the index build and its per-stream errors, the block cache, isolation of damaged, stale and unseekable
streams, call-level refusals, and the work bound (blocks decoded, uploads, launches that do not grow with the number of streams)."""
import ctypes as C

import numpy as np
import pytest

import index_oracle as io_
import range_oracle as ro
from test_gpu_block_cache import PAGE, cached_read, short_middle_block_stream
from test_gpu_block_range import CHAINS
from test_gpu_index import GUARD, abi_read, hl_args, hl_model, make, request_list, to_dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    yield t
    t.cuda.empty_cache()  # the streams and guarded destinations of this module's reads go back to the device with its context


@pytest.fixture(scope="module")
def gpu(kz):
    """A context of this module's own, closed at its end: the scratch its many-stream reads grow (staged requests of up to 4 MiB
    blocks, index builds over hundreds of streams) goes back to the device instead of staying with the session's shared context."""
    ctx = kz.Context(0)
    yield ctx
    ctx.close()


def layout(streams, device):
    """Offsets of the streams in one source buffer: 16-byte aligned with 64 bytes behind each on the device, odd gaps on the host."""
    off, at = [], 0
    for s in streams:
        off.append(at)
        at += len(s) + (64 if device else 3)
        if device:
            at = (at + 15) & ~15
    return np.array(off, np.uint64), at + 64


def streams_read(gpu, torch, streams, ixs, reqs, device, cache=None, src_off=None, caps=None):
    """One kz_read_ranges_streams[_device] call, requests [(stream, off, len)], guard bytes around every destination -> (rc, results).
    caps[s]: at least the decoded length of stream s, the most a request on it gets (default: what its index can decode,
    nblocks x block_size, so that a request of 1 << 62 bytes gets a destination of that size and no more)."""
    nreq = len(reqs)
    if caps is None:
        caps = [0 if x is None else x.info["nblocks"] * x.info["block_size"] for x in ixs]
    rs = np.array([r[0] for r in reqs] or [0], np.uint32)
    off = np.array([r[1] for r in reqs] or [0], np.uint64)
    ln = np.array([r[2] for r in reqs] or [0], np.uint64)
    cap = np.array([caps[r[0]] if r[0] < len(caps) else 0 for r in reqs] or [0], np.uint64)
    slot = np.minimum(ln, cap).astype(np.uint64)
    dst_off = (np.cumsum(slot + np.uint64(2 * GUARD)) - slot - np.uint64(GUARD)).astype(np.uint64)
    total = int((slot + np.uint64(2 * GUARD)).sum())
    so, size = layout(streams, device)
    if src_off is not None:
        so = np.array(src_off, np.uint64)
        size = int(max([int(o) + len(s) for o, s in zip(so, streams)] + [0])) + 128
    sl = np.array([len(s) for s in streams] or [0], np.uint64)
    buf = np.zeros(size, np.uint8)
    for o, s in zip(so, streams):
        buf[int(o): int(o) + len(s)] = s
    ix = (C.c_void_p * max(len(ixs), 1))(*[None if x is None else x.h for x in ixs])
    out_len, status = np.full(max(nreq, 1), 77, np.uint64), np.full(max(nreq, 1), 77, np.int32)
    ch = None if cache is None else cache.h
    args = (nreq, rs.ctypes.data, off.ctypes.data, ln.ctypes.data)
    if device:
        d_src = to_dev(torch, buf)
        d_dst = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        rc = gpu.lib.kz_read_ranges_streams_device(gpu.h, ch, len(streams), C.addressof(ix), d_src.data_ptr(), so.ctypes.data, sl.ctypes.data, *args,
                                                   d_dst.data_ptr(), dst_off.ctypes.data, out_len.ctypes.data, status.ctypes.data)
        dst = d_dst.cpu().numpy()
    else:
        dst = np.full(total + 64, 0xA5, np.uint8)
        rc = gpu.lib.kz_read_ranges_streams(gpu.h, ch, len(streams), C.addressof(ix), buf.ctypes.data, so.ctypes.data, sl.ctypes.data, *args,
                                            dst.ctypes.data, dst_off.ctypes.data, out_len.ctypes.data, status.ctypes.data)
    res, keep = [], np.ones(dst.size, bool)
    for i in range(nreq):
        o, n = int(dst_off[i]), int(out_len[i])
        assert n <= int(ln[i])
        res.append(("ok", dst[o: o + n].tobytes()) if status[i] == 0 else ("err", -int(status[i])))
        if status[i]:
            assert n == 0
        keep[o: o + n] = False
    assert (dst[keep] == 0xA5).all(), "bytes outside a delivered range were written"
    first_bad = next((int(c) for c in status[:nreq] if c), 0)
    assert rc == first_bad, (rc, first_bad)
    return rc, res


def per_stream(gpu, torch, streams, ixs, reqs, device, read=abi_read):
    """What one kz_read_ranges call per stream gives each request, in request order."""
    got = [None] * len(reqs)
    for s in sorted({r[0] for r in reqs}):
        idx = [i for i, r in enumerate(reqs) if r[0] == s]
        _, res = read(gpu, torch, ixs[s], streams[s], [reqs[i][1:] for i in idx], device)
        for i, g in zip(idx, res):
            got[i] = g
    return got


def mixed_streams(kz, oracle, synth):
    """About 60 streams: every chain of CHAINS headered and headerless, checksums 0 / 32 / 64, block sizes 1 KiB to 4 MiB, empty streams
    and streams under 16 bytes -> [(x, stream, headerless args or None, block size)]"""
    out = []
    chains = CHAINS + [("LZ", "HUFFMAN", 32), ("DNA+LZ", "HUFFMAN", 64)]
    for i, chain in enumerate(chains):
        for headerless in (False, True):
            for j, n in enumerate((0, 15, 1025, 5 * 1024 - 300)):
                if (i + j) % 3 == 2 and n == 0:
                    continue
                x, s = make(oracle, synth, chain, n, 1024, headerless, seed=3 + i + j)
                out.append((x, s, hl_args(kz, chain, 1024) if headerless else None, 1024))
    for chain, bs, n in ((CHAINS[4], 65536, 3 * 65536 + 5), (CHAINS[5], 4 << 20, (4 << 20) + 1), (("LZ", "HUFFMAN", 64), 4 << 20, 100000)):
        for headerless in (False, True):
            x, s = make(oracle, synth, chain, n, bs, headerless, seed=21)
            out.append((x, s, hl_args(kz, chain, bs) if headerless else None, bs))
    return out


@pytest.fixture(scope="module")
def corpus(kz, oracle, synth):
    return mixed_streams(kz, oracle, synth)


def test_equivalence_with_one_call_per_stream(kz, gpu, oracle, torch, corpus):
    rng = np.random.default_rng(31)
    streams = [s for _, s, _, _ in corpus]
    assert len(streams) >= 55
    reqs = [(k, o, n) for k, (x, s, hl, bs) in enumerate(corpus) for o, n in request_list(len(x), bs, rng)]
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    models = [io_.build(oracle, s, hl_model(hl) if hl else None) for _, s, hl, _ in corpus]
    want = [None] * len(reqs)
    for k in range(len(corpus)):
        idx = [i for i, r in enumerate(reqs) if r[0] == k]
        for i, w in zip(idx, io_.read(oracle, streams[k], models[k], [reqs[i][1:] for i in idx])):
            want[i] = w
    for device in (False, True):
        ix_one = [gpu.index(s, headerless=hl) for _, s, hl, _ in corpus]
        ix_all = [gpu.index(s, headerless=hl) for _, s, hl, _ in corpus]
        one = per_stream(gpu, torch, streams, ix_one, reqs, device)
        rc, got = streams_read(gpu, torch, streams, ix_all, reqs, device, caps=[len(x) + 16 for x, _, _, _ in corpus])
        assert rc == 0
        bad = [(reqs[i], got[i][0], one[i][0], want[i][0]) for i in range(len(reqs)) if not got[i] == one[i] == want[i]]
        assert not bad, bad[:5]
        assert [x.size for x in ix_all] == [x.size for x in ix_one] == [m["size"] for m in models]
        assert [x.save() for x in ix_all] == [x.save() for x in ix_one]
    # the Python wrappers: host and device
    ixs = [gpu.index(s, headerless=hl) for _, s, hl, _ in corpus]
    sub = [r for r in reqs if r[2] < 1 << 40][:300]
    want = [w for r, w in zip(reqs, want) if r[2] < 1 << 40][:300]
    outs, st = gpu.read_streams(streams, ixs, sub)
    assert [("ok", o) if c == 0 else ("err", -c) for o, c in zip(outs, st)] == want[:300]
    so, size = layout(streams, True)
    buf = np.zeros(size, np.uint8)
    for o, s in zip(so, streams):
        buf[int(o): int(o) + len(s)] = s
    ok = [i for i in range(len(sub)) if want[i][0] == "ok"]
    lens = [len(want[i][1]) for i in ok]
    d_dst = torch.zeros(sum(lens) + 1, dtype=torch.uint8, device="cuda")
    out_len, st = gpu.read_streams_device(to_dev(torch, buf), so, [len(s) for s in streams], ixs, [sub[i][0] for i in ok], [sub[i][1] for i in ok],
                                          lens, d_dst, np.cumsum([0] + lens[:-1]))
    assert not st.any() and out_len.tolist() == lens
    assert d_dst.cpu().numpy()[: sum(lens)].tobytes() == b"".join(want[i][1] for i in ok)


def test_index_build_matches_one_build_per_stream(kz, gpu, oracle, synth, torch, corpus):
    headered = [s for _, s, hl, _ in corpus if hl is None]
    s0 = headered[5]
    hb = ro.header_bits(s0)
    bad_header = np.array(s0)
    bad_header[0] ^= 0x40
    bad_len = ro.flip(s0, hb, 1)  # the first record's length field grows by 16 bits: a length past the end
    streams = headered + [bad_header, s0[: len(s0) // 2], bad_len, s0[:3]]
    want = []
    for s in streams:
        try:
            want.append(("ok", gpu.index(s).save()))
        except kz.KanziError as e:
            want.append(("err", e.code))
    assert sum(w[0] == "err" for w in want[-4:]) >= 3
    for device in (False, True):
        if device:
            so, size = layout(streams, True)
            buf = np.zeros(size, np.uint8)
            for o, s in zip(so, streams):
                buf[int(o): int(o) + len(s)] = s
            ixs, st = gpu.index_streams_device(to_dev(torch, buf), so, [len(s) for s in streams])
        else:
            ixs, st = gpu.index_streams(streams)
        got = [("ok", x.save()) if x is not None else ("err", -int(c)) for x, c in zip(ixs, st)]
        assert [x is None for x in ixs] == [c != 0 for c in st]
        assert got == want
    # the headerless setting applies to every stream
    for chain in (CHAINS[1], CHAINS[6]):
        hl = hl_args(kz, chain, 1024)
        hs = [s for _, s, h, _ in corpus if h == hl]
        ixs, st = gpu.index_streams(hs, headerless=hl)
        assert not st.any() and [x.save() for x in ixs] == [gpu.index(s, headerless=hl).save() for s in hs]
    # one gather launch and two walk launches, for 3 streams as for 300
    small, _ = gpu.compress_streams([synth.markov_text(1500 + 37 * i, seed=i) for i in range(300)], "LZ", "HUFFMAN", 1024)
    counts = []
    for n in (3, 300):
        gpu.launch_count(reset=True)
        ixs, st = gpu.index_streams(small[:n])
        counts.append(gpu.launch_count())
        assert not st.any() and [x.save() for x in ixs[:3]] == [gpu.index(s).save() for s in small[:3]]
    assert counts[0] == counts[1] == 3, counts


def test_cache_budgets_give_the_same_results(kz, gpu, oracle, synth, torch):
    rng = np.random.default_rng(32)
    items = [make(oracle, synth, CHAINS[i % len(CHAINS)], 6 * 1024 - 100 * i, 1024, False, seed=40 + i) for i in range(14)]
    xs, streams = [x for x, _ in items], [s for _, s in items]
    streams.append(streams[2].copy())  # identical records in two slots
    xs.append(xs[2])
    reqs = [(k, o, n) for k, x in enumerate(xs) for o, n in request_list(len(x), 1024, rng)]
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    blocks_all = sum(gpu.index(s).info["nblocks"] for s in streams)  # every block takes at least one page
    for device in (False, True):
        want = streams_read(gpu, torch, streams, [gpu.index(s) for s in streams], reqs, device)
        for budget in (0, blocks_all * PAGE // 4, blocks_all * PAGE):
            ixs = [gpu.index(s) for s in streams]
            with gpu.block_cache(budget) as cache:
                assert streams_read(gpu, torch, streams, ixs, reqs, device, cache) == want, budget
                st1 = cache.stats
                gpu.profile(True)
                try:
                    gpu.profile_reset()
                    assert streams_read(gpu, torch, streams, ixs, reqs, device, cache) == want, budget
                    blocks = gpu.stage_bytes("read:blocks")[1]
                finally:
                    gpu.profile(False)
                    gpu.profile_reset()
                st2 = cache.stats
                pairs = st1["hits"] + st1["misses"]
                assert st2["hits"] + st2["misses"] - pairs == pairs
                assert st1["inserts"] - st1["evictions"] == st1["entries"]
                if budget == blocks_all * PAGE:
                    # a repeated call is all hits; the copy of stream 2 shares its entries
                    assert blocks == 0 and st2["hits"] - st1["hits"] == pairs and st2["misses"] == st1["misses"]
                    nb2 = gpu.index(streams[2]).info["nblocks"]
                    assert st1["entries"] == st1["misses"] - nb2 and st1["inserts"] == st1["entries"]


def test_isolation_of_damaged_stale_and_unseekable_streams(kz, gpu, oracle, synth, torch):
    rng = np.random.default_rng(33)
    chain = ("LZ", "HUFFMAN", 32)
    good = [make(oracle, synth, CHAINS[i], 5 * 1024 - 7 * i, 1024, False, seed=50 + i) for i in range(4)]
    x_d, s_d = make(oracle, synth, chain, 6 * 1024, 1024, False, seed=60)
    recs = ro.walk(s_d, ro.header_bits(s_d))
    damaged = ro.corrupt(s_d, recs[2], "checksum")
    stale = np.array(good[1][1])
    stale[3] ^= 0xFF
    short = short_middle_block_stream(oracle, synth, chain, 1024)
    hl = hl_args(kz, chain, 1024)
    streams = [good[0][1], damaged, stale, good[2][1], short, good[3][1]]
    xs = [good[0][0], x_d, good[1][0], good[2][0], None, good[3][0]]
    reqs = []
    for k, x in enumerate(xs):
        n = len(x) if x is not None else 6 * 1024
        reqs += [(k, o, ln) for o, ln in request_list(n, 1024, rng)]
    reqs += [(1, 2 * 1024 + 5, 10), (4, 3 * 1024 + 1, 4), (4, 5, 4)]
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    for device in (False, True):
        def indexes():
            return [gpu.index(streams[0]), gpu.index(damaged), gpu.index(good[1][1]), gpu.index(streams[3]), gpu.index(short, headerless=hl),
                    gpu.index(streams[5])]
        ix_one, ix_all = indexes(), indexes()
        one = per_stream(gpu, torch, streams, ix_one, reqs, device)
        rc, got = streams_read(gpu, torch, streams, ix_all, reqs, device)
        assert got == one
        assert rc == next((-g[1] for g in got if g[0] == "err"), 0)
        for (k, o, n), g in zip(reqs, got):
            if k == 2:
                assert g == ("err", 18)
            elif k in (0, 3, 5) and n and o < len(xs[k]):
                assert g == ("ok", xs[k][o: o + n].tobytes())
            elif k == 1 and n and o < len(x_d) and not (o // 1024 <= 2 <= (min(o + n, len(x_d)) - 1) // 1024):
                assert g == ("ok", x_d[o: o + n].tobytes())
            elif k == 4 and n and o >= 3 * 1024 and o < 6 * 1024:
                assert g == ("err", 15)
        assert any(g[0] == "err" and k == 1 for (k, _, _), g in zip(reqs, got))
        assert [x.size for x in ix_all] == [x.size for x in ix_one]
    # a NULL index and a loaded index that names a chain without a GPU path fail only their stream, with kz_read_ranges's code
    srt = kz.StreamIndex.load(io_.blob(dict(io_.build(oracle, streams[0]), transform48=kz.transform_type("SRT"))), gpu)
    for device in (False, True):
        single = abi_read(gpu, torch, srt, streams[0], [(0, 10)], device)
        assert single == (-14, [("err", 14)])
        rc, got = streams_read(gpu, torch, [streams[0], streams[3], streams[0]], [None, gpu.index(streams[3]), srt], [(0, 0, 10), (1, 0, 10), (2, 0, 10)],
                               device)
        assert got == [("err", 18), ("ok", good[2][0][:10].tobytes()), ("err", 14)] and rc == -18


def test_call_level_refusals_write_nothing(kz, gpu, oracle, synth, torch):
    items = [make(oracle, synth, CHAINS[4], 3 * 1024 + i, 1024, False, seed=70 + i) for i in range(3)]
    streams = [s for _, s in items]
    reqs = [(0, 0, 10), (2, 5, 100), (1, 1024, 50)]

    def refused(rc_got):
        rc, got = rc_got
        assert rc == -18 and got == [("err", 18)] * len(got), rc_got

    for device in (False, True):
        ixs = [gpu.index(s) for s in streams]
        refused(streams_read(gpu, torch, streams, ixs, reqs + [(3, 0, 1)], device))
        if device:
            refused(streams_read(gpu, torch, streams, ixs, reqs, True, src_off=[0, 4096 + 8, 8192]))
        other = kz.Context(0)
        try:
            with other.block_cache(16 * PAGE) as foreign:
                refused(streams_read(gpu, torch, streams, ixs, reqs, device, foreign))
        finally:
            other.close()
        r = gpu.stream_reader(batch_blocks=2)
        try:
            refused(streams_read(gpu, torch, streams, ixs, reqs, device))
            st = np.zeros(len(streams), np.int32)
            hs = (C.c_void_p * len(streams))()
            src = np.concatenate(streams)
            lens = np.array([len(s) for s in streams], np.uint64)
            offs = np.cumsum(np.r_[0, lens[:-1]]).astype(np.uint64)
            assert gpu.lib.kz_index_build_streams(gpu.h, len(streams), src.ctypes.data, offs.ctypes.data, lens.ctypes.data, C.addressof(hs),
                                                  st.ctypes.data) == -18
            assert (st == -18).all() and not any(hs)
        finally:
            r.close()
        assert streams_read(gpu, torch, streams, ixs, reqs, device)[0] == 0
    # a stream no request names is neither checked nor read: a NULL index and a misaligned offset there are fine
    ixs = [gpu.index(s) for s in streams]
    rc, got = streams_read(gpu, torch, streams, [ixs[0], None, ixs[2]], [(0, 0, 10), (2, 0, 10)], True, src_off=[0, 4096 + 8, 8192])
    assert rc == 0 and got == [("ok", items[0][0][:10].tobytes()), ("ok", items[2][0][:10].tobytes())]


def test_work_follows_blocks_not_streams(kz, gpu, oracle, synth, torch, corpus):
    rng = np.random.default_rng(34)
    sub = [c for c in corpus if c[3] == 1024][:30]
    streams = [s for _, s, _, _ in sub]
    reqs = [(k, int(o), int(n)) for k, (x, _, _, _) in enumerate(sub) if len(x) for o, n in zip(rng.integers(0, len(x), 12), rng.integers(0, 1500, 12))]
    for device in (False, True):
        ixs = [gpu.index(s, headerless=hl) for _, s, hl, _ in sub]
        pairs = {(k, b) for k, o, n in reqs if n for b in range(o // 1024, (min(o + n, ixs[k].info["nblocks"] * 1024) - 1) // 1024 + 1)}
        gpu.profile(True)
        try:
            gpu.profile_reset()
            rc, _ = streams_read(gpu, torch, streams, ixs, reqs, device)
            assert rc == 0
            assert gpu.stage_bytes("read:blocks")[1] == len(pairs)
            if device:
                assert gpu.stage_bytes("read:h2d")[0] == 0
        finally:
            gpu.profile(False)
            gpu.profile_reset()
    # S one-block streams of identical content: the same launches for 4 as for 64
    x = np.ascontiguousarray(synth.markov_text(900, seed=9), np.uint8)
    s = gpu.compress(x, "LZ", "HUFFMAN", block_size=1024, input_size=len(x))
    for device in (False, True):
        counts = []
        for S in (4, 64):
            ixs = [gpu.index(s) for _ in range(S)]
            rq = [(k, 7 * k % 800, 50) for k in range(S)]
            gpu.launch_count(reset=True)
            rc, got = streams_read(gpu, torch, [s] * S, ixs, rq, device)
            counts.append(gpu.launch_count())
            assert rc == 0 and got == [("ok", x[o: o + n].tobytes()) for _, o, n in rq]
        assert counts[0] == counts[1], (device, counts)


@pytest.mark.parametrize("cached", [False, True], ids=["uncached", "cached"])
def test_one_stream_call_matches_the_single_stream_read(kz, gpu, oracle, synth, torch, cached):
    rng = np.random.default_rng(35)
    x, s = make(oracle, synth, CHAINS[3], 9 * 1024 - 50, 1024, False, seed=80)
    reqs = request_list(len(x), 1024, rng)
    names = ["read:blocks", "read:h2d", "read:out", "read:cache_hit", "read:cache_miss", "read:cache_insert", "read:cache_evict"]
    for device in (False, True):
        results = []
        for streams_call in (False, True):
            ix = gpu.index(s)
            cache = gpu.block_cache(8 * PAGE) if cached else None
            gpu.profile(True)
            try:
                gpu.profile_reset()
                gpu.launch_count(reset=True)
                for _ in range(2):
                    if streams_call:
                        r = streams_read(gpu, torch, [s], [ix], [(0, o, n) for o, n in reqs], device, cache)
                    elif cached:
                        r = cached_read(gpu, torch, ix, s, reqs, device, cache)
                    else:
                        r = abi_read(gpu, torch, ix, s, reqs, device)
                launches = gpu.launch_count()
                counters = {k: gpu.stage_bytes(k) for k in names}
            finally:
                gpu.profile(False)
                gpu.profile_reset()
                if cache is not None:
                    cache.close()
            results.append((r, launches, counters, ix.size))
        assert results[0] == results[1], (device, results[0][1:], results[1][1:])
