"""GPU tests of the block cache (kz_cache_*, kz_read_ranges_cached[_device]): a cached read returns what kz_read_ranges returns for the
same arguments on every level chain, headered and headerless, with and without checksums, on both variants, over repeated calls; a
repeated call decodes nothing; eviction follows LRU exactly; entries are keyed by record content (two streams that share length and head,
a loaded and a headerless index, host and device variants); failing blocks are never cached; a short middle block keeps its pattern;
the refusals; and device memory that is the budget, allocated once."""
import numpy as np
import pytest

import headerless_oracle as ho
import range_oracle as ro
from test_gpu_index import GUARD, abi_read, hl_args, make, request_list, to_dev

pytestmark = pytest.mark.gpu

LEVELS = [("NONE", "NONE"), ("LZX", "NONE"), ("DNA+LZ", "HUFFMAN"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")]
PAGE = 64 << 10


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def cached_read(gpu, torch, ix, s, reqs, device, cache):
    """abi_read through kz_read_ranges_cached[_device]: guard bytes around every destination -> (return value, results)."""
    nreq = len(reqs)
    off = np.array([r[0] for r in reqs] or [0], np.uint64)
    ln = np.array([r[1] for r in reqs] or [0], np.uint64)
    slot = np.minimum(ln, np.uint64(1 << 26)).astype(np.uint64)
    dst_off = (np.cumsum(slot + np.uint64(2 * GUARD)) - slot - np.uint64(GUARD)).astype(np.uint64)
    total = int((slot + np.uint64(2 * GUARD)).sum())
    out_len, status = np.full(max(nreq, 1), 77, np.uint64), np.full(max(nreq, 1), 77, np.int32)
    s = np.ascontiguousarray(s, np.uint8)
    args = (nreq, off.ctypes.data, ln.ctypes.data)
    if device:
        d_src = to_dev(torch, s)
        d_dst = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        rc = gpu.lib.kz_read_ranges_cached_device(gpu.h, cache.h, ix.h, d_src.data_ptr(), len(s), *args, d_dst.data_ptr(), dst_off.ctypes.data,
                                                  out_len.ctypes.data, status.ctypes.data)
        dst = d_dst.cpu().numpy()
    else:
        dst = np.full(total + 64, 0xA5, np.uint8)
        rc = gpu.lib.kz_read_ranges_cached(gpu.h, cache.h, ix.h, s.ctypes.data, len(s), *args, dst.ctypes.data, dst_off.ctypes.data, out_len.ctypes.data,
                                           status.ctypes.data)
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


class Profile:
    def __init__(self, gpu):
        self.gpu = gpu

    def __enter__(self):
        self.gpu.profile(True)
        self.gpu.profile_reset()
        return self

    def __exit__(self, *exc):
        self.gpu.profile(False)
        self.gpu.profile_reset()

    def call(self, f):
        """f() under a fresh profile -> (its result, {counter: (bytes_in, bytes_out)})"""
        self.gpu.profile_reset()
        r = f()
        names = ["read:blocks", "read:h2d", "read:cache_hit", "read:cache_miss", "read:cache_insert", "read:cache_evict"]
        return r, {k: self.gpu.stage_bytes(k)[1:] for k in names}


@pytest.mark.parametrize("headerless", [False, True], ids=["headered", "headerless"])
@pytest.mark.parametrize("level", range(6), ids=["l%d" % k for k in range(6)])
def test_cached_reads_equal_uncached_reads(kz, gpu, oracle, synth, torch, level, headerless):
    bs, nb = 1024, 12
    rng = np.random.default_rng(20 + level)
    for ck in (0, 32):
        chain = LEVELS[level] + (ck,)
        hl = hl_args(kz, chain, bs) if headerless else None
        x, s = make(oracle, synth, chain, nb * bs - 300, bs, headerless, seed=level + 3)
        ix_u, ix_c = gpu.index(s, headerless=hl), gpu.index(s, headerless=hl)
        with gpu.block_cache(6 * PAGE) as cache:  # half the blocks: calls evict
            for call in range(5):
                reqs = request_list(len(x), bs, rng) if call % 2 == 0 else [(int(o), 700) for o in rng.integers(0, 4 * bs, 20)]
                for device in (False, True):
                    want = abi_read(gpu, torch, ix_u, s, reqs, device)
                    got = cached_read(gpu, torch, ix_c, s, reqs, device, cache)
                    assert got == want, (chain, call, device)
                    assert ix_c.size == ix_u.size
                    for (o, n), w in zip(reqs, want[1]):
                        assert w == ("ok", x[o: o + n].tobytes())
            st = cache.stats
            assert st["hits"] > 0 and st["evictions"] > 0 and st["entries"] <= 6 and st["resident_bytes"] <= 6 * bs


def test_a_repeated_call_decodes_nothing(kz, gpu, synth, torch):
    bs = 64 << 10
    x = np.ascontiguousarray(synth.silesia_shaped(8 * bs - 100, seed=21), np.uint8)
    s = gpu.compress(x, "TEXT+UTF+PACK+MM+LZX", "HUFFMAN", block_size=bs, input_size=len(x))
    ix = gpu.index(s)
    reqs = [(k * bs + 17 * k, 4096) for k in range(8)] + [(3 * bs - 10, 20)]
    want = [x[o: o + n].tobytes() for o, n in reqs]
    with gpu.block_cache(16 * PAGE) as cache, Profile(gpu) as P:
        (outs, st), c = P.call(lambda: ix.read_many(s, reqs, cache=cache))
        assert outs == want and not any(st)
        assert c["read:blocks"] == (8, len(x)) and c["read:cache_miss"] == (8, len(x)) and c["read:cache_insert"] == (8, len(x))
        assert c["read:cache_hit"] == (0, 0)
        (outs, st), c = P.call(lambda: ix.read_many(s, reqs, cache=cache))
        assert outs == want and not any(st)
        assert c["read:blocks"] == (0, 0) and c["read:cache_hit"] == (8, len(x)) and c["read:h2d"] == (0, 0)
        assert c["read:cache_miss"] == (0, 0) and c["read:cache_insert"] == (0, 0)
        # the device variant: hashed on the device, one launch for the tiles and one for the roots
        d_src, d_dst = to_dev(torch, s), torch.zeros(len(reqs) * 4096, dtype=torch.uint8, device="cuda")
        gpu.profile_reset()
        out_len, st = ix.read_many_device(d_src, len(s), [r[0] for r in reqs], [r[1] for r in reqs], d_dst, [4096 * i for i in range(len(reqs))],
                                          cache=cache)
        assert not st.any() and gpu.stage_bytes("read:blocks")[1:] == (0, 0) and gpu.kernel_time("record_hash")[0] == 2
        got = d_dst.cpu().numpy()
        assert all(got[4096 * i: 4096 * i + n].tobytes() == w for i, ((o, n), w) in enumerate(zip(reqs, want)))
        assert cache.stats["served_bytes"] == 2 * sum(len(w) for w in want)


def test_eviction_is_lru(kz, gpu, synth):
    bs = 64 << 10
    x = np.ascontiguousarray(synth.markov_text(6 * bs, seed=22), np.uint8)
    s = gpu.compress(x, "LZ", "HUFFMAN", block_size=bs, input_size=len(x))
    ix = gpu.index(s)
    with gpu.block_cache(2 * PAGE) as cache, Profile(gpu) as P:  # two blocks
        decoded = []
        for k in (0, 1, 2, 0, 2, 1, 0, 1):
            out, c = P.call(lambda: ix.read(s, k * bs + 5, 100, cache=cache))
            assert out == x[k * bs + 5: k * bs + 105].tobytes()
            decoded.append(c["read:blocks"][0])
        assert decoded == [1, 1, 1, 1, 0, 1, 1, 0]
        st = cache.stats
        assert (st["entries"], st["hits"], st["misses"], st["inserts"], st["evictions"]) == (2, 2, 6, 6, 4)
        cache.clear()
        assert cache.stats["entries"] == 0 and cache.stats["resident_bytes"] == 0
        _, c = P.call(lambda: ix.read(s, 5, 100, cache=cache))
        assert c["read:blocks"][0] == 1
    # a block larger than the whole budget is served and not inserted; a budget of 0 caches nothing
    for budget in (PAGE // 2, 0):
        with gpu.block_cache(budget) as cache:
            for _ in range(2):
                assert ix.read(s, bs - 50, 100, cache=cache) == x[bs - 50: bs + 50].tobytes()
            assert cache.stats["entries"] == 0 and cache.stats["inserts"] == 0 and cache.stats["misses"] == 4
    big = np.ascontiguousarray(synth.markov_text(3 * 2 * bs, seed=23), np.uint8)
    sb = gpu.compress(big, "LZ", "HUFFMAN", block_size=2 * bs, input_size=len(big))
    ixb = gpu.index(sb)
    with gpu.block_cache(PAGE) as cache:
        for _ in range(2):
            assert ixb.read(sb, 2 * bs + 3, 10, cache=cache) == big[2 * bs + 3: 2 * bs + 13].tobytes()
        assert cache.stats["inserts"] == 0


def test_two_streams_with_the_same_head_keep_their_own_bytes(kz, gpu, oracle, synth, torch):
    bs, nb = 1024, 8
    a = np.ascontiguousarray(synth.markov_text(nb * bs, seed=24), np.uint8)
    b = a.copy()
    b[3 * bs + 100: 3 * bs + 140] ^= 0x5A  # block 3 only
    sa = oracle.compress(a, "NONE", "NONE", block_size=bs, input_size=len(a))
    sb = oracle.compress(b, "NONE", "NONE", block_size=bs, input_size=len(b))
    assert len(sa) == len(sb) and bytes(sa[:32]) == bytes(sb[:32]) and bytes(sa) != bytes(sb)
    ix = gpu.index(sa)
    reqs = [(3 * bs + 90, 60), (2 * bs, 3 * bs), (0, 10)]
    with gpu.block_cache(16 * PAGE) as cache:
        for rnd in range(2):
            for device in (False, True):
                for s, x in ((sa, a), (sb, b)):
                    rc, got = cached_read(gpu, torch, ix, s, reqs, device, cache)
                    assert rc == 0 and got == [("ok", x[o: o + n].tobytes()) for o, n in reqs], (rnd, device)
        assert cache.stats["entries"] == nb // 2 + 1  # blocks 0, 2, 3, 4 of either stream and block 3 of the other


def test_failing_blocks_are_never_cached(kz, gpu, oracle, synth, torch):
    bs, nb = 1024, 12
    for chain in (("LZ", "HUFFMAN", 32), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0)):
        x, s = make(oracle, synth, chain, nb * bs - 300, bs, False, seed=25)
        recs = ro.walk(s, ro.header_bits(s))
        for kind in ["header"] + (["checksum"] if chain[2] else []):
            victim = 5
            bad = ro.corrupt(s, recs[victim], kind)
            ix = gpu.index(bad)
            reqs = [(k * bs + 3, 50) for k in range(nb)] + [(victim * bs - 10, 20), (0, nb * bs)]
            want = abi_read(gpu, torch, ix, bad, reqs, False)
            assert want[1][victim][0] == "err" and want[1][0] == ("ok", x[3:53].tobytes())
            with gpu.block_cache(32 * PAGE) as cache, Profile(gpu) as P:
                for call in range(3):
                    for device in (False, True):
                        got, c = P.call(lambda: cached_read(gpu, torch, ix, bad, reqs, device, cache))
                        assert got == want, (chain, kind, call, device)
                        assert c["read:cache_miss"][0] == (nb if call == 0 and not device else 1)
                assert cache.stats["entries"] == nb - 1 and cache.stats["inserts"] == nb - 1


def short_middle_block_stream(oracle, synth, chain, bs):
    """records of blocks 0..2, a block of bs - 16 bytes, then blocks 4..5: a stream no kanzi writer produces (as in test_gpu_index)"""
    x = np.ascontiguousarray(synth.markov_text(6 * bs, seed=4), np.uint8)
    pieces = [x[0: bs], x[bs: 2 * bs], x[2 * bs: 3 * bs], x[3 * bs: 4 * bs - 16], x[4 * bs: 5 * bs], x[5 * bs:]]
    body = ho.records(oracle, np.concatenate(pieces[:3]), *chain[:2], bs, chain[2])
    parts = [np.unpackbits(body)[: ho.end_bit(body, 0) - 8]]
    for p in pieces[3:]:
        r = ho.records(oracle, p, *chain[:2], bs, chain[2])
        parts.append(np.unpackbits(r)[: ho.end_bit(r, 0) - 8])
    return np.packbits(np.concatenate(parts + [np.zeros(8, np.uint8)]))


def test_a_short_middle_block_keeps_its_pattern_hit_or_miss(kz, gpu, oracle, synth, torch):
    bs = 1024
    chain = ("LZ", "HUFFMAN", 32)
    s = short_middle_block_stream(oracle, synth, chain, bs)
    hl = hl_args(kz, chain, bs)
    reqs = [(0, 10), (2 * bs + 5, 100), (3 * bs - 5, 10), (3 * bs, 1), (4 * bs, 10), (5 * bs + 1, 5), (bs, bs), (2 * bs, 3 * bs)]
    ix_u, ix_c = gpu.index(s, headerless=hl), gpu.index(s, headerless=hl)
    want = abi_read(gpu, torch, ix_u, s, reqs, False)
    assert [w[0] for w in want[1]] == ["ok", "ok", "err", "err", "err", "err", "ok", "err"] and want[0] == -15
    with gpu.block_cache(32 * PAGE) as cache:
        # block 3 alone first: a miss in a call of its own, then a hit under the other requests
        for sel in ([3], list(range(len(reqs))), list(range(len(reqs))), [2, 5], [0, 3]):
            sub = [reqs[i] for i in sel]
            for device in (False, True):
                assert cached_read(gpu, torch, ix_c, s, sub, device, cache) == abi_read(gpu, torch, ix_u, s, sub, device), sel
        assert cache.stats["hits"] > 0
    assert ix_c.size == ix_u.size == -1


def test_other_indexes_and_the_other_variant_hit_the_same_entries(kz, gpu, oracle, synth, torch):
    bs, chain = 4096, ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 32)
    x, s = make(oracle, synth, chain, 10 * bs - 77, bs, False, seed=26)
    _, shl = make(oracle, synth, chain, 10 * bs - 77, bs, True, seed=26)
    hl = hl_args(kz, chain, bs)
    ix = gpu.index(s)
    reqs = [(k * bs + 11, 300) for k in range(10)]
    want = [x[o: o + n].tobytes() for o, n in reqs]
    with gpu.block_cache(16 * PAGE) as cache, Profile(gpu) as P:
        d_src, d_dst = to_dev(torch, s), torch.zeros(300 * len(reqs), dtype=torch.uint8, device="cuda")
        (out_len, st), c = P.call(lambda: ix.read_many_device(d_src, len(s), [r[0] for r in reqs], [300] * len(reqs), d_dst,
                                                              [300 * i for i in range(len(reqs))], cache=cache))
        assert not st.any() and c["read:blocks"][0] == 10 and d_dst.cpu().numpy().tobytes() == b"".join(want)
        # the host variant hits what the device variant inserted
        (outs, st), c = P.call(lambda: ix.read_many(s, reqs, cache=cache))
        assert outs == want and not any(st) and c["read:blocks"] == (0, 0) and c["read:h2d"] == (0, 0) and c["read:cache_hit"][0] == 10
        # a loaded index, and the index of the headerless stream of the same data (its records start at other bits)
        loaded = kz.StreamIndex.load(ix.save(), gpu)
        ixh = gpu.index(shl, headerless=hl)
        for other, stream in ((loaded, s), (ixh, shl)):
            for device in (False, True):
                (rc, got), c = P.call(lambda: cached_read(gpu, torch, other, stream, reqs, device, cache))
                assert rc == 0 and got == [("ok", w) for w in want] and c["read:blocks"] == (0, 0)
        assert cache.stats["entries"] == 10 and cache.stats["inserts"] == 10
        assert ixh.size == loaded.size == len(x)


def test_refusals(kz, gpu, oracle, synth, torch):
    bs = 1024
    x, s = make(oracle, synth, ("LZ", "HUFFMAN", 0), 5 * bs, bs, False)
    ix = gpu.index(s)
    other = kz.Context(0)
    try:
        with other.block_cache(PAGE) as foreign:
            for device in (False, True):
                assert cached_read(gpu, torch, ix, s, [(0, 10), (bs, 5)], device, foreign) == (-18, [("err", 18)] * 2)
        st = np.zeros(1, np.int32)
        assert gpu.lib.kz_read_ranges_cached(gpu.h, None, ix.h, s.ctypes.data, len(s), 1, None, None, None, None, None, st.ctypes.data) == -18
        assert st[0] == -18
        # a cache whose context was destroyed first answers INVALID_PARAM and is still freed
        orphan = other.block_cache(PAGE)
        other.close()
        assert gpu.lib.kz_cache_clear(orphan.h) == -18 and orphan.stats["budget_bytes"] == PAGE
        orphan.close()
    finally:
        other.close()
    with gpu.block_cache(4 * PAGE) as cache:
        r = gpu.stream_reader(batch_blocks=2)
        try:
            assert cached_read(gpu, torch, ix, s, [(0, 10)], False, cache) == (-18, [("err", 18)])
        finally:
            r.close()
        assert cached_read(gpu, torch, ix, s, [(0, 10)], True, cache) == (0, [("ok", x[:10].tobytes())])
        assert cache.stats["entries"] == 1


def test_device_memory_is_the_budget_allocated_once(kz, synth):
    bs = 64 << 10
    ctx = kz.Context(0)
    try:
        x = np.ascontiguousarray(synth.silesia_shaped(40 * bs, seed=27), np.uint8)
        s = ctx.compress(x, "TEXT+UTF+PACK+MM+LZX", "HUFFMAN", block_size=bs, input_size=len(x))
        ix = ctx.index(s)
        rng = np.random.default_rng(28)
        ix.read_many(s, [(0, len(x))])  # the context's scratch for one pass over every block of the stream
        base = ctx.device_bytes()
        budget = 48 << 20
        cache = ctx.block_cache(budget + 1000)  # rounded down to whole pages
        assert ctx.device_bytes() - base == budget
        sets = [[(int(o), 4096) for o in rng.zipf(1.3, 200) % len(x)] for _ in range(6)]
        sizes = []
        for rnd in range(4):  # the same calls again and again: the cache fills, the memory stays
            for reqs in sets:
                outs, st = ix.read_many(s, reqs, cache=cache)
                assert not any(st) and all(o == x[a: a + n].tobytes() for o, (a, n) in zip(outs, reqs))
            sizes.append(ctx.device_bytes())
        assert sizes[-1] - base <= budget + (1 << 20), sizes  # the budget, and no more scratch than one pass of this stream
        assert sizes[-1] - sizes[0] <= 1 << 20, sizes  # never with the number of calls
        assert cache.stats["hits"] > 0
        cache.close()
        assert ctx.device_bytes() == sizes[-1] - budget
    finally:
        ctx.close()
