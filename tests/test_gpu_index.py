"""GPU tests of the stream index and the batched range reads (kz_index_*, kz_read_ranges[_device]) through the C ABI and the Python
wrappers, against the model of tests/index_oracle.py: the index and its blob, every kind of request on headered and headerless streams of
many shapes, bytes around each destination, host against device variant, a loaded index, a stale index, damaged and short blocks, the
work a call does (kz_profile), and the session rule."""
import ctypes as C

import numpy as np
import pytest

import headerless_oracle as ho
import index_oracle as io_
import range_oracle as ro
from test_gpu_block_range import CHAINS, IDS

pytestmark = pytest.mark.gpu

GUARD = 24


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def to_dev(torch, a, extra=64):
    d = torch.zeros(len(a) + extra, dtype=torch.uint8, device="cuda")
    if len(a):
        d[: len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    return d


def hl_args(kz, chain, bs):
    return {"transform": kz.transform_type(chain[0]), "entropy": kz.entropy_type(chain[1]), "block_size": bs, "checksum_bits": chain[2]}


def hl_model(a):
    return {"transform48": a["transform"], "entropy": a["entropy"], "block_size": a["block_size"], "checksum_bits": a["checksum_bits"]}


def make(oracle, synth, chain, n, bs, headerless, seed=5):
    tr, en, ck = chain
    x = np.ascontiguousarray(synth.markov_text(max(n, 1), seed=seed)[:n], np.uint8)
    if headerless:
        return x, ho.compress(oracle, x, tr, en, bs, ck)
    return x, oracle.compress(x, tr, en, block_size=bs, checksum_bits=ck, input_size=n)


def abi_read(gpu, torch, ix, s, reqs, device):
    """One kz_read_ranges[_device] call with guard bytes around every destination -> (return value, [("ok", bytes) | ("err", code)])."""
    nreq = len(reqs)
    off = np.array([r[0] for r in reqs] or [0], np.uint64)
    ln = np.array([r[1] for r in reqs] or [0], np.uint64)
    slot = np.minimum(ln, np.uint64(1 << 26)).astype(np.uint64)  # what the test gives a huge request; the stream is shorter
    dst_off = (np.cumsum(slot + np.uint64(2 * GUARD)) - slot - np.uint64(GUARD)).astype(np.uint64)
    total = int((slot + np.uint64(2 * GUARD)).sum())
    out_len, status = np.full(max(nreq, 1), 77, np.uint64), np.full(max(nreq, 1), 77, np.int32)
    s = np.ascontiguousarray(s, np.uint8)
    args = (nreq, off.ctypes.data, ln.ctypes.data)
    if device:
        d_src = to_dev(torch, s)
        d_dst = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        rc = gpu.lib.kz_read_ranges_device(gpu.h, ix.h, d_src.data_ptr(), len(s), *args, d_dst.data_ptr(), dst_off.ctypes.data, out_len.ctypes.data,
                                           status.ctypes.data)
        dst = d_dst.cpu().numpy()
    else:
        dst = np.full(total + 64, 0xA5, np.uint8)
        rc = gpu.lib.kz_read_ranges(gpu.h, ix.h, s.ctypes.data, len(s), *args, dst.ctypes.data, dst_off.ctypes.data, out_len.ctypes.data, status.ctypes.data)
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


def request_list(n, bs, rng):
    """Every kind of request on a stream of n decoded bytes"""
    r = [(0, n), (0, 0), (n, 0), (n, 10), (n + 5 * bs, 100), (1 << 62, 1 << 62), (0, n + 100), (max(n - 7, 0), 7), (max(n - 7, 0), 50)]
    if n:
        r += [(n // 2, 1), (min(3, n - 1), min(bs // 2, n)), (0, min(n, bs)), (0, min(n, bs + 1))]
        r += [(max(bs - 3, 0), 6), (max(bs - 3, 0), 2 * bs + 6), (bs, bs), (2 * bs + 1, 3 * bs)]
        r += [(int(o), int(k)) for o, k in zip(rng.integers(0, n, 40), rng.integers(0, 3 * bs, 40))]
    r += r[:6]                    # duplicates
    return [r[i] for i in rng.permutation(len(r))]


def check_stream(kz, gpu, torch, oracle, s, x, hl, reqs_of):
    """index, info, blob and reads of stream s (decoding to x) against the model, on both variants and through a loaded index"""
    m = io_.build(oracle, s, hl_model(hl) if hl else None)
    ix = gpu.index(s, headerless=hl)
    d_src = to_dev(torch, s)
    ix_dev = gpu.index_device(d_src, len(s), headerless=hl)
    assert ix.info == io_.info(m) and ix_dev.info == io_.info(m)
    assert ix.save() == io_.blob(m) == ix_dev.save()
    assert ix.size == (0 if len(x) == 0 else -1)
    first = True
    for reqs in reqs_of:
        want = io_.read(oracle, s, dict(m), reqs)
        for w, (o, n) in zip(want, reqs):
            assert w == ("ok", x[o: o + n].tobytes()), (o, n)
        for device in (False, True):
            ixx = kz.StreamIndex.load(ix.save(), gpu) if first else ix
            rc, got = abi_read(gpu, torch, ixx, s, reqs, device)
            assert rc == 0 and got == want, [(r, g[0], len(g[1])) for r, g, w in zip(reqs, got, want) if g != w][:5]
            touches_last = any(o < len(x) and n and o + n > (len(x) - 1) // m["block_size"] * m["block_size"] for o, n in reqs)
            if first and touches_last:
                assert ixx.size == len(x)
            if touches_last:
                ix = ixx
        first = False
    if len(x):
        assert ix.read(s, len(x) - 1, 5) == x[-1:].tobytes()
        assert ix.size == len(x)
        assert ix.save() == io_.blob(dict(m, size=len(x)))
        outs, st = ix.read_many(s, [(0, 3), (len(x), 4), (1, 0)])
        assert outs == [x[:3].tobytes(), b"", b""] and st == [0, 0, 0]


@pytest.mark.parametrize("headerless", [False, True], ids=["headered", "headerless"])
@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_reads_match_the_model_1k_blocks(kz, gpu, oracle, synth, torch, chain, headerless):
    bs = 1024
    rng = np.random.default_rng(11)
    hl = hl_args(kz, chain, bs) if headerless else None
    for n in (0, 1, 15, 16, bs, bs + 1, 12 * bs - 300):
        x, s = make(oracle, synth, chain, n, bs, headerless)
        check_stream(kz, gpu, torch, oracle, s, x, hl, [request_list(n, bs, rng), [(n // 3, 5)]])


@pytest.mark.parametrize("chain,bs,n", [(CHAINS[3], 65536, 5 * 65536 + 1), (CHAINS[0], 65536, 65536), (CHAINS[6], 65536, 9 * 65536 - 9),
                                        (CHAINS[1], 4 << 20, (4 << 20) + 1), (CHAINS[3], 4 << 20, 3 * (4 << 20) - 5), (CHAINS[5], 4 << 20, 1)],
                         ids=lambda v: str(v) if isinstance(v, int) else "%s-%s-x%d" % v)
def test_reads_match_the_model_large_blocks(kz, gpu, oracle, synth, torch, chain, bs, n):
    rng = np.random.default_rng(12)
    for headerless in (False, True):
        x, s = make(oracle, synth, chain, n, bs, headerless, seed=8)
        check_stream(kz, gpu, torch, oracle, s, x, hl_args(kz, chain, bs) if headerless else None, [request_list(n, bs, rng)])


def test_ten_thousand_random_requests_in_one_call(kz, gpu, oracle, synth, torch):
    bs, n = 65536, 40 * 65536 - 1234
    x, s = make(oracle, synth, CHAINS[3], n, bs, False, seed=2)
    rng = np.random.default_rng(13)
    reqs = [(int(o), int(k)) for o, k in zip(rng.integers(0, n + bs, 10000), rng.integers(0, 8192, 10000))]
    ix = gpu.index(s)
    for device in (False, True):
        rc, got = abi_read(gpu, torch, ix, s, reqs, device)
        assert rc == 0
        for (o, k), g in zip(reqs, got):
            assert g == ("ok", x[o: o + k].tobytes())
    # the index built from the GPU's stream equals the one built from the oracle's
    assert gpu.index(gpu.compress(x, *CHAINS[3][:2], block_size=bs, input_size=n)).save() == io_.blob(io_.build(oracle, s))


def test_stale_index_is_refused_before_any_decode(kz, gpu, oracle, synth, torch):
    bs = 1024
    x, s = make(oracle, synth, CHAINS[4], 6 * bs, bs, False)
    ix = gpu.index(s)
    other = np.array(s)
    other[3] ^= 0xFF  # within the first 32 bytes: another stream of the same length
    gpu.profile(True)
    try:
        gpu.profile_reset()
        for device in (False, True):
            for bad in (other, s[:-1]):
                rc, got = abi_read(gpu, torch, ix, bad, [(0, 10), (3 * bs, 10)], device)
                assert rc == -18 and got == [("err", 18)] * 2
        assert gpu.kernel_time("block_header")[0] == 0 and gpu.stage_bytes("read:blocks")[0] == 0
    finally:
        gpu.profile(False)
        gpu.profile_reset()
    assert abi_read(gpu, torch, ix, s, [(0, 10)], False) == (0, [("ok", x[:10].tobytes())])
    # bad arguments are call-level too
    st = np.zeros(1, np.int32)
    assert gpu.lib.kz_read_ranges(gpu.h, ix.h, s.ctypes.data, len(s), 1, None, None, None, None, None, st.ctypes.data) == -18 and st[0] == -18
    assert gpu.lib.kz_index_load(None, 0, C.byref(C.c_void_p())) == -15
    with pytest.raises(kz.KanziError):
        kz.StreamIndex.load(ix.save()[:-3])
    hdr, bits = gpu.stream_header(kz.transform_type("SRT"), kz.entropy_type("ANS0"), bs)  # a chain the GPU path lacks, then the end marker
    with pytest.raises(kz.KanziError) as e:
        gpu.index(np.concatenate([hdr[: bits // 8], np.zeros(1, np.uint8)]))
    assert e.value.code == 14
    # walk and header errors are the codes kz_decompress_stream gives for the same bytes
    for cut in (len(s) - 1, len(s) // 2, 10):
        want = ro.outcome(gpu.decompress, s[:cut], len(x) + 64)
        with pytest.raises(kz.KanziError) as e:
            gpu.index(s[:cut])
        assert ("err", e.value.code) == want
    assert ro.outcome(gpu.decompress, s[:-1], len(x) + 64) == ("err", 13)


@pytest.mark.parametrize("chain", [CHAINS[3], CHAINS[5], CHAINS[1]], ids=[IDS[3], IDS[5], IDS[1]])
def test_damage_fails_only_the_requests_on_that_block(kz, gpu, oracle, synth, torch, chain):
    bs, nb = 1024, 12
    x, s = make(oracle, synth, chain, nb * bs - 300, bs, False, seed=9)
    recs = ro.walk(s, ro.header_bits(s))
    rng = np.random.default_rng(14)
    for kind in ["header", "payload"] + (["checksum"] if chain[2] else []):
        for victim in (0, 5, nb - 1):
            bad = ro.corrupt(s, recs[victim], kind)
            m = io_.build(oracle, bad)
            ix = gpu.index(bad)
            reqs = request_list(len(x), bs, rng) + [(victim * bs + 5, 10), (victim * bs - 5 if victim else 0, 10)]
            want = io_.read(oracle, bad, m, reqs)
            failing = [w for w in want if w[0] == "err"]
            if kind != "payload":
                assert failing and any(w[0] == "ok" and w[1] for w in want)
            else:  # a payload defect may decode to other bytes without an error: then the GPU must agree with itself
                want = None
            outs = [abi_read(gpu, torch, ix, bad, reqs, device)[1] for device in (False, True)]
            assert outs[0] == outs[1]
            if want is not None:
                assert outs[0] == want, (kind, victim)
            for (o, n), g in zip(reqs, outs[0]):
                lo, hi = o // bs, (min(o + n, len(x)) - 1) // bs
                if n and o < len(x) and not lo <= victim <= hi:
                    assert g == ("ok", x[o: o + n].tobytes()), (kind, victim, o, n)


def test_a_short_middle_block_makes_later_offsets_unseekable(kz, gpu, oracle, synth, torch):
    bs = 1024
    chain = ("LZ", "HUFFMAN", 32)
    x = np.ascontiguousarray(synth.markov_text(6 * bs, seed=4), np.uint8)
    # records of blocks 0..2, a block of bs - 16 bytes, then blocks 4..5: a stream no kanzi writer produces
    pieces = [x[0: bs], x[bs: 2 * bs], x[2 * bs: 3 * bs], x[3 * bs: 4 * bs - 16], x[4 * bs: 5 * bs], x[5 * bs:]]
    body = ho.records(oracle, np.concatenate(pieces[:3]), *chain[:2], bs, chain[2])
    parts = [np.unpackbits(body)[: ho.end_bit(body, 0) - 8]]
    for p in pieces[3:]:
        r = ho.records(oracle, p, *chain[:2], bs, chain[2])
        parts.append(np.unpackbits(r)[: ho.end_bit(r, 0) - 8])
    s = np.packbits(np.concatenate(parts + [np.zeros(8, np.uint8)]))
    hl = hl_args(kz, chain, bs)
    assert len(ro.walk(s, 0)) == 6
    ix = gpu.index(s, headerless=hl)
    reqs = [(0, 10), (2 * bs + 5, 100), (3 * bs - 5, 10), (3 * bs, 1), (4 * bs, 10), (5 * bs + 1, 5), (bs, bs), (2 * bs, 3 * bs)]
    want = io_.read(oracle, s, io_.build(oracle, s, hl_model(hl)), reqs)
    assert [w[0] for w in want] == ["ok", "ok", "err", "err", "err", "err", "ok", "err"]
    assert all(w == ("err", 15) for w in want if w[0] == "err")
    for device in (False, True):
        rc, got = abi_read(gpu, torch, ix, s, reqs, device)
        assert got == want and rc == -15
    assert ix.size == -1


def test_a_call_decodes_only_the_blocks_it_touches(kz, gpu, oracle, synth, torch):
    bs, nb = 64 << 10, 48
    tr, en = "TEXT+UTF+BWT+RANK+ZRLT", "ANS0"
    x = np.ascontiguousarray(synth.silesia_shaped(nb * bs - 500, seed=17), np.uint8)
    s = gpu.compress(x, tr, en, block_size=bs, input_size=len(x))
    recs = ro.walk(s, ro.header_bits(s))
    assert len(recs) == nb
    ix = gpu.index(s)
    stages = ["stage:inv:%d" % t for t in (kz.T_BWT, kz.T_RANK, kz.T_ZRLT)]
    gpu.profile(True)
    try:
        gpu.profile_reset()
        got = [gpu.decompress(s, len(x) + 64, k + 1, k + 2) for k in (3, 40)]
        alone = {st: gpu.stage_bytes(st)[1:] for st in stages}
        assert gpu.kernel_time("stream_walk")[0] == 2
        gpu.profile_reset()
        outs, st = ix.read_many(s, [(40 * bs + 9, 4096), (3 * bs + 100, 10)])
        assert st == [0, 0] and outs == [got[1][9: 9 + 4096].tobytes(), got[0][100: 110].tobytes()]
        assert gpu.stage_bytes("read:blocks") == (1, 2, 2 * bs)
        assert {st: gpu.stage_bytes(st)[1:] for st in stages} == alone
        assert gpu.kernel_time("stream_walk")[0] == 0
        assert gpu.stage_bytes("read:out") == (1, 2, 4106)
        windows, up = gpu.stage_bytes("read:h2d")[1:]
        assert windows == 2 and up <= sum((recs[k][1] + 7) // 8 + 1 + 16 + 64 + 16 for k in (3, 40))
        # 1,000 requests inside one block decode it once
        gpu.profile_reset()
        rng = np.random.default_rng(15)
        reqs = [(7 * bs + int(o), 64) for o in rng.integers(0, bs - 64, 1000)]
        outs, st = ix.read_many(s, reqs)
        assert not any(st) and all(o == x[a: a + 64].tobytes() for o, (a, _) in zip(outs, reqs))
        assert gpu.stage_bytes("read:blocks") == (1, 1, bs) and gpu.stage_bytes("read:out") == (1, 1000, 64000)
        # the device variant: no upload at all
        gpu.profile_reset()
        d_src, d_dst = to_dev(torch, s), torch.zeros(8192, dtype=torch.uint8, device="cuda")
        out_len, st = ix.read_many_device(d_src, len(s), [40 * bs, 3 * bs], [4096, 4096], d_dst, [0, 4096])
        assert out_len.tolist() == [4096, 4096] and st.tolist() == [0, 0]
        assert d_dst.cpu().numpy().tobytes() == x[40 * bs: 40 * bs + 4096].tobytes() + x[3 * bs: 3 * bs + 4096].tobytes()
        assert gpu.stage_bytes("read:blocks") == (1, 2, 2 * bs) and gpu.stage_bytes("read:h2d")[0] == 0
    finally:
        gpu.profile(False)
        gpu.profile_reset()


def test_scratch_follows_a_pass_not_the_requests(kz, synth):
    bs, nb = 4 << 20, 120  # more blocks than one pass holds (1 GiB / three slots of a little over 4 MiB)
    ctx = kz.Context(0)
    try:
        x = np.ascontiguousarray(synth.silesia_shaped(nb * bs, seed=3), np.uint8)
        s = ctx.compress(x, "LZ", "HUFFMAN", block_size=bs)
        ix = ctx.index(s)
        rng = np.random.default_rng(16)
        reqs = [(int(o), 4096) for o in rng.integers(0, len(x) - 4096, 10000)]
        before = ctx.device_bytes()
        outs, st = ix.read_many(s, reqs)
        assert not any(st) and all(o == x[a: a + 4096].tobytes() for o, (a, _) in zip(outs[::97], reqs[::97]))
        grown = ctx.device_bytes() - before
        staging = 10000 * 4096
        assert grown <= (1 << 30) + (1 << 30) // 8 + 2 * staging + (64 << 20), grown
        # a request over every block is staged and delivered whole
        assert ix.read(s, bs - 1, (nb - 2) * bs + 2) == x[bs - 1: (nb - 1) * bs + 1].tobytes()
    finally:
        ctx.close()


def test_reads_are_refused_while_a_session_is_open(kz, gpu, oracle, synth, torch):
    bs = 1024
    x, s = make(oracle, synth, CHAINS[4], 5 * bs, bs, False)
    ix = gpu.index(s)
    r = gpu.stream_reader(batch_blocks=2)
    try:
        rc, got = abi_read(gpu, torch, ix, s, [(0, 10)], False)
        assert rc == -18 and got == [("err", 18)]
        with pytest.raises(kz.KanziError) as e:
            gpu.index(s)
        assert e.value.code == 18
    finally:
        r.close()
    assert abi_read(gpu, torch, ix, s, [(0, 10)], True) == (0, [("ok", x[:10].tobytes())])
