"""GPU tests of the block range (kz_set_block_range, kanzi d --from / --to) on every stream-level decode path: kz_decompress_stream, its
device variant, kz_decompress_streams and its device variant, and the reader session, each against the range decode of tests/range_oracle.py
byte for byte; defects inside and outside the range give the same status on every path; skipped blocks do no stage work; the record limit
of a small output buffer applies to the decoded blocks only; the block-level entry points ignore the range; a range session stays in a full
session's memory."""
import hashlib
import itertools

import numpy as np
import pytest

import range_oracle as ro

pytestmark = pytest.mark.gpu

BS = 1024
NBLK = 12
CHAINS = [("DNA+LZ", "HUFFMAN", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 0), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE", 0),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0), ("LZ", "HUFFMAN", 0), ("NONE", "NONE", 32), ("NONE", "NONE", 64)]
IDS = ["%s-%s-x%d" % c for c in CHAINS]
GRID = [-1, 0, 1, 2, NBLK - 1, NBLK, NBLK + 1]


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def stream_of(oracle, synth, chain, seed=5, n=NBLK * BS - 300, bs=BS):
    tr, en, ck = chain
    x = np.ascontiguousarray(synth.markov_text(max(n, 1), seed=seed)[:n], np.uint8)
    return x, oracle.compress(x, tr, en, block_size=bs, checksum_bits=ck, input_size=len(x))


def to_dev(torch, a, extra=64):
    d = torch.zeros(len(a) + extra, dtype=torch.uint8, device="cuda")
    if len(a):
        d[: len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    return d


def dev_decompress(gpu, torch, s, cap, frm, to):
    d_src, d_dst = to_dev(torch, s), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    n = gpu.decompress_device(d_src.data_ptr(), len(s), d_dst.data_ptr(), cap, frm, to)
    return d_dst[:n].cpu().numpy()


def dev_streams(gpu, torch, streams, caps, frm, to):
    """kz_decompress_streams_device -> [("ok", bytes) or ("err", code)]"""
    s_off, o = [], 0
    for s in streams:
        s_off.append(o)
        o += (len(s) + 15) // 16 * 16 + 64
    d_src = torch.zeros(o + 64, dtype=torch.uint8, device="cuda")
    for s, so in zip(streams, s_off):
        if len(s):
            d_src[so: so + len(s)] = torch.from_numpy(np.ascontiguousarray(s, np.uint8)).cuda()
    d_off, o = [], 0
    for c in caps:
        d_off.append(o)
        o += (c + 15) // 16 * 16 + 32
    d_dst = torch.zeros(o + 64, dtype=torch.uint8, device="cuda")
    out_len, st = gpu.decompress_streams_device(d_src, s_off, [len(s) for s in streams], d_dst, d_off, caps, frm, to)
    h = d_dst.cpu().numpy()
    return [("ok", h[do: do + int(n)].tobytes()) if c == 0 else ("err", -int(c)) for do, n, c in zip(d_off, out_len, st)]


def host_streams(gpu, streams, caps, frm, to):
    outs, st = gpu.decompress_streams(streams, caps, frm, to)
    return [("ok", o.tobytes()) if c == 0 else ("err", -int(c)) for o, c in zip(outs, st)]


def read(gpu, s, bb, sizes, frm, to):
    with gpu.stream_reader(batch_blocks=bb, from_block=frm, to_block=to) as r:
        parts, pos = [], 0
        for p in sizes:
            parts.append(r.write(s[pos: pos + p]))
            pos += p
        parts.append(r.finish())
    return np.concatenate(parts)


def sizes_of(n, mode):
    if mode == "1mib":
        return [min(1 << 20, n - o) for o in range(0, n, 1 << 20)] or [0]
    out, odd = [], itertools.cycle([1, 13, 777, 4099, 3])
    while sum(out) < n:
        out.append(min(next(odd), n - sum(out)))
    return out or [0]


def every_path(gpu, torch, s, cap, frm, to, readers=((1, "1mib"), (4, "odd"), (1, "odd"), (4, "1mib"))):
    """(path name, outcome) of the range decode of s on every stream-level path"""
    s = np.ascontiguousarray(s, np.uint8)
    res = [("stream", ro.outcome(gpu.decompress, s, cap, frm, to)), ("device", ro.outcome(dev_decompress, gpu, torch, s, cap, frm, to)),
           ("streams", host_streams(gpu, [s], [cap], frm, to)[0]), ("streams_device", dev_streams(gpu, torch, [s], [cap], frm, to)[0])]
    for bb, mode in readers:
        res.append(("reader-%d-%s" % (bb, mode), ro.outcome(read, gpu, s, bb, sizes_of(len(s), mode), frm, to)))
    return res


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_every_path_matches_the_oracle_range(gpu, oracle, synth, torch, chain):
    x, s = stream_of(oracle, synth, chain)
    cap = len(x) + 64
    for i, (frm, to) in enumerate(itertools.product(GRID, GRID)):
        want = ro.outcome(ro.decompress_range, oracle, s, frm, to)
        assert want[0] == "ok"
        readers = [((1, "1mib"), (4, "odd"), (1, "odd"), (4, "1mib"))[i % 4]] if i % 5 else ((1, "1mib"), (4, "odd"), (1, "odd"), (4, "1mib"))
        for path, got in every_path(gpu, torch, s, cap, frm, to, readers):
            assert got == want, (path, frm, to, got[0], len(got[1]) if got[0] == "ok" else got[1], len(want[1]))


def test_many_streams_with_mixed_headers_and_an_empty_range(gpu, oracle, synth, torch):
    streams = []
    for i, chain in enumerate(CHAINS):
        n = (NBLK * BS - 300, 2 * BS - 7, 9 * BS, 0)[i % 4]
        streams.append(stream_of(oracle, synth, chain, seed=40 + i, n=n)[1])
    streams.append(stream_of(oracle, synth, ("LZ", "HUFFMAN", 64), seed=3, n=50 * BS, bs=4 * BS)[1])
    caps = [NBLK * BS + 64] * len(streams)
    caps[-1] = 50 * BS + 64
    for frm, to in [(3, 6), (-1, 2), (NBLK, -1), (5, 5), (2, 14), (-1, -1)]:
        want = [ro.outcome(ro.decompress_range, oracle, s, frm, to) for s in streams]
        assert any(w == ("ok", b"") for w in want), "no stream with an empty range"
        assert host_streams(gpu, streams, caps, frm, to) == want, (frm, to)
        assert dev_streams(gpu, torch, streams, caps, frm, to) == want, (frm, to)


@pytest.mark.parametrize("chain", [CHAINS[3], CHAINS[5], CHAINS[1]], ids=[IDS[3], IDS[5], IDS[1]])
def test_defects_give_one_status_on_every_path(gpu, oracle, synth, torch, chain):
    x, s = stream_of(oracle, synth, chain, seed=9)
    cap = len(x) + 64
    recs = ro.walk(s, ro.header_bits(s))
    kinds = ["header", "payload"] + (["checksum"] if chain[2] else [])
    readers = ((1, "1mib"), (4, "odd"))
    for kind, victim in itertools.product(kinds, (0, 5, NBLK - 1)):
        bad = ro.corrupt(s, recs[victim], kind)
        full = ro.outcome(gpu.decompress, bad, cap)
        if kind != "payload":
            assert full == ro.outcome(oracle.decompress, bad, cap), (kind, victim)
            assert full[0] == "err"
        vid = victim + 1
        for frm, to in ((vid + 1, -1), (-1, vid), (vid + 1, vid + 3), (vid, vid + 1), (vid - 1, vid + 2), (-1, -1)):
            if frm > NBLK or to == 0:
                continue
            got_all = every_path(gpu, torch, bad, cap, frm, to, readers)
            if not ro.in_range(vid, frm, to):
                want = ro.outcome(ro.decompress_range, oracle, bad, frm, to)
                assert want[0] == "ok"
            elif full[0] == "err":
                want = full
            else:  # a payload defect that decodes to other bytes without an error: every path gives the same bytes
                want = got_all[0][1]
            for path, got in got_all:
                assert got == want, (kind, victim, frm, to, path, got[0], got[1] if got[0] == "err" else len(got[1]), want[0])
    # a walk error behind the range: truncation inside the last record, and inside record 7
    for cut in (len(s) - 1, (recs[-1][0] + recs[-1][1] // 2) // 8, (recs[6][0] + 3) // 8):
        t = s[:cut]
        full = ro.outcome(gpu.decompress, t, cap)
        assert full[0] == "err" and full == ro.outcome(oracle.decompress, t, cap), cut
        for frm, to in ((1, 2), (2, 4), (NBLK + 1, -1)):
            for path, got in every_path(gpu, torch, t, cap, frm, to, readers):
                assert got == full, (cut, frm, to, path, got)


def test_skipped_blocks_do_no_stage_work(kz, gpu, oracle, synth):
    bs = 16 << 10
    tr, en = "TEXT+UTF+BWT+RANK+ZRLT", "ANS0"
    x = np.ascontiguousarray(synth.silesia_shaped(NBLK * bs - 500, seed=17), np.uint8)
    s = oracle.compress(x, tr, en, block_size=bs, input_size=len(x))
    recs = ro.walk(s, ro.header_bits(s))
    assert len(recs) == NBLK
    stages = ["stage:inv:%d" % t for t in (kz.T_TEXT, kz.T_UTF, kz.T_BWT, kz.T_RANK, kz.T_ZRLT)]
    gpu.profile(True)
    try:
        gpu.profile_reset()
        gpu.decompress(s, len(x) + 64)
        full = {st: gpu.stage_bytes(st)[1:] for st in stages}
        for victim in (0, 6, NBLK - 1):
            gpu.profile_reset()
            got = gpu.decompress(s, len(x) + 64, victim + 1, victim + 2)
            assert np.array_equal(got, x[victim * bs: (victim + 1) * bs])
            ranged = {st: gpu.stage_bytes(st)[1:] for st in stages}
            # that one block decoded on its own through the block-level entry point
            gpu.profile_reset()
            p, n = recs[victim]
            alone = gpu.decode_blocks(kz.transform_type(tr), kz.entropy_type(en), [(ro.payload(s, p, n), n)], bs)
            assert np.array_equal(alone[0], got)
            one = {st: gpu.stage_bytes(st)[1:] for st in stages}
            assert ranged == one, (victim, ranged, one)
            # RANK and BWT ran on this block only (the entropy stage's output is the ZRLT inverse's input)
            for st in ("stage:inv:%d" % kz.T_RANK, "stage:inv:%d" % kz.T_BWT, "stage:inv:%d" % kz.T_ZRLT):
                assert 0 < ranged[st][0] < full[st][0], (st, ranged[st], full[st])
    finally:
        gpu.profile(False)
        gpu.profile_reset()


def test_walk_limit_with_a_small_output_buffer(kz, gpu, oracle, torch):
    x = np.random.default_rng(1).integers(0, 256, 5000 * 1024, dtype=np.uint8)
    s = oracle.compress(x, "NONE", "NONE", block_size=1024, input_size=len(x))
    want = x[4989 * 1024: 4991 * 1024].tobytes()
    assert ro.decompress_range(oracle, s, 4990, 4992).tobytes() == want
    cap = 2048
    for path, got in every_path(gpu, torch, s, cap, 4990, 4992, readers=((4, "1mib"),)):
        assert got == ("ok", want), (path, got[0], got[1] if got[0] == "err" else len(got[1]))
    # without a range the record limit of such a buffer (cap / 1024 + 16 records) still applies, as before
    assert ro.outcome(gpu.decompress, s, cap)[0] == "err"


def test_range_state_and_block_level_entry_points(kz, gpu, oracle, synth, torch):
    chain = ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 32)
    x, s = stream_of(oracle, synth, chain, seed=23)
    cap = len(x) + 64
    recs = ro.walk(s, ro.header_bits(s))
    t48, et = kz.transform_type(chain[0]), kz.entropy_type(chain[1])
    try:
        gpu.set_block_range(3, 5)
        assert np.array_equal(gpu.decompress(s, cap), x[2 * BS: 4 * BS])
        # a call's own range is restored afterwards
        assert np.array_equal(gpu.decompress(s, cap, 1, 2), x[:BS])
        assert np.array_equal(gpu.decompress(s, cap), x[2 * BS: 4 * BS])
        # the block-level entry points decode every block they are given
        blocks = gpu.decode_blocks(t48, et, [(ro.payload(s, p, n), n) for p, n in recs], BS, 32)
        assert np.array_equal(np.concatenate(blocks), x)
        d_src = to_dev(torch, s)
        idx = gpu.stream_index_device(d_src.data_ptr(), len(s), 64)
        assert idx["nblocks"] == NBLK
        d_dst = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        n = gpu.decompress_fragment_device(d_src.data_ptr(), len(s), idx["rec_bit"][0], NBLK, d_dst.data_ptr(), cap, t48, et, BS, 32)
        assert np.array_equal(d_dst[:n].cpu().numpy(), x)
        # a session captures the range when it opens
        r = gpu.stream_reader(batch_blocks=2)
        gpu.set_block_range(-1, -1)
        with r:
            got = np.concatenate([r.write(s), r.finish()])
        assert np.array_equal(got, x[2 * BS: 4 * BS])
    finally:
        gpu.set_block_range(-1, -1)
    assert np.array_equal(gpu.decompress(s, cap), x)
    with gpu.stream_reader(batch_blocks=2) as r:
        assert np.array_equal(np.concatenate([r.write(s), r.finish()]), x)
    assert kz.Reader(s, ctx=gpu, from_block=2, to_block=3).read_all(cap).tobytes() == x[BS: 2 * BS].tobytes()
    assert np.array_equal(kz.Reader(s, ctx=gpu).read_all(cap), x)


def test_range_session_memory_1gib(kz, synth):
    tr, en, bs, bb = "TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 4 << 20, 8
    base = np.ascontiguousarray(synth.silesia_shaped(64 << 20, seed=21), np.uint8)
    npieces = 16  # 1 GiB, generated piecewise
    piece = lambda i: np.roll(base, 7919 * i)  # noqa: E731
    ctx = kz.Context(0)
    with ctx.stream_writer(tr, en, bs, batch_blocks=bb) as w:
        stream = np.concatenate([w.write(piece(i)) for i in range(npieces)] + [w.finish()])
    ctx.close()

    def session(frm, to):
        c = kz.Context(0)
        h, peak = hashlib.sha256(), 0
        with c.stream_reader(batch_blocks=bb, from_block=frm, to_block=to) as r:
            for o in range(0, stream.size, 1 << 20):
                h.update(r.write(stream[o: o + (1 << 20)]))
                peak = max(peak, c.device_bytes())
            h.update(r.finish())
            peak = max(peak, c.device_bytes())
        c.close()
        return h.digest(), peak

    full_digest, full_peak = session(-1, -1)
    lo, hi = 100, 110  # blocks 100 .. 109 of 256 (4 MiB each)
    want = hashlib.sha256()
    for b in range(lo - 1, hi - 1):
        i, o = divmod(b * bs, base.size)
        want.update(piece(i)[o: o + bs])
    got, peak = session(lo, hi)
    assert got == want.digest()
    assert peak <= full_peak, (peak, full_peak)
    h = hashlib.sha256()
    for i in range(npieces):
        h.update(piece(i))
    assert full_digest == h.digest()


def test_device_variants_follow_the_callers_default_stream(kz, gpu, oracle, synth, torch):
    """the device variants run after what the caller queued on its default stream: the input reaches its device buffer, and the output
    buffer is cleared, only behind a kernel of some 50 ms, and every call still reads all of its input and keeps all of its output"""
    x, s = stream_of(oracle, synth, CHAINS[6])
    cap, ecap = len(x) + 64, int(gpu.lib.kz_max_stream_output(len(x), BS))
    src_s, src_x = to_dev(torch, s), to_dev(torch, x)
    d_src, d_x = torch.zeros_like(src_s), torch.zeros_like(src_x)
    d_dst = torch.full((max(cap, ecap) + 64,), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def behind_a_kernel(dst, src):
        dst.zero_()
        torch.cuda._sleep(100_000_000)
        dst.copy_(src)
        d_dst.fill_(0)

    behind_a_kernel(d_src, src_s)
    n = gpu.decompress_device(d_src.data_ptr(), len(s), d_dst.data_ptr(), cap)
    assert n == len(x) and np.array_equal(d_dst[:n].cpu().numpy(), x)
    behind_a_kernel(d_src, src_s)
    out_len, st = gpu.decompress_streams_device(d_src, [0], [len(s)], d_dst, [0], [cap])
    assert list(st) == [0] and int(out_len[0]) == len(x) and np.array_equal(d_dst[: len(x)].cpu().numpy(), x)
    behind_a_kernel(d_x, src_x)
    n = gpu.compress_device(d_x.data_ptr(), len(x), d_dst.data_ptr(), ecap, kz.transform_type("NONE"), kz.E_NONE, BS, 64, input_size=len(x))
    assert n == len(s) and np.array_equal(d_dst[:n].cpu().numpy(), s)
