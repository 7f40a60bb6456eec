"""GPU tests of kanzi's skipBlocks option (kz_set_skip_blocks, kanzi c --skip). Every encode path writes the stream of the skip model
(tests/skip_oracle.py, checked against the oracle by tests/test_oracle_skip_blocks.py) byte for byte, kz_encode_blocks the oracle's
records; every decode path reads those streams back, with and without a block range; the setting is off by default, captured by sessions
and restored by the Python keywords, and costs nothing when off; and a stored block never reaches a transform stage."""
import bz2
import gzip
import itertools
import lzma

import numpy as np
import pytest

import range_oracle as ro
import skip_oracle as so

pytestmark = pytest.mark.gpu

BS = 1 << 16
CHAINS = [("NONE", "NONE", 0), ("LZ", "HUFFMAN", 32), ("DNA+LZ", "HUFFMAN", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 64),
          ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE", 0), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 32), ("BWT", "ANS1", 64), ("BWT+RANK+ZRLT", "RANGE", 0)]
IDS = ["%s-%s-x%d" % c for c in CHAINS]
T_TEXT, T_UTF, T_BWT, T_RANK, T_ZRLT = 10, 17, 1, 8, 6


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def _text(synth, n, seed):
    return np.ascontiguousarray(synth.markov_text(n, seed=seed)[:n], np.uint8)


def _led(synth, head, seed):
    return np.concatenate([np.frombuffer(head, np.uint8), _text(synth, BS - len(head), seed)])


def corpus_blocks(synth, seed=0):
    """BS-byte blocks: text, uniform random, stdlib gzip / bz2 / xz members, compressible text led by a PNG signature (stored for its magic
    number alone) and by FFD8FFE1 (not stored), the blocks of entropy 972 (not stored) and 973 (stored), text"""
    rng = np.random.default_rng(seed)
    t = _text(synth, 8 * BS, seed + 1).tobytes() + rng.integers(0, 256, BS, dtype=np.uint8).tobytes()
    blocks = [_text(synth, BS, seed + 2), rng.integers(0, 256, BS, dtype=np.uint8)]
    for member in (gzip.compress(t, mtime=0), bz2.compress(t), lzma.compress(t, format=lzma.FORMAT_XZ)):
        blocks.append(np.frombuffer((member * (BS // len(member) + 1))[:BS], np.uint8))
    blocks += [_led(synth, b"\x89PNG\r\n\x1a\n", seed + 3), _led(synth, b"\xff\xd8\xff\xe1", seed + 4), so.entropy_block(972, BS, seed + 5),
               so.entropy_block(973, BS, seed + 6), _text(synth, BS, seed + 7)]
    return blocks


REASONS = [None, "entropy", "magic", "magic", "magic", "magic", None, None, "entropy", None]


def corpus(synth, tail, seed=0):
    """the blocks, then a final block of `tail` bytes (15: stored as every short block; 16: led by gzip's magic number, stored)"""
    last = np.frombuffer(b"\x1f\x8b" + bytes(range(3, 3 + tail - 2)), np.uint8)
    return np.concatenate(corpus_blocks(synth, seed) + [last])


@pytest.fixture(scope="module")
def x15(synth):
    return corpus(synth, 15)


@pytest.fixture(scope="module")
def x16(synth):
    return corpus(synth, 16, seed=1)


def test_corpus(synth, x15, x16):
    assert [so.reason(b) for b in corpus_blocks(synth)] == REASONS
    assert [so.reason(b) for b in corpus_blocks(synth, 1)] == REASONS
    assert so.reason(x15[-15:]) == "small" and so.reason(x16[-16:]) == "magic"


def to_dev(torch, a, extra=64):
    """a on the device, the copy finished: the library's calls run on their own non-blocking stream"""
    d = torch.zeros(len(a) + extra, dtype=torch.uint8, device="cuda")
    if len(a):
        d[: len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    torch.cuda.synchronize()
    return d


def pieces(n, mode):
    if mode == "mib":
        return [1 << 20] * (n >> 20) + [n & ((1 << 20) - 1)]
    out, odd = [], itertools.cycle([1, 13, 77777, 4099, 3, 150001])
    while sum(out) < n:
        out.append(min(next(odd), n - sum(out)))
    return out


def session(sess, s, sizes):
    with sess as r:
        parts, pos = [], 0
        for p in sizes:
            parts.append(r.write(s[pos: pos + p]))
            pos += p
        parts.append(r.finish())
    return np.concatenate(parts)


# ---- encode ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_stream_encodes_write_the_skip_stream(kz, gpu, oracle, torch, x15, x16, chain):
    tr, en, ck = chain
    t48, et = kz.transform_type(tr), kz.entropy_type(en)
    for x, hl in ((x15, False), (x16, True)):
        want = so.compress(oracle, x, tr, en, BS, ck, input_size=x.size, headerless=hl).tobytes()
        assert want != so.compress(oracle, x, tr, en, BS, ck, input_size=x.size, headerless=hl, skip=False).tobytes()
        assert gpu.compress(x, tr, en, BS, ck, x.size, headerless=hl, skip_blocks=True).tobytes() == want
        cap = gpu.lib.kz_max_stream_output(len(x), BS)
        d_src, d_dst = to_dev(torch, x), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        n = gpu.compress_device(d_src.data_ptr(), len(x), d_dst.data_ptr(), cap, t48, et, BS, ck, x.size, headerless=hl, skip_blocks=True)
        assert d_dst[:n].cpu().numpy().tobytes() == want
        for bb, mode in ((1, "mib"), (4, "odd")):
            got = session(gpu.stream_writer(tr, en, BS, ck, batch_blocks=bb, input_size=x.size, headerless=hl, skip_blocks=True), x, pieces(len(x), mode))
            assert got.tobytes() == want, (bb, mode)
        w = kz.Writer(tr, en, BS, checksum=ck, file_size=x.size, ctx=gpu, headerless=hl, skip_blocks=True)
        w.write(x)
        assert w.getvalue().tobytes() == want


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_many_stream_encodes(kz, gpu, oracle, torch, x15, chain):
    """files at unaligned offsets of one buffer, some shorter than 16 bytes, and the device variant"""
    tr, en, ck = chain
    cuts = [0, 7, 7 + 15, 7 + 15 + 16, 3 * BS + 5, 3 * BS + 1000, 6 * BS + 3, x15.size]
    xs = [x15[a:b] for a, b in zip(cuts, cuts[1:])] + [x15[:0]]
    want = [so.compress(oracle, x, tr, en, BS, ck, input_size=x.size).tobytes() for x in xs]
    outs, st = gpu.compress_streams(xs, tr, en, BS, ck, input_sizes=[x.size for x in xs], skip_blocks=True)
    assert list(st) == [0] * len(xs)
    assert [o.tobytes() for o in outs] == want
    lens = [x.size for x in xs]
    s_off = list(itertools.accumulate([0] + [(n + 15) // 16 * 16 + 64 for n in lens]))[:-1]
    d_src = torch.zeros(s_off[-1] + lens[-1] + 128, dtype=torch.uint8, device="cuda")
    for x, o in zip(xs, s_off):
        if x.size:
            d_src[o: o + x.size] = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    torch.cuda.synchronize()
    caps = [int(gpu.lib.kz_max_stream_output(n, BS)) for n in lens]
    d_off = list(itertools.accumulate([0] + [(c + 15) // 16 * 16 for c in caps]))[:-1]
    d_dst = torch.zeros(d_off[-1] + caps[-1] + 64, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    out_len, st = gpu.compress_streams_device(d_src, s_off, lens, d_dst, d_off, caps, tr, en, BS, ck, input_sizes=lens, skip_blocks=True)
    assert list(st) == [0] * len(xs)
    h = d_dst.cpu().numpy()
    assert [h[o: o + int(n)].tobytes() for o, n in zip(d_off, out_len)] == want


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_fragments_and_encode_blocks(kz, gpu, oracle, torch, x16, chain):
    tr, en, ck = chain
    t48, et = kz.transform_type(tr), kz.entropy_type(en)
    # a header plus the records of two fragments plus the end marker: the single stream
    want = so.compress(oracle, x16, tr, en, BS, ck, input_size=x16.size)
    hdr, hbits = gpu.stream_header(t48, et, BS, ck, x16.size)
    cut = 4 * BS
    frags, fbits = [], []
    for part in (x16[:cut], x16[cut:]):
        cap = gpu.lib.kz_max_stream_output(part.size, BS)
        d_src, d_dst = to_dev(torch, part), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        fbits.append(gpu.compress_fragment_device(d_src.data_ptr(), part.size, d_dst.data_ptr(), cap, t48, et, BS, ck, skip_blocks=True))
        frags.append(d_dst)
    d_hdr, d_end = to_dev(torch, hdr), torch.zeros(64, dtype=torch.uint8, device="cuda")
    cap = want.size + 64
    d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    total = gpu.concat_bits_device([d_hdr.data_ptr()] + [f.data_ptr() for f in frags] + [d_end.data_ptr()], [hbits] + fbits + [8], d_out.data_ptr(), cap)
    assert (total + 7) // 8 == want.size
    assert np.array_equal(d_out[: want.size].cpu().numpy(), want)
    # kz_encode_blocks: the oracle's record of every block (TEXT sizes its hash map from the longest block, so the short tail goes alone)
    blocks = [x16[o: o + BS] for o in range(0, x16.size, BS)]
    for batch in (blocks[:-1], blocks[-1:]):
        got = gpu.encode_blocks(t48, et, batch, ck, skip_blocks=True)
        for b, (payload, bits) in zip(batch, got):
            wp, wb = oracle.encode_block(b, t48, et, ck, skip_blocks=True)
            assert bits == wb and np.array_equal(payload, wp)
            assert bool(payload[0] & 0x80) == so.stored(b)


def test_setting_off_and_its_state(kz, gpu, oracle, x15, x16):
    tr, en, ck = CHAINS[5]
    want_off = oracle.compress(x15, tr, en, BS, ck, input_size=x15.size).tobytes()
    want_on = so.compress(oracle, x15, tr, en, BS, ck, input_size=x15.size).tobytes()
    launches = []
    for toggled in (False, True):  # off by default, and off again after on: the same bytes and the same kernel launches
        c = kz.Context(0)
        if toggled:
            c.set_skip_blocks(True)
            c.set_skip_blocks(False)
        c.launch_count(reset=True)
        assert c.compress(x15, tr, en, BS, ck, x15.size).tobytes() == want_off
        launches.append(c.launch_count(reset=True))
        c.close()
    assert launches[0] == launches[1]
    assert gpu.compress(x15, tr, en, BS, ck, x15.size, skip_blocks=False).tobytes() == want_off
    # a per-call keyword restores the previous value, either way
    gpu.set_skip_blocks(True)
    try:
        assert gpu.compress(x15, tr, en, BS, ck, x15.size, skip_blocks=False).tobytes() == want_off
        assert gpu.compress(x15, tr, en, BS, ck, x15.size).tobytes() == want_on
        # a session keeps the value it opened with
        w = gpu.stream_writer(tr, en, BS, ck, batch_blocks=2, input_size=x15.size)
        gpu.set_skip_blocks(False)
        assert session(w, x15, pieces(x15.size, "odd")).tobytes() == want_on
    finally:
        gpu.set_skip_blocks(False)
    assert gpu.compress(x15, tr, en, BS, ck, x15.size, skip_blocks=True).tobytes() == want_on
    assert gpu.compress(x15, tr, en, BS, ck, x15.size).tobytes() == want_off
    # the stored blocks and bytes by reason, under "skip:magic" / "skip:entropy"
    gpu.profile(True)
    gpu.profile_reset()
    try:
        gpu.compress(x16, tr, en, BS, ck, x16.size, skip_blocks=True)
        blocks = [x16[o: o + BS] for o in range(0, x16.size, BS)]
        for r in ("magic", "entropy"):
            sel = [b for b in blocks if so.reason(b) == r]
            assert gpu.stage_bytes("skip:" + r)[1:] == (len(sel), sum(b.size for b in sel)), r
        assert gpu.kernel_time("skip_hist")[0] == 1 and gpu.kernel_time("skip_decide")[0] == 1
    finally:
        gpu.profile(False)
        gpu.profile_reset()


# ---- decode ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_every_decode_path_reads_skip_streams(kz, gpu, oracle, torch, x15, x16, chain):
    tr, en, ck = chain
    for x, hl in ((x15, False), (x16, True)):
        s = so.compress(oracle, x, tr, en, BS, ck, input_size=x.size, headerless=hl)
        p = dict(transform=tr, entropy=en, block_size=BS, checksum_bits=ck, output_size=x.size) if hl else None
        cap = x.size + 64
        blocks = [x[o: o + BS] for o in range(0, x.size, BS)]
        # (2, 3): the random block alone, stored; (3, 6): the three stdlib members, stored; (1, 2) and (6, 8): not stored
        for frm, to in ((-1, -1), (2, 3), (3, 6), (1, 2), (6, 8), (9, -1)):
            want = np.concatenate([b for i, b in enumerate(blocks) if ro.in_range(i + 1, frm, to)]).tobytes()
            assert bytes(gpu.decompress(s, cap, frm, to, headerless=p)) == want, (frm, to)
            d_src, d_dst = to_dev(torch, s), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
            n = gpu.decompress_device(d_src.data_ptr(), s.size, d_dst.data_ptr(), cap, frm, to, headerless=p)
            assert d_dst[:n].cpu().numpy().tobytes() == want
            outs, st = gpu.decompress_streams([s], [cap], frm, to, headerless=p)
            assert st[0] == 0 and outs[0].tobytes() == want
            for bb, mode in ((1, "odd"), (4, "mib")):
                assert session(gpu.stream_reader(bb, frm, to, headerless=p), s, pieces(s.size, mode)).tobytes() == want
        if not hl:
            assert np.array_equal(oracle.decompress(s, cap), x)


def test_stored_blocks_reach_no_stage(kz, gpu, oracle):
    """all-random 4 MiB blocks at -l 5: with the option on no TEXT / UTF / BWT / RANK / ZRLT work in either direction"""
    tr, en = "TEXT+UTF+BWT+RANK+ZRLT", "ANS0"
    x = np.random.default_rng(11).integers(0, 256, 3 * (4 << 20) + 12345, dtype=np.uint8)
    gpu.profile(True)
    gpu.profile_reset()
    try:
        s = gpu.compress(x, tr, en, 4 << 20, 32, x.size, skip_blocks=True)
        y = gpu.decompress(s, x.size + 64)
        for t in (T_TEXT, T_UTF, T_BWT, T_RANK, T_ZRLT):
            for d in ("fwd", "inv"):
                assert gpu.stage_bytes("stage:%s:%d" % (d, t))[1:] == (0, 0), (d, t)
        assert gpu.stage_bytes("skip:entropy")[1:] == (4, x.size)
        gpu.profile_reset()
        gpu.compress(x, tr, en, 4 << 20, 32, x.size)  # off: every stage runs
        assert gpu.stage_bytes("stage:fwd:%d" % T_BWT)[1] > 0
    finally:
        gpu.profile(False)
        gpu.profile_reset()
    assert np.array_equal(y, x)
    assert s.tobytes() == so.compress(oracle, x, tr, en, 4 << 20, 32, input_size=x.size).tobytes()
