"""GPU tests of headerless streams (kz_set_headerless_writer / kz_set_headerless_reader: kanzi's NewWriter(..., headerless) and
NewHeaderlessReader). Every stream-level encode path writes the oracle's headerless stream byte for byte (tests/headerless_oracle.py);
every stream-level decode path decodes it, with and without a block range; defects give one error code on the whole-stream and reader
paths; the setting is checked as validateHeaderless checks it, captured by sessions and restored by the Python keywords; turning it off
brings back the headered bytes; a headerless reader session holds the device memory of a headered one."""
import itertools

import numpy as np
import pytest

import headerless_oracle as hlo
import range_oracle as ro

pytestmark = pytest.mark.gpu

BS = 1024
LEVELS = [("NONE", "NONE"), ("LZX", "NONE"), ("DNA+LZ", "HUFFMAN"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")]
CHAINS = [(tr, en, 0) for tr, en in LEVELS] + [("BWTS+MTFT+ZRLT", "ANS0", 32), ("BWT+RANK+ZRLT", "ANS1", 64), ("LZ", "RANGE", 0), ("NONE", "NONE", 32),
                                               ("NONE", "NONE", 64)]
IDS = ["%s-%s-x%d" % c for c in CHAINS]
SIZES = [0, 1, BS - 1, 3 * BS, 7 * BS + 123]


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def data_of(synth, n, seed):
    return np.ascontiguousarray(synth.markov_text(max(n, 1), seed=seed)[:n], np.uint8)


def params(chain, hint=-1, bs=BS):
    tr, en, ck = chain
    return dict(transform=tr, entropy=en, block_size=bs, checksum_bits=ck, output_size=hint)


def to_dev(torch, a, extra=64):
    d = torch.zeros(len(a) + extra, dtype=torch.uint8, device="cuda")
    if len(a):
        d[: len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    return d


def packed_dev(torch, arrays, lens):
    """arrays at 16-byte aligned offsets with >= 64 zero bytes behind each, on the device -> (tensor, offsets); lens: room per entry"""
    offs, o = [], 0
    for n in lens:
        offs.append(o)
        o += (n + 15) // 16 * 16 + 64
    d = torch.zeros(o + 64, dtype=torch.uint8, device="cuda")
    for a, so in zip(arrays, offs):
        if len(a):
            d[so: so + len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    return d, offs


def pieces(n, mode):
    if mode == "byte":
        return [1] * n or [0]
    out, odd = [], itertools.cycle([1, 13, 777, 4099, 3])
    while sum(out) < n:
        out.append(min(next(odd), n - sum(out)))
    return out or [0]


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
def test_every_encode_path_writes_the_oracle_stream(kz, gpu, oracle, synth, torch, chain):
    tr, en, ck = chain
    t48, et = kz.transform_type(tr), kz.entropy_type(en)
    xs = [data_of(synth, n, seed=3 + i) for i, n in enumerate(SIZES)]
    for hint in (False, True):
        isz = [len(x) if hint else 0 for x in xs]
        want = [hlo.compress(oracle, x, tr, en, BS, ck, input_size=h).tobytes() for x, h in zip(xs, isz)]
        assert want[0] == b"\x00"  # an empty input: the end marker alone
        for x, h, w in zip(xs, isz, want):
            assert gpu.compress(x, tr, en, BS, ck, h, headerless=True).tobytes() == w
            cap = gpu.lib.kz_max_stream_output(len(x), BS)
            d_src, d_dst = to_dev(torch, x), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
            n = gpu.compress_device(d_src.data_ptr(), len(x), d_dst.data_ptr(), cap, t48, et, BS, ck, h, headerless=True)
            assert d_dst[:n].cpu().numpy().tobytes() == w
            for bb, mode in ((1, "odd"), (4, "odd"), (4, "byte")):
                if mode == "byte" and len(x) > 3 * BS:
                    continue
                got = session(gpu.stream_writer(tr, en, BS, ck, batch_blocks=bb, input_size=h, headerless=True), x, pieces(len(x), mode))
                assert got.tobytes() == w, (bb, mode, len(x))
        outs, st = gpu.compress_streams(xs, tr, en, BS, ck, input_sizes=isz, headerless=True)
        assert list(st) == [0] * len(xs)
        assert [o.tobytes() for o in outs] == want
        caps = [int(gpu.lib.kz_max_stream_output(len(x), BS)) for x in xs]
        d_src, s_off = packed_dev(torch, xs, [len(x) for x in xs])
        d_dst, d_off = packed_dev(torch, [], caps)
        out_len, st = gpu.compress_streams_device(d_src, s_off, [len(x) for x in xs], d_dst, d_off, caps, tr, en, BS, ck, input_sizes=isz,
                                                  headerless=True)
        assert list(st) == [0] * len(xs)
        h = d_dst.cpu().numpy()
        assert [h[o: o + int(n)].tobytes() for o, n in zip(d_off, out_len)] == want
        # the setting off again: the headered bytes
        assert [gpu.compress(x, tr, en, BS, ck, i).tobytes() for x, i in zip(xs, isz)] == \
            [oracle.compress(x, tr, en, BS, ck, input_size=i).tobytes() for x, i in zip(xs, isz)]


# ---- decode ---------------------------------------------------------------------------------------------------------------------------
def every_decode(gpu, torch, s, cap, p, frm, to, readers=((1, "odd"), (4, "byte"), (4, "odd"))):
    """(path, outcome) of the headerless decode of s (parameters p) with the block range [frm, to) on every stream-level path"""
    s = np.ascontiguousarray(s, np.uint8)
    res = [("stream", ro.outcome(gpu.decompress, s, cap, frm, to, headerless=p))]

    def dev():
        d_src, d_dst = to_dev(torch, s), torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        n = gpu.decompress_device(d_src.data_ptr(), len(s), d_dst.data_ptr(), cap, frm, to, headerless=p)
        return d_dst[:n].cpu().numpy()

    res.append(("device", ro.outcome(dev)))
    outs, st = gpu.decompress_streams([s], [cap], frm, to, headerless=p)
    res.append(("streams", ("ok", outs[0].tobytes()) if st[0] == 0 else ("err", -int(st[0]))))
    d_src, s_off = packed_dev(torch, [s], [len(s)])
    d_dst, d_off = packed_dev(torch, [], [cap])
    out_len, st = gpu.decompress_streams_device(d_src, s_off, [len(s)], d_dst, d_off, [cap], frm, to, headerless=p)
    res.append(("streams_device", ("ok", d_dst[: int(out_len[0])].cpu().numpy().tobytes()) if st[0] == 0 else ("err", -int(st[0]))))
    for bb, mode in readers:
        if mode == "byte" and len(s) > 6000:
            continue
        res.append(("reader-%d-%s" % (bb, mode), ro.outcome(lambda: session(gpu.stream_reader(bb, frm, to, headerless=p), s, pieces(len(s), mode)))))
    return res


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_every_decode_path_reads_the_oracle_stream(kz, gpu, oracle, synth, torch, chain):
    tr, en, ck = chain
    xs = [data_of(synth, n, seed=30 + i) for i, n in enumerate(SIZES)]
    hls = [hlo.compress(oracle, x, tr, en, BS, ck) for x in xs]
    p = params(chain, hint=len(xs[-1]))
    cap = len(xs[-1]) + 64
    for x, s in zip(xs, hls):
        for frm, to in ((-1, -1), (2, 5), (3, -1), (-1, 1), (7, 9)):
            want = ro.outcome(hlo.decompress, oracle, s, tr, en, BS, ck, frm, to)
            assert want[0] == "ok"
            if (frm, to) == (-1, -1):
                assert want[1] == x.tobytes()
            for path, got in every_decode(gpu, torch, s, cap, p, frm, to):
                assert got == want, (path, len(x), frm, to, got[0], got[1] if got[0] == "err" else len(got[1]))
        # the index: the setting's fields, records from bit 0
        d_src = to_dev(torch, s)
        idx = gpu.stream_index_device(d_src.data_ptr(), len(s), 64, headerless=p)
        recs = ro.walk(s, 0)
        assert idx["nblocks"] == len(recs)
        assert idx["rec_bit"] == [0] + [q + n for q, n in recs]
        assert (idx["transform48"], idx["entropy"], idx["block_size"], idx["checksum_bits"], idx["input_size"]) == \
            (kz.transform_type(tr), kz.entropy_type(en), BS, ck, len(xs[-1]))
    # many streams in one call, empty ones included, with and without a range
    for frm, to in ((-1, -1), (2, 4)):
        want = [ro.outcome(hlo.decompress, oracle, s, tr, en, BS, ck, frm, to) for s in hls]
        outs, st = gpu.decompress_streams(hls, [cap] * len(hls), frm, to, headerless=p)
        assert [("ok", o.tobytes()) if c == 0 else ("err", -int(c)) for o, c in zip(outs, st)] == want
        d_src, s_off = packed_dev(torch, hls, [len(s) for s in hls])
        d_dst, d_off = packed_dev(torch, [], [cap] * len(hls))
        out_len, st = gpu.decompress_streams_device(d_src, s_off, [len(s) for s in hls], d_dst, d_off, [cap] * len(hls), frm, to, headerless=p)
        h = d_dst.cpu().numpy()
        assert [("ok", h[o: o + int(n)].tobytes()) if c == 0 else ("err", -int(c)) for o, n, c in zip(d_off, out_len, st)] == want


@pytest.mark.parametrize("chain", [CHAINS[5], CHAINS[6], CHAINS[9], CHAINS[10], CHAINS[3]], ids=[IDS[5], IDS[6], IDS[9], IDS[10], IDS[3]])
def test_defects_give_one_code_on_the_whole_stream_and_reader_paths(gpu, oracle, synth, chain):
    tr, en, ck = chain
    x = data_of(synth, 12 * 4096 - 300, seed=9)
    s = hlo.compress(oracle, x, tr, en, 4096, ck)
    headered = oracle.compress(x, tr, en, 4096, ck)
    hb = ro.header_bits(headered)
    recs = ro.walk(s, 0)
    p = params(chain, bs=4096)
    cap = len(x) + 64
    bad = {"cut-last": s[:-1], "cut-mid": s[: (recs[6][0] + 3) // 8], "cut-prefix": s[: recs[2][0] // 8 - 1]}
    for i, k in itertools.product((0, 5), ("length-lsb", "length-msb")):
        q, n = recs[i]
        # the record's length field is bit_length(n) bits wide (lw = log2(n / 8) + 4) and ends where its payload starts: flip its lowest
        # bit, or its top bit (the length loses its highest power of two)
        bad["%s-%d" % (k, i)] = ro.flip(s, q - 1) if k == "length-lsb" else ro.flip(s, q - n.bit_length())
    for name, b in bad.items():
        whole = ro.outcome(gpu.decompress, b, cap, headerless=p)
        for bb, mode in ((1, "odd"), (4, "odd")):
            got = ro.outcome(lambda: session(gpu.stream_reader(bb, headerless=p), b, pieces(len(b), mode)))
            if whole[0] == "err":
                assert got == whole, (name, bb, mode, got, whole)
            elif ck:
                assert got[0] == "err" or got[1] == whole[1], (name, bb)
        if whole[0] == "ok" and ck:
            assert whole[1] == x.tobytes(), name  # never wrong bytes with checksums on
        # the same defect behind a header (160 bits: whole bytes) gives the same code
        assert hb == 160
        hb_bits = np.unpackbits(np.frombuffer(bytes(headered), np.uint8))[:hb]
        with_header = np.packbits(np.concatenate([hb_bits, np.unpackbits(np.frombuffer(bytes(b), np.uint8))]))
        if whole[0] == "err":
            assert ro.outcome(gpu.decompress, with_header, cap) == whole, name
    # a wrong block size in the setting
    for wrong in (1024, 2048):
        q = params(chain, bs=wrong)
        whole = ro.outcome(gpu.decompress, s, cap, headerless=q)
        for bb in (1, 4):
            got = ro.outcome(lambda: session(gpu.stream_reader(bb, headerless=q), s, pieces(len(s), "odd")))
            assert got == whole, (wrong, bb, got, whole)
        assert whole[0] == "err" or whole[1] == x.tobytes(), wrong


# ---- the setting ----------------------------------------------------------------------------------------------------------------------
T_BWT, T_SRT, T_TEXT = 1 << 42, 13 << 42, 10 << 42


@pytest.mark.parametrize("args,code", [
    ((T_BWT, 5, BS, 0, -1, 7), 18), ((T_BWT, 5, BS, 0, -1, 5), 16), ((T_BWT, 3, BS, 0, -1, 6), 18), ((T_BWT, 10, BS, 0, -1, 6), 18),
    ((4 << 42, 5, BS, 0, -1, 6), 18), ((20 << 42, 5, BS, 0, -1, 6), 18), ((1 << 48, 5, BS, 0, -1, 6), 18), ((T_BWT, 5, 1023, 0, -1, 6), 18),
    ((T_BWT, 5, (1 << 30) + 16, 0, -1, 6), 18), ((T_BWT, 5, BS, 16, -1, 6), 18),
    ((T_SRT, 5, BS, 0, -1, 6), 14), ((T_TEXT, 8, BS, 0, -1, 6), 14), ((T_BWT, 6, BS, 0, -1, 6), 14), ((5 << 42, 0, BS, 0, -1, 6), 14),
    ((T_BWT, 5, BS, 0, -1, 6), 0), ((T_BWT, 5, 1025, 64, 1 << 48, 6), 0), ((0, 0, 1 << 30, 32, -5, 6), 0),
])
def test_setting_is_checked_as_validate_headerless(kz, gpu, args, code):
    t48, et, bs, ck, osz, ver = args
    want_oracle = hlo.validate(t48, et, bs, ck, ver)
    assert want_oracle == (0 if code == 14 else code)  # CREATE_CODEC: a valid kanzi setting the GPU path lacks
    gpu.set_headerless_reader(T_BWT, 5, 4096, 32, 77, 6)
    try:
        if code:
            with pytest.raises(kz.KanziError) as e:
                gpu.set_headerless_reader(t48, et, bs, ck, osz, ver)
            assert e.value.code == code
            assert gpu._hl_reader == (T_BWT, 5, 4096, 32, 77, 6)
        else:
            gpu.set_headerless_reader(t48, et, bs, ck, osz, ver)
        assert gpu.lib.kz_set_headerless_reader(gpu.h, t48, et, bs, ck, osz, ver) == -code
    finally:
        gpu.clear_headerless_reader()


def test_setting_state_sessions_and_python_mirror(kz, gpu, oracle, synth):
    chain = ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 32)
    tr, en, ck = chain
    x = data_of(synth, 9 * BS + 5, seed=41)
    headered = oracle.compress(x, tr, en, BS, ck, input_size=len(x)).tobytes()
    hl = hlo.compress(oracle, x, tr, en, BS, ck, input_size=len(x)).tobytes()
    p = params(chain)
    assert gpu.compress(x, tr, en, BS, ck, len(x)).tobytes() == headered
    try:
        gpu.set_headerless_writer(True)
        assert gpu.compress(x, tr, en, BS, ck, len(x)).tobytes() == hl
        assert gpu.compress(x, tr, en, BS, ck, len(x), headerless=False).tobytes() == headered  # a call's own setting, then restored
        assert gpu.compress(x, tr, en, BS, ck, len(x)).tobytes() == hl
        w = gpu.stream_writer(tr, en, BS, ck, batch_blocks=2, input_size=len(x))  # a session keeps the setting it opened with
        gpu.set_headerless_writer(False)
        assert session(w, x, pieces(len(x), "odd")).tobytes() == hl
        assert gpu.compress(x, tr, en, BS, ck, len(x)).tobytes() == headered
        gpu.set_headerless_reader(**p)
        assert gpu.decompress(hl, len(x) + 64).tobytes() == x.tobytes()
        assert gpu.decompress(hl, len(x) + 64, 2, 3).tobytes() == x[BS: 2 * BS].tobytes()
        r = gpu.stream_reader(batch_blocks=2)
        gpu.clear_headerless_reader()
        assert session(r, hl, pieces(len(hl), "odd")).tobytes() == x.tobytes()
        assert gpu.decompress(headered, len(x) + 64).tobytes() == x.tobytes()
        # a headered stream read as headerless fails; it never decodes to wrong bytes (its checksums are on)
        got = ro.outcome(gpu.decompress, headered, len(x) + 64, headerless=p)
        assert got[0] == "err" or got[1] == x.tobytes()
        assert gpu._hl_reader is None and gpu._hl_writer is False
    finally:
        gpu.set_headerless_writer(False)
        gpu.clear_headerless_reader()
    # the io mirrors
    wr = kz.Writer(tr, en, BS, checksum=ck, file_size=len(x), ctx=gpu, headerless=True)
    wr.write(x[:100])
    wr.write(x[100:])
    assert wr.getvalue().tobytes() == hl
    rd = kz.HeaderlessReader(hl, 1, tr, en, BS, ck, len(x), 6, ctx=gpu)
    assert rd.read_all(len(x) + 64).tobytes() == x.tobytes()
    assert kz.HeaderlessReader(hl, 1, tr, en, BS, ck, ctx=gpu, from_block=9, to_block=11).read_all(len(x)).tobytes() == x[8 * BS:].tobytes()
    with pytest.raises(kz.KanziError) as e:
        kz.HeaderlessReader(hl, 1, tr, en, BS, 16, ctx=gpu)
    assert e.value.code == 18
    with pytest.raises(kz.KanziError) as e:
        kz.HeaderlessReader(hl, 1, "SRT", en, BS, ck, ctx=gpu)
    assert e.value.code == 14
    assert gpu._hl_reader is None


def test_reader_session_device_bytes_match_the_headered_session(kz, oracle, synth):
    tr, en, ck, bs = "TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 64, 64 << 10
    x = data_of(synth, 40 * bs + 999, seed=5)
    headered = oracle.compress(x, tr, en, bs, ck)
    hl = hlo.compress(oracle, x, tr, en, bs, ck)

    def run(s, p):
        c = kz.Context(0)
        try:
            with c.stream_reader(batch_blocks=4, headerless=p) as r:
                out = [r.write(s[o: o + 7777]) for o in range(0, len(s), 7777)] + [r.finish()]
                return np.concatenate(out).tobytes(), c.device_bytes()
        finally:
            c.close()

    a, bytes_a = run(headered, None)
    b, bytes_b = run(hl, dict(transform=tr, entropy=en, block_size=bs, checksum_bits=ck))
    assert a == b == x.tobytes()
    assert bytes_a == bytes_b
