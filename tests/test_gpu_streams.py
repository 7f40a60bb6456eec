"""GPU tests of the many-stream entry points (kz_compress_streams / kz_decompress_streams and their _device variants): every stream of a batch
equals the oracle's stream and the single-stream call's, one decode call takes streams of different headers, a corrupt stream gets the code
a single-stream call gives for its bytes while every other stream decodes exactly, and nothing outside a stream's destination range is
written."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BS = 64 << 10
LEVELS = {"l0": ("NONE", "NONE"), "l1": ("LZX", "NONE"), "l2": ("DNA+LZ", "HUFFMAN"), "l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"),
          "l4": ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")}
CHAINS = [(tr, en, 0) for tr, en in LEVELS.values()] + [
    ("BWTS+MTFT+ZRLT", "ANS0", 0), ("BWT+RANK+ZRLT", "ANS1", 0), ("LZ", "RANGE", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 32), ("NONE", "ANS0", 64)]


def inputs(synth, seed):
    """streams of sizes 0, 1, 15, 16, 17, block - 1, block, block + 1, 3.5 blocks and random, in three kinds of data"""
    rng = np.random.default_rng(seed)
    sizes = [0, 1, 15, 16, 17, BS - 1, BS, BS + 1, BS * 7 // 2, int(rng.integers(1, 4 * BS))]
    gens = [lambda n, s: synth.markov_text(n, seed=s), lambda n, s: synth.x86_like(n, seed=s), lambda n, s: synth.uniform_bytes(n, seed=s)]
    out = []
    for k, g in enumerate(gens):
        for i, n in enumerate(sizes):
            out.append(np.ascontiguousarray(g(n, seed + 31 * k + i)[:n], np.uint8) if n else np.zeros(0, np.uint8))
    return out


@pytest.mark.parametrize("chain", CHAINS, ids=["%s-%s-x%d" % c for c in CHAINS])
def test_chain_matches_oracle_and_single_calls(gpu, oracle, synth, chain):
    tr, en, ck = chain
    xs = inputs(synth, seed=len(tr) + ck)
    isz = [len(x) if i % 2 else 0 for i, x in enumerate(xs)]
    outs, st = gpu.compress_streams(xs, tr, en, BS, ck, isz)
    assert (st == 0).all(), st
    wants = []
    for i, x in enumerate(xs):
        want = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=isz[i])
        assert np.array_equal(outs[i], want), (chain, i, len(x))
        assert np.array_equal(outs[i], gpu.compress(x, tr, en, BS, ck, isz[i])), (chain, i, len(x))
        wants.append(want)
    ys, st = gpu.decompress_streams(wants, [len(x) + 64 for x in xs])
    assert (st == 0).all(), st
    for i, x in enumerate(xs):
        assert np.array_equal(ys[i], x), (chain, i, len(x))


def test_mixed_headers_in_one_decode_call(gpu, oracle, synth):
    rng = np.random.default_rng(5)
    streams, xs = [], []
    for i in range(36):
        tr, en = list(LEVELS.values())[i % 6]
        bs = [1024, BS, 1 << 20][(i // 6) % 3]
        ck = [0, 32, 64][(i // 18) % 2 + (i % 2)]
        x = synth.markov_text(int(rng.integers(0, 3 * bs)), seed=100 + i)
        xs.append(x)
        streams.append(oracle.compress(x, tr, en, block_size=bs, checksum_bits=ck, input_size=len(x)))
    ys, st = gpu.decompress_streams(streams, [len(x) + 16 for x in xs])
    assert (st == 0).all(), st
    for i, x in enumerate(xs):
        assert np.array_equal(ys[i], x), i


def single_code(gpu, kz, s, cap):
    try:
        gpu.decompress(s, cap)
    except kz.KanziError as e:
        return e.code
    return 0


def test_corrupt_streams_fail_alone(gpu, oracle, synth, kz):
    """bad magic, truncation, checksum mismatch and a too-small cap at known indexes, in groups shared with healthy streams"""
    rng = np.random.default_rng(9)
    kinds = [("NONE", "NONE", 32), ("NONE", "ANS0", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 0), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0)]
    xs, streams, caps = [], [], []
    for i in range(48):
        tr, en, ck = kinds[i % 4]
        x = synth.zipf_bytes(int(rng.integers(1000, 200000)), 1.0, seed=200 + i)
        xs.append(x)
        streams.append(oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=len(x)))
        caps.append(len(x) + 64)
    bad = {}
    s = streams[4].copy()  # NONE / NONE, 32-bit checksums
    s[0] ^= 0x01
    streams[4], bad[4] = s, "magic"
    s = streams[13]  # NONE / ANS0
    streams[13], bad[13] = s[: len(s) // 2].copy(), "truncated"
    s = streams[20].copy()  # NONE / NONE, 32-bit checksums
    s[len(s) // 2] ^= 0x10
    streams[20], bad[20] = s, "checksum"
    caps[27], bad[27] = len(xs[27]) - 1, "cap"  # l5
    caps[34], bad[34] = len(xs[34]) // 2, "cap"  # l3
    ys, st = gpu.decompress_streams(streams, caps)
    for i in range(len(xs)):
        if i in bad:
            code = single_code(gpu, kz, streams[i], caps[i])
            assert code != 0 and st[i] == -code, (i, bad[i], st[i], code)
            assert ys[i] is None
        else:
            assert st[i] == 0 and np.array_equal(ys[i], xs[i]), (i, st[i])
    assert -st[20] == 19 and -st[27] == 12 and -st[34] == 12


def test_too_small_compress_cap_fails_alone(gpu, synth, kz):
    lib = gpu.lib
    xs = [synth.markov_text(n, seed=n) for n in (5000, 70000, 300)]
    src = np.concatenate(xs)
    src_len = np.array([len(x) for x in xs], np.uint64)
    src_off = np.array([0, 5000, 75000], np.uint64)
    full = [gpu.compress(x, "TEXT+UTF+BWT+RANK+ZRLT", "ANS0", BS) for x in xs]
    cap = np.array([len(full[0]), len(full[1]) - 1, len(full[2]) + 100], np.uint64)
    dst_off = np.array([0, 8192, 8192 + 100000], np.uint64)
    dst = np.full(8192 + 100000 + 2000, 0xA5, np.uint8)
    out_len, st = np.zeros(3, np.uint64), np.zeros(3, np.int32)
    rc = lib.kz_compress_streams(gpu.h, kz.transform_type("TEXT+UTF+BWT+RANK+ZRLT"), kz.E_ANS0, BS, 0, 3, src.ctypes.data, src_off.ctypes.data,
                                 src_len.ctypes.data, None, dst.ctypes.data, dst_off.ctypes.data, cap.ctypes.data, out_len.ctypes.data, st.ctypes.data)
    assert rc == -12 and list(st) == [0, -12, 0]
    assert int(out_len[1]) == len(full[1])
    assert np.array_equal(dst[: len(full[0])], full[0]) and np.array_equal(dst[108192: 108192 + len(full[2])], full[2])
    assert (dst[len(full[0]): 8192] == 0xA5).all() and (dst[8192: 108192] == 0xA5).all() and (dst[108192 + len(full[2]):] == 0xA5).all()


def test_canary_host_and_device(gpu, oracle, synth, kz):
    """dst is pre-filled; bytes outside every [dst_off, dst_off + dst_cap) stay as they were, in both directions and both variants"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    xs = [synth.markov_text(int(n), seed=int(n)) for n in rng.integers(0, 150000, 24)]
    tr, en = LEVELS["l3"]
    wants = [oracle.compress(x, tr, en, block_size=BS) for x in xs]
    # host, decompress: gaps of 48 bytes between the ranges
    caps = np.array([len(x) + 32 for x in xs], np.uint64)
    dst_off = np.zeros(len(xs), np.uint64)
    o = 48
    for i, c in enumerate(caps):
        dst_off[i] = o
        o += int(c) + 48
    dst = np.full(o, 0x5A, np.uint8)
    src = np.concatenate(wants)
    src_len = np.array([len(w) for w in wants], np.uint64)
    src_off = np.zeros(len(xs), np.uint64)
    src_off[1:] = np.cumsum(src_len)[:-1]
    out_len, st = np.zeros(len(xs), np.uint64), np.zeros(len(xs), np.int32)
    assert gpu.lib.kz_decompress_streams(gpu.h, len(xs), src.ctypes.data, src_off.ctypes.data, src_len.ctypes.data, dst.ctypes.data, dst_off.ctypes.data,
                                         caps.ctypes.data, out_len.ctypes.data, st.ctypes.data) == 0
    inside = np.zeros(o, bool)
    for i, x in enumerate(xs):
        a = int(dst_off[i])
        assert int(out_len[i]) == len(x) and np.array_equal(dst[a: a + len(x)], x), i
        inside[a: a + int(caps[i])] = True
    assert (dst[~inside] == 0x5A).all()
    # device, both directions: offsets multiples of 16, gaps of 32 bytes
    dev = torch.device("cuda:0")
    d_src = torch.zeros(int(sum((len(x) + 15) // 16 * 16 for x in xs)) + 64, dtype=torch.uint8, device=dev)
    s_off, o = [], 0
    for x in xs:
        s_off.append(o)
        d_src[o: o + len(x)] = torch.from_numpy(x).to(dev)
        o += (len(x) + 15) // 16 * 16
    ccap = [int(gpu.lib.kz_max_stream_output(len(x), BS)) for x in xs]
    c_off, o = [], 32
    for c in ccap:
        c_off.append(o)
        o += (c + 15) // 16 * 16 + 32
    d_cmp = torch.full((o,), 0x5A, dtype=torch.uint8, device=dev)
    clen, st = gpu.compress_streams_device(d_src, s_off, [len(x) for x in xs], d_cmp, c_off, ccap, tr, en, BS)
    assert (st == 0).all()
    h = d_cmp.cpu().numpy()
    inside = np.zeros(o, bool)
    for i, w in enumerate(wants):
        assert int(clen[i]) == len(w) and np.array_equal(h[c_off[i]: c_off[i] + len(w)], w), i
        inside[c_off[i]: c_off[i] + ccap[i]] = True
    assert (h[~inside] == 0x5A).all()
    dcap = [len(x) + 16 for x in xs]
    d_off, o = [], 32
    for c in dcap:
        d_off.append(o)
        o += (c + 15) // 16 * 16 + 32
    d_dec = torch.full((o,), 0x5A, dtype=torch.uint8, device=dev)
    dlen, st = gpu.decompress_streams_device(d_cmp, c_off, clen, d_dec, d_off, dcap)
    assert (st == 0).all()
    h = d_dec.cpu().numpy()
    inside = np.zeros(o, bool)
    for i, x in enumerate(xs):
        assert int(dlen[i]) == len(x) and np.array_equal(h[d_off[i]: d_off[i] + len(x)], x), i
        inside[d_off[i]: d_off[i] + dcap[i]] = True
    assert (h[~inside] == 0x5A).all()


@pytest.mark.parametrize("level", ["l3", "l5"])
def test_twenty_thousand_small_streams(gpu, oracle, synth, level):
    tr, en = LEVELS[level]
    rng = np.random.default_rng(11)
    sizes = rng.integers(0, 4097, 20000)
    slab = synth.markov_text(int(sizes.sum()) + 1, seed=12)
    xs, o = [], 0
    for n in sizes:
        xs.append(slab[o: o + int(n)])
        o += int(n)
    outs, st = gpu.compress_streams(xs, tr, en, BS)
    assert (st == 0).all()
    for i, x in enumerate(xs):
        assert np.array_equal(outs[i], oracle.compress(x, tr, en, block_size=BS)), i
    ys, st = gpu.decompress_streams(outs, [len(x) for x in xs])
    assert (st == 0).all()
    for i, x in enumerate(xs):
        assert np.array_equal(ys[i], x), i


def test_empty_batch_and_bad_arguments(gpu, kz):
    outs, st = gpu.compress_streams([], "NONE", "NONE", BS)
    assert outs == [] and len(st) == 0
    ys, st = gpu.decompress_streams([], [])
    assert ys == [] and len(st) == 0
    outs, st = gpu.compress_streams([np.zeros(10, np.uint8)] * 3, "NONE", "NONE", 1000)  # not a multiple of 16: the call fails
    assert list(st) == [-18] * 3 and outs == [None] * 3  # KZ_ERR_INVALID_PARAM
