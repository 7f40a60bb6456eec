"""GPU tests of many streams with a block size each (kz_compress_streams_bs[_device], kanzi's `-b auto` over many files) and of one decode call
over streams that differ in block size: every stream equals the single-stream call with its block size (and the oracle's), TEXT sizes each
block's hash map by its own stream's block size, streams that differ only in block size share every launch, and a bad block size, a small
output or a corrupt stream fails only its own stream."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CHAINS = {"l2": ("DNA+LZ", "HUFFMAN"), "l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0"),
          "bwts-ans1": ("BWTS", "ANS1"), "none": ("NONE", "NONE")}
INVALID_PARAM = -18


def files(synth, n=300, seed=1):
    """n files of log-normal sizes from 0 B to 2 MiB in three kinds of data"""
    rng = np.random.default_rng(seed)
    sizes = np.minimum(rng.lognormal(np.log(24 << 10), 1.6, n).astype(np.int64), 2 << 20)
    sizes[rng.integers(0, n, 8)] = 0
    gens = [lambda k, s: synth.markov_text(k, seed=s), lambda k, s: synth.english_text(k, seed=s), lambda k, s: synth.x86_like(k, seed=s)]
    return [np.ascontiguousarray(gens[i % 3](int(k), seed + i)[: int(k)], np.uint8) if k else np.zeros(0, np.uint8) for i, k in enumerate(sizes)]


def pack_device(torch, arrs, pad=64):
    """arrs on the device at 16-byte aligned offsets with pad readable bytes behind each -> (tensor, offsets)"""
    offs, o = [], 0
    for a in arrs:
        offs.append(o)
        o += (len(a) + 15) // 16 * 16
    d = torch.zeros(o + pad, dtype=torch.uint8, device="cuda:0")
    for a, at in zip(arrs, offs):
        if len(a):
            d[at: at + len(a)] = torch.from_numpy(a).to(d.device)
    return d, offs


@pytest.fixture(scope="module")
def corpus(synth, kz):
    xs = files(synth)
    return xs, [kz.auto_block_size(len(x), 4) for x in xs]


@pytest.mark.parametrize("ck", [0, 32, 64])
@pytest.mark.parametrize("level", list(CHAINS))
def test_parity_with_single_calls(gpu, oracle, kz, corpus, level, ck):
    torch = pytest.importorskip("torch")
    tr, en = CHAINS[level]
    xs, bs = corpus
    assert len(set(bs)) > len(xs) // 2 and sum(-(-len(x) // b) >= 2 for x, b in zip(xs, bs)) > len(xs) // 2
    isz = [len(x) if i % 3 == 0 else 0 for i, x in enumerate(xs)]
    outs, st = gpu.compress_streams(xs, tr, en, bs, ck, isz)
    assert (st == 0).all(), st
    for i, x in enumerate(xs):
        assert np.array_equal(outs[i], gpu.compress(x, tr, en, bs[i], ck, isz[i])), (level, i, len(x), bs[i])
    for i in np.random.default_rng(ck + len(tr)).choice(len(xs), 20, replace=False):
        want = oracle.compress(xs[i], tr, en, block_size=bs[i], checksum_bits=ck, input_size=isz[i])
        assert np.array_equal(outs[i], want), (level, i, len(xs[i]), bs[i])
    caps = [len(x) + 64 for x in xs]
    ys, st = gpu.decompress_streams(outs, caps)
    assert (st == 0).all(), st
    for i, x in enumerate(xs):
        assert np.array_equal(ys[i], x), (level, i)
    # the device variants give what the host variants give
    d_src, s_off = pack_device(torch, xs)
    ccap = [int(gpu.lib.kz_max_stream_output(len(x), b)) for x, b in zip(xs, bs)]
    c_off = np.concatenate([[0], np.cumsum([(c + 15) // 16 * 16 for c in ccap])]).astype(np.uint64)
    d_cmp = torch.zeros(int(c_off[-1]) + 64, dtype=torch.uint8, device="cuda:0")
    clen, st = gpu.compress_streams_device(d_src, s_off, [len(x) for x in xs], d_cmp, c_off[:-1], ccap, tr, en, bs, ck, isz)
    assert (st == 0).all(), st
    h = d_cmp.cpu().numpy()
    for i in range(len(xs)):
        assert int(clen[i]) == len(outs[i]) and np.array_equal(h[int(c_off[i]): int(c_off[i]) + int(clen[i])], outs[i]), (level, i)
    d_off = np.concatenate([[0], np.cumsum([(c + 15) // 16 * 16 for c in caps])]).astype(np.uint64)
    d_dec = torch.zeros(int(d_off[-1]) + 16, dtype=torch.uint8, device="cuda:0")
    dlen, st = gpu.decompress_streams_device(d_cmp, c_off[:-1], clen, d_dec, d_off[:-1], caps)
    assert (st == 0).all(), st
    h = d_dec.cpu().numpy()
    for i, x in enumerate(xs):
        assert int(dlen[i]) == len(x) and np.array_equal(h[int(d_off[i]): int(d_off[i]) + len(x)], x), (level, i)
    del d_src, d_cmp, d_dec
    torch.cuda.empty_cache()


def words_text(n, seed, vocab=None):
    """n bytes of random lower-case words of 3 to 8 letters, from a vocabulary of `vocab` words (None: every word drawn afresh, so almost
    all are distinct): many distinct words, so the size of TEXT's hash map matters"""
    rng = np.random.default_rng(seed)
    if vocab is None:
        out = rng.integers(97, 123, n).astype(np.uint8)
        ends = np.cumsum(rng.integers(4, 10, n // 4 + 1))  # a word and its space
        out[ends[ends <= n] - 1] = 0x20
        return out
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8)
    words = [bytes(letters[rng.integers(0, 26, int(rng.integers(3, 9)))]) + b" " for _ in range(vocab)]
    picks = rng.integers(0, vocab, n // 3 + 1)
    return np.frombuffer(b"".join(words[int(k)] for k in picks)[:n], np.uint8).copy()


TEXT_SIZES = [512 << 10, 1 << 20, 4 << 20, 16 << 20]  # lg 14, 15, 17, 19


@pytest.mark.parametrize("skip", [False, True], ids=["noskip", "skip"])
@pytest.mark.parametrize("level", ["l3", "l5"])
def test_text_hash_size_per_block(gpu, level, skip):
    tr, en = CHAINS[level]
    x = words_text(256 << 10, 7, 20000)
    single = [gpu.compress(x, tr, en, b, skip_blocks=skip) for b in TEXT_SIZES]
    # the payloads must depend on the hash size, or this test could not tell per-block sizes from one shared size
    assert len({len(s) for s in single}) >= 2, [len(s) for s in single]
    order = [0, 3, 1, 2, 2, 0, 3, 1, 1, 3, 0, 2]
    outs, st = gpu.compress_streams([x] * len(order), tr, en, [TEXT_SIZES[k] for k in order], skip_blocks=skip)
    assert (st == 0).all(), st
    for i, k in enumerate(order):
        assert np.array_equal(outs[i], single[k]), (level, i, TEXT_SIZES[k])
    ys, st = gpu.decompress_streams(outs, [len(x)] * len(order))
    assert (st == 0).all(), st
    for y in ys:
        assert np.array_equal(y, x)


def test_text_large_blocks_with_mixed_sizes(gpu, oracle):
    """5 MiB blocks of about 680,000 distinct words beside small blocks, at hash sizes 2^17 .. 2^19 in one batch"""
    tr, en = CHAINS["l3"]
    big = words_text(5 << 20, 9)
    small = words_text(200 << 10, 10, 20000)
    xs, bs = [big, small, big, small], [8 << 20, 2 << 20, 16 << 20, 16 << 20]
    outs, st = gpu.compress_streams(xs, tr, en, bs)
    assert (st == 0).all(), st
    for i, x in enumerate(xs):
        want = oracle.compress(x, tr, en, block_size=bs[i])
        assert np.array_equal(outs[i], want), (i, bs[i])
    ys, st = gpu.decompress_streams(outs, [len(x) for x in xs])
    assert (st == 0).all(), st
    for x, y in zip(xs, ys):
        assert np.array_equal(y, x)


def single_result(gpu, kz, s, cap):
    try:
        return 0, gpu.decompress(s, cap)
    except kz.KanziError as e:
        return e.code, None


def test_text_serial_walk_with_mixed_sizes(gpu, kz):
    """TEXT blocks whose tokens name dictionary entries that do not exist yet leave the data-parallel inverse for the serial walk, which
    then runs over blocks of four hash sizes in one batch (each with its own map slice): every stream gets what decoding it alone gives"""
    x = words_text(256 << 10, 7, 20000)
    order = [0, 3, 1, 2, 2, 0, 3, 1]
    outs, st = gpu.compress_streams([x] * len(order), "TEXT", "NONE", [TEXT_SIZES[k] for k in order])
    assert (st == 0).all(), st
    streams = [o.copy() for o in outs]
    for i in (1, 2, 5, 6):  # index tokens past the dictionary in the block payload (TEXT + NONE: the payload is TEXT's output)
        s = streams[i]
        for p in range(len(s) // 4, len(s) - 64, len(s) // 9):
            s[p: p + 3] = 0xFF
    caps = [len(x) + 4096] * len(order)
    gpu.profile(True)
    gpu.profile_reset()
    try:
        ys, st = gpu.decompress_streams(streams, caps)
        walked = gpu.kernel_time("text_inverse_serial")[0]
    finally:
        gpu.profile(False)
    assert walked >= 1, walked
    for i in range(len(order)):
        code, want = single_result(gpu, kz, streams[i], caps[i])
        assert st[i] == -code, (i, st[i], code)
        if code == 0:
            assert np.array_equal(ys[i], want), i
    for i in (0, 3, 4, 7):
        assert st[i] == 0 and np.array_equal(ys[i], x), i


@pytest.mark.parametrize("chain", [("LZX", "HUFFMAN"), ("BWT+RANK+ZRLT", "ANS0")], ids=["lzx-huffman", "bwt-ans0"])
def test_block_sizes_share_launches(gpu, synth, chain):
    tr, en = chain
    x = synth.markov_text(3 << 10, seed=21)
    xs = [x] * 64
    counts = {}
    for name, bs in [("U", [4096] * 64), ("M", [4096 + 64 * s for s in range(64)])]:
        gpu.launch_count(reset=True)
        outs, st = gpu.compress_streams(xs, tr, en, bs)
        assert (st == 0).all()
        c_comp = gpu.launch_count(reset=True)
        ys, st = gpu.decompress_streams(outs, [len(x)] * 64)
        assert (st == 0).all() and all(np.array_equal(y, x) for y in ys)
        counts[name] = (c_comp, gpu.launch_count(reset=True))
    assert counts["U"][0] == counts["M"][0], counts
    assert counts["U"][1] == counts["M"][1], counts


def test_text_hash_sizes_share_launches(gpu, synth):
    """-l 3 with one block per stream and block sizes of 512 KiB and 1 MiB (TEXT hash sizes 2^14 and 2^15) in one batch, whose blocks share
    one compress pass and one decode pass (their decode slots are within a factor of two). The dictionary rounds run until every block of a
    sub-batch settles, and how many a block needs depends on its hash size; with the same content in every stream, the mixed batch makes as
    many launches as the uniform batch of its slowest hash size: no launch depends on the number of hash sizes."""
    tr, en = CHAINS["l3"]
    x = synth.english_text(3 << 10, seed=22)
    sizes = [512 << 10, 1 << 20]

    def launches(bs):
        gpu.launch_count(reset=True)
        outs, st = gpu.compress_streams([x] * len(bs), tr, en, bs)
        assert (st == 0).all()
        c_comp = gpu.launch_count(reset=True)
        ys, st = gpu.decompress_streams(outs, [len(x)] * len(bs))
        assert (st == 0).all() and all(np.array_equal(y, x) for y in ys)
        return c_comp, gpu.launch_count(reset=True)

    uniform = [launches([b] * 32) for b in sizes]
    mixed = launches([sizes[s % 2] for s in range(32)])
    assert mixed == (max(u[0] for u in uniform), max(u[1] for u in uniform)), (mixed, uniform)


def test_decode_pass_over_a_grid_of_blocks(gpu, synth):
    """65,600 blocks of one block size in one decode call: two passes (a pass holds at most 65,535 blocks, the rows of a grid), and no
    stream falls back to the single-stream decode"""
    n, size = 4100, 16 << 10
    slab = synth.zipf_bytes(n * size, 1.1, seed=23)
    xs = [slab[i * size: (i + 1) * size] for i in range(n)]
    outs, st = gpu.compress_streams(xs, "LZX", "NONE", [1024] * n)
    assert (st == 0).all()
    gpu.profile(True)
    gpu.profile_reset()
    try:
        ys, st = gpu.decompress_streams(outs, [size] * n)
        walks, passes = gpu.kernel_time("stream_walk")[0], gpu.kernel_time("block_header")[0]
    finally:
        gpu.profile(False)
    assert (st == 0).all()
    assert all(np.array_equal(y, x) for x, y in zip(xs, ys))
    assert walks == 1 and passes == 2, (walks, passes)


def test_bad_block_sizes_fail_alone(gpu, synth):
    tr, en = CHAINS["l3"]
    xs = [synth.markov_text(n, seed=n) for n in (5000, 70000, 3000, 9000, 40000, 1200)]
    bs = [4096, 1000, 16384, 1032, (1 << 30) + 16, 1024]
    outs, st = gpu.compress_streams(xs, tr, en, bs)
    assert list(st) == [0, INVALID_PARAM, 0, INVALID_PARAM, INVALID_PARAM, 0]
    for i in (0, 2, 5):
        assert np.array_equal(outs[i], gpu.compress(xs[i], tr, en, bs[i])), i
    assert outs[1] is None and outs[3] is None and outs[4] is None


def test_small_dst_cap_and_empty_inputs(gpu, synth, kz):
    tr, en = CHAINS["l5"]
    xs = [synth.markov_text(5000, seed=1), synth.markov_text(70000, seed=2), np.zeros(0, np.uint8), synth.markov_text(300, seed=3),
          np.zeros(0, np.uint8)]
    bs = np.array([1024, 8192, 1 << 30, 2048, 1040], np.uint32)
    full = [gpu.compress(x, tr, en, int(b)) for x, b in zip(xs, bs)]
    cap = np.array([len(full[0]), len(full[1]) - 1, len(full[2]), len(full[3]) + 100, len(full[4])], np.uint64)
    dst_off = np.array([0, 8192, 108192, 108288, 110000], np.uint64)
    dst = np.full(111000, 0xA5, np.uint8)
    src = np.concatenate(xs)
    src_len = np.array([len(x) for x in xs], np.uint64)
    src_off = np.concatenate([[0], np.cumsum(src_len)[:-1]]).astype(np.uint64)
    out_len, st = np.zeros(5, np.uint64), np.zeros(5, np.int32)
    rc = gpu.lib.kz_compress_streams_bs(gpu.h, kz.transform_type(tr), kz.entropy_type(en), bs.ctypes.data, 0, 5, src.ctypes.data, src_off.ctypes.data,
                                        src_len.ctypes.data, None, dst.ctypes.data, dst_off.ctypes.data, cap.ctypes.data, out_len.ctypes.data,
                                        st.ctypes.data)
    assert rc == -12 and list(st) == [0, -12, 0, 0, 0]  # KZ_ERR_WRITE_FILE for the stream that does not fit, and only for it
    assert int(out_len[1]) == len(full[1])
    inside = np.zeros(len(dst), bool)
    for i in (0, 2, 3, 4):
        a = int(dst_off[i])
        assert int(out_len[i]) == len(full[i]) and np.array_equal(dst[a: a + len(full[i])], full[i]), i
        inside[a: a + len(full[i])] = True
    assert (dst[~inside] == 0xA5).all()
    ys, st = gpu.decompress_streams([full[i] for i in (0, 2, 3, 4)], [6000, 16, 400, 16])
    assert (st == 0).all() and [len(y) for y in ys] == [5000, 0, 300, 0]


def test_null_block_size_array_is_a_call_level_error(gpu, kz):
    xs = [np.zeros(100, np.uint8), np.zeros(5000, np.uint8)]
    src = np.concatenate(xs)
    src_off, src_len = np.array([0, 100], np.uint64), np.array([100, 5000], np.uint64)
    cap = np.array([10000, 10000], np.uint64)
    dst_off = np.array([0, 10000], np.uint64)
    dst = np.zeros(20000, np.uint8)
    out_len, st = np.full(2, 7, np.uint64), np.zeros(2, np.int32)
    rc = gpu.lib.kz_compress_streams_bs(gpu.h, 0, 0, None, 0, 2, src.ctypes.data, src_off.ctypes.data, src_len.ctypes.data, None, dst.ctypes.data,
                                        dst_off.ctypes.data, cap.ctypes.data, out_len.ctypes.data, st.ctypes.data)
    assert rc == INVALID_PARAM and list(st) == [INVALID_PARAM] * 2 and list(out_len) == [0, 0]
    assert (dst == 0).all()
    with pytest.raises(kz.KanziError):
        gpu.compress_streams(xs, "NONE", "NONE", [4096])  # one block size for two streams


def single_code(gpu, kz, s, cap):
    try:
        gpu.decompress(s, cap)
    except kz.KanziError as e:
        return e.code
    return 0


def test_corrupt_stream_in_mixed_block_sizes(gpu, oracle, synth, kz):
    rng = np.random.default_rng(4)
    kinds = [("NONE", "NONE", 32), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 0), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 32)]
    xs, streams, caps = [], [], []
    for i in range(30):
        tr, en, ck = kinds[i % 3]
        x = synth.zipf_bytes(int(rng.integers(1000, 120000)), 1.0, seed=300 + i)
        xs.append(x)
        streams.append(oracle.compress(x, tr, en, block_size=kz.auto_block_size(len(x), 4), checksum_bits=ck, input_size=len(x)))
        caps.append(len(x) + 64)
    bad = {}
    s = streams[3].copy()  # NONE / NONE, 32-bit checksums
    s[len(s) // 2] ^= 0x10
    streams[3], bad[3] = s, "checksum"
    s = streams[7]
    streams[7], bad[7] = s[: len(s) // 2].copy(), "truncated"
    s = streams[11].copy()
    s[len(s) - 40] ^= 0xFF
    streams[11], bad[11] = s, "payload"
    caps[14], bad[14] = len(xs[14]) - 1, "cap"
    ys, st = gpu.decompress_streams(streams, caps)
    for i in range(len(xs)):
        code = single_code(gpu, kz, streams[i], caps[i])
        if i in bad and code:
            assert st[i] == -code and ys[i] is None, (i, bad[i], st[i], code)
        else:
            assert code == 0 and st[i] == 0 and np.array_equal(ys[i], xs[i]), (i, st[i])
    assert -st[3] == 19 and -st[14] == 12 and st[7] != 0
