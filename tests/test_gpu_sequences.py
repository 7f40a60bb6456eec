"""GPU parity tests for RANK / MTFT (SBRT), ZRLT and transform sequences such as BWT+RANK+ZRLT (the chain of kanzi -l 5):
single transforms through kz_transform_forward/inverse, sequences through the block batch and whole stream entry points
(ByteTransformSequence skip flags included)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def cases(synth, n, seed):
    rng = np.random.default_rng(seed)
    yield "text", synth.markov_text(n, seed=seed)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 1)
    yield "const0", np.zeros(n, np.uint8)
    yield "const", np.full(n, 65, np.uint8)
    yield "geometric", (np.minimum(rng.geometric(0.45, n), 255) - 1).astype(np.uint8)
    z = synth.uniform_bytes(n, seed=seed + 4)
    z[z < 200] = 0
    yield "zero_runs", z
    f = synth.uniform_bytes(n, seed=seed + 5)
    f[f < 128] = 0xFF
    f[(f >= 128) & (f < 160)] = 0xFE
    f[(f >= 160) & (f < 200)] = 0
    yield "escapes", f
    yield "ramp", (np.arange(n) % 256).astype(np.uint8)
    lo = synth.uniform_bytes(n, seed=seed + 6) & 1
    yield "bits", lo.astype(np.uint8)


SIZES = [1, 2, 3, 15, 16, 17, 100, 4095, 4096, 4097, 8191, 8192, 8193, 16384, 20000, 65536 + 5, 300000, (1 << 20) + 3]


@pytest.mark.parametrize("name", ["RANK", "MTFT", "ZRLT"])
@pytest.mark.parametrize("n", SIZES)
def test_single_transform_parity(gpu, oracle, synth, kz, name, n):
    t = kz.TRANSFORM_IDS[name]
    for cname, x in cases(synth, n, seed=n):
        want, _ = oracle.transform_forward(t, x)
        got, _ = gpu.transform_forward(t, x)
        if want is None:
            assert got is None, (name, cname, n)
            continue
        assert got is not None, (name, cname, n)
        assert len(got) == len(want) and np.array_equal(got, want), (name, cname, n, len(got), len(want),
                                                                      int(np.argmax(got[: min(len(got), len(want))] != want[: min(len(got), len(want))])))
        back = gpu.transform_inverse(t, want, n + 64)
        assert np.array_equal(back, x), (name, cname, n)


@pytest.mark.parametrize("name", ["RANK", "MTFT"])
def test_single_transform_parity_above_16mib(gpu, oracle, synth, kz, name):
    """a block longer than 16 MiB: the inverse takes the one-warp kernel with 64-bit list entries, the only one for such blocks"""
    n = (16 << 20) + 4097
    t = kz.TRANSFORM_IDS[name]
    x = synth.markov_text(n, seed=n)
    want, _ = oracle.transform_forward(t, x)
    got, _ = gpu.transform_forward(t, x)
    assert want is not None and got is not None and np.array_equal(got, want), (name, n)
    assert np.array_equal(gpu.transform_inverse(t, want, n + 64), x), name


BWTS_SIZES = [1, 2, 3, 7, 16, 100, 255, 256, 257, 1000, 4096, 65536, 100003, 1 << 20]


@pytest.mark.parametrize("n", BWTS_SIZES)
def test_bwts_parity(gpu, oracle, synth, kz, n):
    """BWTS.Forward / BWTS.Inverse (transform/BWTS.go): rotations of the Lyndon factors in infinite-periodic order"""
    extra = [("abab", np.resize(np.array([1, 2], np.uint8), n)), ("descending", (255 - (np.arange(n) * 255 // max(n, 1))).astype(np.uint8)),
             ("repeat7", np.resize(synth.markov_text(max(n // 7, 1), seed=n + 3), n)), ("aab", np.resize(np.array([1, 1, 2], np.uint8), n))]
    for cname, x in list(cases(synth, n, seed=n)) + extra:
        want, _ = oracle.transform_forward(kz.T_BWTS, x)
        got, _ = gpu.transform_forward(kz.T_BWTS, x)
        assert want is not None and got is not None, (cname, n)
        assert np.array_equal(got, want), (cname, n, int(np.argmax(got != want)))
        assert np.array_equal(gpu.transform_inverse(kz.T_BWTS, want, n + 64), x), (cname, n)


def test_zrlt_long_runs(gpu, oracle, synth, kz):
    """runs that cross many tiles, a block that is one run, a run at the very end"""
    for n, pat in [(1 << 20, "all"), (1 << 20, "tail"), (300000, "mid")]:
        x = np.zeros(n, np.uint8)
        if pat == "tail":
            x[: n // 3] = synth.markov_text(n // 3, seed=1)
        elif pat == "mid":
            x[:1000] = 7
            x[-1000:] = 9
        want, _ = oracle.transform_forward(kz.T_ZRLT, x)
        got, _ = gpu.transform_forward(kz.T_ZRLT, x)
        assert want is not None and got is not None and np.array_equal(got, want), (n, pat)
        assert np.array_equal(gpu.transform_inverse(kz.T_ZRLT, want, n + 64), x)


@pytest.mark.parametrize("seq,entropy", [("BWT+RANK+ZRLT", "ANS0"), ("BWT+MTFT+ZRLT", "HUFFMAN"), ("RANK", "ANS0"), ("ZRLT", "NONE"), ("RANK+ZRLT", "ANS1"),
                                         ("BWT+ZRLT", "RANGE"), ("BWTS", "ANS0"), ("BWTS+MTFT+ZRLT", "HUFFMAN")])
@pytest.mark.parametrize("n,bs", [(10, 1024), (5000, 1024), (70000, 65536), (3 * (1 << 20) + 777, 1 << 20)])
def test_stream_parity_sequences(gpu, oracle, synth, kz, seq, entropy, n, bs):
    for kind in ("text", "uniform"):
        x = synth.markov_text(n, seed=n + 1) if kind == "text" else synth.uniform_bytes(n, seed=n + 2)
        want = oracle.compress(x, seq, entropy, block_size=bs, jobs=8, input_size=n)
        got = gpu.compress(x, seq, entropy, block_size=bs, input_size=n)
        assert len(got) == len(want) and np.array_equal(got, want), (seq, entropy, n, bs, kind, len(got), len(want))
        assert np.array_equal(gpu.decompress(want, n + 64), x), (seq, entropy, n, bs, kind)


def test_block_batch_sequence(gpu, oracle, synth, kz):
    lens = [1, 15, 16, 300, 5000, 70000, 200000]
    blocks = [synth.markov_text(n, seed=500 + i) if i % 2 == 0 else synth.uniform_bytes(n, seed=500 + i) for i, n in enumerate(lens)]
    t48 = kz.transform_type("BWT+RANK+ZRLT")
    et = oracle.parse_entropy("ANS0")
    got = gpu.encode_blocks(t48, et, blocks)
    payloads = []
    for i, (b, (g, gbits)) in enumerate(zip(blocks, got)):
        w, wbits = oracle.encode_block(b, t48, et)
        assert gbits == wbits and np.array_equal(g, w), (i, lens[i], gbits, wbits)
        payloads.append((w, wbits))
    dec = gpu.decode_blocks(t48, et, payloads, block_size=1 << 18)
    for i, (b, d) in enumerate(zip(blocks, dec)):
        assert np.array_equal(b, d), (i, lens[i])


def test_level5_chain_4mib_blocks(gpu, oracle, synth, kz):
    """-t BWT+RANK+ZRLT -e ANS0 on 16 MiB of text in 4 MiB blocks (the GPU covered part of kanzi -l 5)"""
    n = 16 << 20
    x = synth.markov_text(n, seed=77)
    got = gpu.compress(x, "BWT+RANK+ZRLT", "ANS0", block_size=4 << 20, input_size=n)
    assert np.array_equal(gpu.decompress(got, n + 64), x)
    want = oracle.compress(x, "BWT+RANK+ZRLT", "ANS0", block_size=4 << 20, jobs=8, input_size=n)
    assert len(got) == len(want) and np.array_equal(got, want)
