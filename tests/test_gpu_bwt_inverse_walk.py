"""The BWT inverse's walk (bwt_inverse_batch, kz_bwt.cu): one-word LF entries (32-bit below 2^24 bytes per block, 64-bit above), one walk
per sub-list into a staging slot, the copy of the slots and the walk on past a full slot. Every result is checked against the oracle's
inverse; the walk shape (kz_bwt_profile bits 8-19: stride and slot size) never changes the bytes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _bwt(oracle, x):
    enc, _ = oracle.transform_forward(oracle.T_BWT, x)
    return enc


def _check_inverse(gpu, oracle, kz, enc, x=None):
    want = oracle.transform_inverse(oracle.T_BWT, enc, len(enc) + 64)
    if x is not None:
        assert np.array_equal(want, x)
    got = gpu.transform_inverse(kz.T_BWT, enc, len(enc) + 64)
    assert len(got) == len(want) and np.array_equal(got, want)


@pytest.fixture
def shaped(gpu):
    """the session context with a walk shape for one test; the default shape again afterwards"""

    def set_shape(stride=0, stage=0):
        gpu.bwt_profile(inverse_stride=stride, inverse_stage=stage)

    yield set_shape
    gpu.bwt_profile()


def test_random_4mib_blocks(gpu, oracle, kz):
    """incompressible bytes: sub-list lengths are about geometric, so many sub-lists are longer than the staging slot"""
    rng = np.random.default_rng(11)
    for k in range(2):
        x = rng.integers(0, 256, 4 << 20, dtype=np.uint8)
        enc, _ = gpu.transform_forward(kz.T_BWT, x)
        _check_inverse(gpu, oracle, kz, enc, x)


@pytest.mark.parametrize("n", [2, 3, 255, 256, 1000, 100000])
def test_one_repeated_byte(gpu, oracle, kz, n):
    _check_inverse(gpu, oracle, kz, _bwt(oracle, np.full(n, 97, np.uint8)))


@pytest.mark.parametrize("x", [[1, 2], [2, 1], [5, 5], [1, 2, 3], [3, 2, 1], [7, 7, 1], [0, 255, 0]])
def test_two_and_three_bytes(gpu, oracle, kz, x):
    x = np.array(x, np.uint8)
    _check_inverse(gpu, oracle, kz, _bwt(oracle, x), x)


@pytest.mark.parametrize("n", [31, 33, 63, 65, 127, 129, 4095, 4097, 65536 + 17, 300001])
def test_lengths_off_the_stride(gpu, oracle, synth, kz, n):
    x = synth.markov_text(n, seed=n) if n % 2 else synth.zipf_bytes(n, 1.1, seed=n)
    _check_inverse(gpu, oracle, kz, _bwt(oracle, x), x)


def test_primary_on_stride_multiples(gpu, oracle, synth, kz):
    """blocks whose first primary rank is a multiple of the stride (the primary head coincides with a stride head and is dropped)"""
    found = 0
    for seed in range(1000):
        n = 1000 + seed * 37
        x = synth.zipf_bytes(n, 1.2, seed=seed)
        enc = _bwt(oracle, x)
        psize = int(enc[0] & 3) + 1
        if int.from_bytes(bytes(enc[1: 1 + psize]), "big") % 32:  # the first primary rank, as the header stores it
            continue
        found += 1
        _check_inverse(gpu, oracle, kz, enc, x)
        if found >= 6:
            break
    assert found >= 3


@pytest.fixture(scope="module")
def mixed_batch(oracle, synth, kz):
    rng = np.random.default_rng(3)
    sizes = [int(s) for s in rng.choice([2, 3, 17, 64, 255, 256, 1000, 4096, 33333, 100000, 250000], 256)]
    blocks = []
    for i, n in enumerate(sizes):
        if i % 3 == 0:
            blocks.append(rng.integers(0, 256, n, dtype=np.uint8))
        elif i % 3 == 1:
            blocks.append(synth.markov_text(n, seed=i))
        else:
            blocks.append(np.full(n, i & 255, np.uint8))
    t = kz.transform_type("BWT")
    payloads = [oracle.encode_block(b, t, oracle.E_NONE) for b in blocks]
    for b in blocks:
        assert np.array_equal(oracle.transform_inverse(oracle.T_BWT, _bwt(oracle, b), len(b) + 64), b)
    return t, blocks, payloads


@pytest.mark.parametrize("shape", [(0, 0), (64, 16), (16, 16), (32, 256), (2, 16)])
def test_batch_of_256_mixed_blocks(gpu, kz, shaped, mixed_batch, shape):
    """256 blocks of mixed sizes in one batch (every thread of the walk takes sub-lists of several blocks), with small and large slots"""
    shaped(*shape)
    t, blocks, payloads = mixed_batch
    dec = gpu.decode_blocks(t, kz.E_NONE, payloads, block_size=256 << 10)
    for i, (b, d) in enumerate(zip(blocks, dec)):
        assert np.array_equal(d, b), (i, len(b))


@pytest.mark.parametrize("n", [(1 << 24) - 1, 1 << 24])
def test_blocks_around_the_word_width(gpu, oracle, kz, n):
    """the largest block of 32-bit LF words and the smallest of 64-bit ones"""
    rng = np.random.default_rng(n & 0xFF)
    x = rng.integers(0, 64, n, dtype=np.uint8)
    enc, _ = gpu.transform_forward(kz.T_BWT, x)
    _check_inverse(gpu, oracle, kz, enc, x)


def test_block_32mib_wide_words(gpu, oracle, synth, kz):
    n = 32 << 20
    x = synth.markov_text(n, seed=9)
    enc, _ = gpu.transform_forward(kz.T_BWT, x)
    _check_inverse(gpu, oracle, kz, enc, x)


def _single_list(enc):
    """numpy model of the LF mapping bwt_inverse_batch builds: does the list from the first primary rank run through all n ranks?"""
    mode = int(enc[0])
    chunks, psize = 1 << ((mode >> 2) & 7), (mode & 3) + 1
    data = enc[1 + chunks * psize:]
    n = len(data)
    p0 = int.from_bytes(bytes(enc[1: 1 + psize]), "big")
    if p0 + 1 > n:
        return None
    i = np.arange(n)
    val = np.where(i < p0 + 1, i - 1, i)
    nxt = val[np.argsort(data, kind="stable")]
    g, steps = p0, 1
    while steps <= n:
        if nxt[g] < 0:
            break
        g = int(nxt[g])
        steps += 1
    return steps == n


def test_corrupt_payloads_are_reported(gpu, oracle, synth, kz, shaped):
    """several cycles (a changed primary index or data byte) and out-of-range primary indexes: an error, then the engine decodes again"""
    x = synth.markov_text(50000, seed=21)
    enc = _bwt(oracle, x)
    psize = int(enc[0] & 3) + 1
    rng = np.random.default_rng(8)
    multi = 0
    for shape in [(0, 0), (64, 16), (16, 64)]:
        shaped(*shape)
        for trial in range(24):
            bad = enc.copy()
            if trial < 12:
                p = int(rng.integers(0, len(x)))
                bad[1: 1 + psize] = np.frombuffer(p.to_bytes(psize, "big"), np.uint8)
            else:
                pos = int(rng.integers(40, len(bad)))
                bad[pos] ^= 1 << int(rng.integers(0, 8))
            single = _single_list(bad)
            if single:
                got = gpu.transform_inverse(kz.T_BWT, bad, len(x) + 64)
                assert len(got) == len(x)
                continue
            multi += 1
            with pytest.raises(kz.KanziError):
                gpu.transform_inverse(kz.T_BWT, bad, len(x) + 64)
        for p in (len(x), len(x) + 5, (1 << (8 * int(psize))) - 1):  # primary rank past the block
            bad = enc.copy()
            bad[1: 1 + psize] = np.frombuffer(p.to_bytes(psize, "big"), np.uint8)
            with pytest.raises(kz.KanziError):
                gpu.transform_inverse(kz.T_BWT, bad, len(x) + 64)
        assert np.array_equal(gpu.transform_inverse(kz.T_BWT, enc, len(x) + 64), x)
    assert multi >= 10
