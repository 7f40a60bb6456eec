"""GPU parity of the RANK / MTFT forward (kz_sbrt.cu): 32-bit keys in a shared-memory table for batches whose blocks are at most 16 MiB,
64-bit keys for a batch with a longer block. Every batch mixes block lengths and is checked block by block against the oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def tie_heavy(n, seed):
    """RANK q = (l1 + l2) >> 1 collides for different symbols all the time: a 3-symbol alphabet, and pairs of symbols placed symmetrically
    around one centre with gaps above 2 x 254 (clipped keys, equal q) in random filler"""
    r = np.random.default_rng(seed)
    if seed % 2:
        return r.integers(0, 3, n).astype(np.uint8)
    x = r.integers(16, 256, n).astype(np.uint8)
    for b in range(0, n - 2048, 2048):
        a, c = 2 * (b // 2048 % 8), 2 * (b // 2048 % 8) + 1
        x[b], x[b + 1000], x[b + 100 + (b // 2048 & 1)], x[b + 900] = a, a, c, c
        x[b + 1001], x[b + 1002] = c, a
    return x


def check_batch(gpu, oracle, kz, name, blocks):
    t48 = kz.transform_type(name)
    blocks = [np.ascontiguousarray(b, np.uint8) for b in blocks]
    got = gpu.encode_blocks(t48, kz.E_NONE, blocks)
    for i, b in enumerate(blocks):
        w, wbits = oracle.encode_block(b, t48, oracle.E_NONE)
        g, gbits = got[i]
        assert gbits == wbits and np.array_equal(g, w), (name, i, len(b))


@pytest.mark.parametrize("name", ["RANK", "MTFT"])
def test_mixed_lengths_32bit_keys(gpu, oracle, synth, kz, name):
    """1 byte .. exactly 16 MiB (the longest block with 32-bit keys) in one batch; tie-heavy, uniform and text blocks"""
    blocks = [np.array([200], np.uint8), synth.uniform_bytes(15, seed=1), tie_heavy(4095, 2), tie_heavy(4097, 3), synth.uniform_bytes(4096, seed=4),
              tie_heavy(300001, 6), synth.uniform_bytes(MIB + 7, seed=7), synth.markov_text(4 * MIB, seed=8), tie_heavy(16 * MIB, 9)]
    check_batch(gpu, oracle, kz, name, blocks)


@pytest.mark.parametrize("name", ["RANK", "MTFT"])
def test_mixed_lengths_with_a_block_above_16mib(gpu, oracle, synth, kz, name):
    """a block of 16 MiB + 1 sends the batch to the 64-bit keys; the 1-byte and tie-heavy blocks beside it take the same kernel"""
    blocks = [np.array([3], np.uint8), tie_heavy(16 * MIB + 1, 10), synth.uniform_bytes(70000, seed=11), tie_heavy(5000, 12)]
    check_batch(gpu, oracle, kz, name, blocks)


def test_level5_stream_of_silesia_shaped_blocks(gpu, oracle, synth):
    """kanzi -l 5 (TEXT+UTF+BWT+RANK+ZRLT & ANS0) on 3 x 4 MiB of the bench's silesia-shaped data: the whole stream equals the oracle's"""
    x = synth.silesia_shaped(12 * MIB, seed=21)
    got = gpu.compress(x, "TEXT+UTF+BWT+RANK+ZRLT", "ANS0", block_size=4 * MIB, input_size=len(x))
    want = oracle.compress(x, "TEXT+UTF+BWT+RANK+ZRLT", "ANS0", block_size=4 * MIB, jobs=3, input_size=len(x))
    assert np.array_equal(got, want)
    assert np.array_equal(gpu.decompress(got, len(x) + 1024), x)
