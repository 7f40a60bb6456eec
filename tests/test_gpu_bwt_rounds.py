"""GPU parity of the BWT forward's later doubling rounds: groups of at most BWT_SMALL_GROUP suffixes sorted on chip, larger groups sorted
globally on (large-group ordinal, 23-bit second key), batches with a block above 4 MiB on the 56-bit rounds. Every batch is checked against
the oracle and against the same context forced onto the 56-bit rounds (kz_bwt_profile bit 1)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

G = 256  # BWT_SMALL_GROUP (kz_bwt_core.cuh)


@pytest.fixture(scope="module")
def ctx(kz):
    c = kz.Context(0)
    yield c
    c.close()


def motif_block(n, copies, seed, motif_len=40):
    """random bytes with `copies` copies of one motif: the suffixes at each motif offset form a group of exactly `copies` members for
    the rounds h = 6 .. 24 (random bytes follow every copy)"""
    r = np.random.default_rng(seed)
    x = r.integers(0, 256, n).astype(np.uint8)
    motif = r.integers(0, 256, motif_len).astype(np.uint8)
    step = n // (copies + 1)
    assert step > motif_len + 8
    for k in range(copies):
        o = (k + 1) * step
        x[o: o + motif_len] = motif
    return x


def check_batch(ctx, oracle, kz, blocks):
    t48 = kz.transform_type("BWT")
    blocks = [np.ascontiguousarray(b, np.uint8) for b in blocks]
    got = ctx.encode_blocks(t48, kz.E_NONE, blocks)
    ctx.bwt_profile(wide_rounds=True)
    try:
        wide = ctx.encode_blocks(t48, kz.E_NONE, blocks)
    finally:
        ctx.bwt_profile()
    for i, b in enumerate(blocks):
        w, wbits = oracle.encode_block(b, t48, oracle.E_NONE)
        g, gbits = got[i]
        assert gbits == wbits and np.array_equal(g, w), (i, len(b))
        assert wide[i][1] == gbits and np.array_equal(wide[i][0], g), (i, len(b))


@pytest.mark.parametrize("copies", [G - 1, G, G + 1, 2 * G])
def test_groups_at_the_small_group_limit(ctx, oracle, kz, copies):
    blocks = [motif_block(300000, copies, seed=copies)]
    # the same sizes side by side in one block: small and large groups in one round
    blocks.append(np.concatenate([motif_block(200000, G, seed=1), motif_block(200000, G + 1, seed=2), motif_block(200000, 3, seed=3)]))
    check_batch(ctx, oracle, kz, blocks)


@pytest.mark.parametrize("name", ["repeat7", "abab", "const", "period300"])
def test_one_group_lives_through_every_round(ctx, oracle, synth, kz, name):
    n = 1 << 20
    if name == "repeat7":
        x = np.resize(synth.markov_text(n // 7, seed=4), n)
    elif name == "abab":
        x = np.resize(np.array([1, 2], np.uint8), n)
    elif name == "const":
        x = np.full(n, 65, np.uint8)
    else:
        x = np.resize(np.random.default_rng(5).integers(0, 256, 300).astype(np.uint8), n)
    check_batch(ctx, oracle, kz, [x, synth.markov_text(5000, seed=6)])


def test_small_blocks_beside_a_4mib_block(ctx, oracle, synth, kz):
    blocks = [synth.markov_text(n, seed=10 + n) for n in (2, 3, 17, 255, 256, 4097, 70000)]
    blocks.insert(3, synth.records_like(4 << 20, seed=9))  # exactly 4 MiB: the narrow rounds' largest block
    check_batch(ctx, oracle, kz, blocks)


def test_block_above_4mib_takes_the_wide_rounds(ctx, oracle, synth, kz):
    check_batch(ctx, oracle, kz, [synth.markov_text((4 << 20) + 1, seed=12), synth.markov_text(3000, seed=13)])


def test_tiny_blocks_and_sentinels(ctx, oracle, kz):
    r = np.random.default_rng(14)
    blocks = [np.array([a, b], np.uint8) for a, b in ((0, 0), (0, 255), (255, 0), (7, 7))]
    blocks += [np.array([0, 0, 0], np.uint8), np.array([255, 255, 255], np.uint8), np.array([1, 0, 1], np.uint8)]
    for v in range(256):  # every byte value at the end of a block, after a run of the same value and after random bytes
        blocks.append(np.concatenate([np.full(40, v, np.uint8), np.array([v], np.uint8)]))
        blocks.append(np.concatenate([r.integers(0, 256, 20).astype(np.uint8), np.array([v, v], np.uint8)]))
    check_batch(ctx, oracle, kz, blocks)


def test_silesia_shaped_blocks(ctx, oracle, synth, kz):
    x = synth.silesia_shaped(12 << 20, seed=21)
    check_batch(ctx, oracle, kz, [x[o: o + (4 << 20)] for o in range(0, len(x), 4 << 20)])
