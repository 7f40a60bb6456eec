"""Every transform alone, as a one-stage plan, through the transform-sequence path that also runs the level chains: the stream equals
the oracle's and decodes through the whole stream and the block batch entry points, with COPY blocks and a block the stage is likely
to decline in the same batch. A decoded stream that does not fit the output buffer is a write error for one stage and for several."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAMES = ["BWT", "BWTS", "LZ", "LZX", "ROLZ", "RANK", "MTFT", "ZRLT", "PACK", "DNA", "MM", "TEXT", "UTF", "EXE"]


def _utf(n, seed):
    rng = np.random.default_rng(seed)
    words = ["héllo ", "wörld ", "naïve ", "日本語", "テキスト", "данные ", "текст ", "abc ", "\n", "€", "ß"]
    s = "".join(words[int(i)] for i in rng.integers(0, len(words), n)).encode("utf-8")
    return np.frombuffer(s[:n], np.uint8)


def block_for(synth, name, n, seed):
    """a block of the kind the stage is meant for"""
    if name in ("PACK", "DNA"):
        return np.frombuffer(b"ACGT", np.uint8)[synth.uniform_bytes(n, seed=seed) & 3]
    if name == "MM":
        t = np.arange(n)
        return (128 + 100 * np.sin(t / 40.0) + np.random.default_rng(seed).normal(0, 1.5, n)).astype(np.uint8)
    if name == "TEXT":
        return synth.english_text(n, seed=seed)[:n]
    if name == "UTF":
        return _utf(n, seed)
    if name == "EXE":
        return synth.x86_like(n, seed=seed)[:n]
    return synth.markov_text(n, seed=seed)


@pytest.mark.parametrize("name", NAMES)
def test_one_stage_stream(gpu, oracle, synth, kz, name):
    bs = 1 << 16
    # last block: 15 bytes, a COPY block
    x = np.concatenate([block_for(synth, name, bs, 1), synth.uniform_bytes(bs, seed=2), block_for(synth, name, bs, 3), synth.markov_text(15, seed=4)])
    want = oracle.compress(x, name, "ANS0", block_size=bs, jobs=4, input_size=len(x))
    got = gpu.compress(x, name, "ANS0", block_size=bs, input_size=len(x))
    assert len(got) == len(want) and np.array_equal(got, want), (name, len(got), len(want))
    assert np.array_equal(gpu.decompress(want, len(x) + 64), x), name


@pytest.mark.parametrize("name", NAMES)
def test_one_stage_block_batch(gpu, oracle, synth, kz, name):
    lens = [1, 15, 16, 70000, 50000, 200000]
    blocks = [block_for(synth, name, m, 10 + i) for i, m in enumerate(lens)]
    blocks[4] = synth.uniform_bytes(lens[4], seed=14)
    t48 = kz.transform_type(name)
    et = oracle.parse_entropy("ANS0")
    got = gpu.encode_blocks(t48, et, blocks)
    payloads = []
    for i, (b, (g, gbits)) in enumerate(zip(blocks, got)):
        w, wbits = oracle.encode_block(b, t48, et)
        assert gbits == wbits and np.array_equal(g, w), (name, i, lens[i], gbits, wbits)
        payloads.append((w, wbits))
    dec = gpu.decode_blocks(t48, et, payloads, block_size=1 << 18)
    for i, (b, d) in enumerate(zip(blocks, dec)):
        assert np.array_equal(b, d), (name, i, lens[i])


@pytest.mark.parametrize("seq", ["BWT", "LZ", "BWT+RANK+ZRLT"])
def test_output_too_small_is_a_write_error(gpu, synth, kz, seq):
    x = synth.markov_text(5 * 4096 + 100, seed=9)
    stream = gpu.compress(x, seq, "ANS0", block_size=4096, input_size=len(x))
    with pytest.raises(kz.KanziError) as e:
        gpu.decompress(stream, len(x) - 1)
    assert e.value.code == 12, (seq, str(e.value))  # KZ_ERR_WRITE_FILE
