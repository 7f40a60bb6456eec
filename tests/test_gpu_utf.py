"""GPU parity tests for UTF (UTFCodec, transform/UTFCodec.go:87-383) and for the complete transform chains of kanzi -l 3 and -l 5
(TEXT+UTF+PACK+MM+LZX & HUFFMAN, TEXT+UTF+BWT+RANK+ZRLT & ANS0), which need every stage on the GPU. The per-block logic of UTF is
kz_utf_core.cuh, already checked against the oracle on the CPU by tests/test_utf_core_host.py."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T_UTF = 17


def utf_text(n_bytes, seed, n_symbols=0):
    r = np.random.default_rng(seed)
    words = ["héllo", "wörld", "naïve", "日本語", "テキスト", "данные", "текст", "abc", "xyz", " ", "\n", "😀", "€", "ß"]
    if n_symbols:
        cps = [chr(c) for c in r.choice(np.arange(0x400, 0x3000), n_symbols, replace=False)]
        words = words + ["".join(r.choice(cps, 3)) for _ in range(400)]
    out, size = [], 0
    while size < n_bytes + 8:
        w = words[int(r.integers(0, len(words)))]
        out.append(w)
        size += len(w.encode("utf-8"))
    return np.frombuffer("".join(out).encode("utf-8")[:n_bytes], np.uint8)


def cases(synth, n, seed):
    yield "utf", utf_text(n, seed)
    yield "utf_many_symbols", utf_text(n, seed + 1, n_symbols=min(2000, max(1, n // 20)))
    yield "bom", np.concatenate([np.frombuffer(b"x\xef\xbb\xbf", np.uint8), utf_text(n - 4, seed + 2)])
    yield "mid_sequence_start", utf_text(n + 1, seed + 3)[1:]
    yield "ascii", synth.markov_text(n, seed=seed + 4)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 5)
    bad = utf_text(n, seed + 6).copy()
    bad[n // 2] = 0xC0
    yield "forbidden_byte", bad
    bad2 = utf_text(n, seed + 7).copy()
    bad2[n - 6] = 0xF8
    yield "forbidden_byte_in_last_window", bad2


@pytest.mark.parametrize("n", [1000, 1024, 1027, 4096, 50001, 300000, 1 << 20])
def test_utf_transform_parity(gpu, oracle, synth, kz, n):
    for cname, x in cases(synth, n, seed=n):
        for dt in (0, 8):
            want, wdt = oracle.transform_forward(T_UTF, x, dt)
            got, gdt = gpu.transform_forward(T_UTF, x, dt)
            assert gdt == wdt, (cname, n, dt, gdt, wdt)
            if want is None:
                assert got is None, (cname, n, dt)
                continue
            assert got is not None, (cname, n, dt)
            m = min(len(got), len(want))
            assert len(got) == len(want) and np.array_equal(got, want), (cname, n, dt, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
            back = gpu.transform_inverse(T_UTF, want, n + 64)
            wback = oracle.transform_inverse(T_UTF, want, n + 64)
            wback = wback[0] if isinstance(wback, tuple) else wback
            assert np.array_equal(back, wback), (cname, n, dt)
            if dt == 0:  # validated input round-trips; with the data type forced to UTF-8 the reference itself accepts malformed sequences
                assert np.array_equal(back, x), (cname, n, dt)


@pytest.mark.parametrize("dt", [1, 2, 3, 6, 7])
def test_utf_declines_other_data_types(gpu, oracle, synth, kz, dt):
    x = utf_text(50000, 3)
    want, wdt = oracle.transform_forward(T_UTF, x, dt)
    got, gdt = gpu.transform_forward(T_UTF, x, dt)
    assert want is None and got is None and gdt == wdt


def _mixed(synth, bs, seed):
    t = np.arange(bs)
    r = np.random.default_rng(seed)
    wave = (128 + 100 * np.sin(t / 40.0) + r.normal(0, 1.5, bs)).astype(np.uint8)
    dna = np.frombuffer(b"ACGT", np.uint8)[synth.uniform_bytes(bs, seed=seed + 1) & 3]
    parts = [synth.markov_text(bs, seed=seed), utf_text(bs, seed + 2), wave, dna, synth.uniform_bytes(bs, seed=seed + 3),
             utf_text(bs, seed + 4, n_symbols=500), synth.markov_text(bs // 2 + 11, seed=seed + 5)]
    return np.concatenate(parts)


@pytest.mark.parametrize("chain,entropy", [("UTF", "ANS0"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0"),
                                           ("TEXT+UTF+PACK+MM+ROLZ", "NONE")])
@pytest.mark.parametrize("bs", [4096, 1 << 17])
def test_stream_parity_level_chains(gpu, oracle, synth, kz, chain, entropy, bs):
    """-l 3 and -l 5 end to end (five transforms: the block header carries the skip flags in a byte of its own), -l 4 minus EXE"""
    x = _mixed(synth, bs, seed=bs)
    n = len(x)
    want = oracle.compress(x, chain, entropy, block_size=bs, jobs=8, input_size=n)
    got = gpu.compress(x, chain, entropy, block_size=bs, input_size=n)
    m = min(len(got), len(want))
    assert len(got) == len(want) and np.array_equal(got, want), (chain, entropy, bs, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
    assert np.array_equal(gpu.decompress(want, n + 64), x), (chain, entropy, bs)
