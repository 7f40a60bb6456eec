"""GPU parity tests for PACK / DNA (AliasCodec, transform/AliasCodec.go:74-434), for LZ / LZX as stages of a sequence ("DNA+LZ" is
the transform chain of kanzi -l 2) and for the data type a block's magic number sets before the transforms run
(io/CompressedStream.go:806-816)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T_PACK, T_DNA, T_MM = 18, 19, 15


def _dna(synth, n, seed, noise=0.0):
    x = np.frombuffer(b"ACGT", np.uint8)[synth.uniform_bytes(n, seed=seed) & 3].copy()
    if noise:
        r = np.random.default_rng(seed)
        k = int(n * noise)
        x[r.integers(0, n, k)] = r.integers(0, 256, k).astype(np.uint8)
    return x


def cases(synth, n, seed):
    yield "dna4", _dna(synth, n, seed)
    yield "dna_noisy", _dna(synth, n, seed + 1, 0.02)  # still DT_DNA, but too many symbols to bit pack: digram aliases
    yield "hex16", np.frombuffer(b"0123456789abcdef", np.uint8)[synth.uniform_bytes(n, seed=seed + 2) & 15]
    yield "two", np.frombuffer(b"xy", np.uint8)[synth.uniform_bytes(n, seed=seed + 3) & 1]
    yield "three", np.frombuffer(b"xyz", np.uint8)[synth.uniform_bytes(n, seed=seed + 4) % 3]
    yield "one", np.full(n, 0x41, np.uint8)
    yield "text", synth.markov_text(n, seed=seed + 5)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 6)
    yield "zipf", synth.zipf_bytes(n, 1.5, seed=seed + 7)
    yield "periodic", np.resize(np.frombuffer(b"abracadabra, ", np.uint8), n)
    yield "few_digrams", np.resize(np.frombuffer(b"ab" * 7 + b"cd", np.uint8), n)


@pytest.mark.parametrize("ttype", [T_PACK, T_DNA])
@pytest.mark.parametrize("n", [100, 1023, 1024, 1025, 1026, 1027, 4096, 4097, 20000, 65537, 300001, 1 << 20])
def test_alias_transform_parity(gpu, oracle, synth, kz, ttype, n):
    for cname, x in cases(synth, n, seed=n):
        want, wdt = oracle.transform_forward(ttype, x)
        got, gdt = gpu.transform_forward(ttype, x)
        assert gdt == wdt, (cname, n, gdt, wdt)
        if want is None:
            assert got is None, (cname, n)
            continue
        assert got is not None, (cname, n)
        m = min(len(got), len(want))
        assert len(got) == len(want) and np.array_equal(got, want), (cname, n, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
        back = gpu.transform_inverse(ttype, want, n + 64)
        assert np.array_equal(back, x), (cname, n)


@pytest.mark.parametrize("dt", [1, 2, 3, 6, 7, 8, 9])
def test_alias_respects_incoming_data_type(gpu, oracle, synth, kz, dt):
    for ttype in (T_PACK, T_DNA):
        for cname, x in (("dna4", _dna(synth, 50000, 1)), ("text", synth.markov_text(50000, seed=2))):
            want, wdt = oracle.transform_forward(ttype, x, dt)
            got, gdt = gpu.transform_forward(ttype, x, dt)
            assert (want is None) == (got is None) and gdt == wdt, (cname, dt, ttype)
            if want is not None:
                assert np.array_equal(got, want), (cname, dt, ttype)


def _mixed(synth, bs, seed):
    """blocks of different kinds: DNA, text, random, small alphabet, short tail"""
    parts = [_dna(synth, bs, seed), synth.markov_text(bs, seed=seed + 1), synth.uniform_bytes(bs, seed=seed + 2),
             np.frombuffer(b"0123456789abcdef", np.uint8)[synth.uniform_bytes(bs, seed=seed + 3) & 15], _dna(synth, bs, seed + 4, 0.02),
             synth.markov_text(bs // 3 + 5, seed=seed + 5)]
    return np.concatenate(parts)


@pytest.mark.parametrize("chain,entropy", [("DNA+LZ", "HUFFMAN"), ("PACK+LZX", "HUFFMAN"), ("PACK+ROLZ", "NONE"), ("PACK", "ANS0"), ("DNA+LZ", "NONE"),
                                           ("PACK+BWT+RANK+ZRLT", "ANS0")])
@pytest.mark.parametrize("bs", [4096, 65536, 1 << 18])
def test_stream_parity_pack_chains(gpu, oracle, synth, kz, chain, entropy, bs):
    x = _mixed(synth, bs, seed=bs)
    n = len(x)
    want = oracle.compress(x, chain, entropy, block_size=bs, jobs=8, input_size=n)
    got = gpu.compress(x, chain, entropy, block_size=bs, input_size=n)
    m = min(len(got), len(want))
    assert len(got) == len(want) and np.array_equal(got, want), (chain, entropy, bs, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
    assert np.array_equal(gpu.decompress(want, n + 64), x), (chain, entropy, bs)


MAGICS = [b"\x7fELF", b"MZ\x90\x00", b"\x89PNG", b"PK\x03\x04", b"BM\x36\x00", b"RIFF", b"\x1f\x8b\x08\x00", b"%PDF", b"\xff\xd8\xff\xe0", b"\xff\xd8\xff\xe1",
          b"P5\n2", b"P5x2", b"BZh9", b"ID3\x03", b"\xfe\xed\xfa\xce"]


@pytest.mark.parametrize("chain,entropy", [("ROLZ", "NONE"), ("PACK+LZ", "HUFFMAN"), ("LZX", "HUFFMAN")])
def test_block_magic_sets_data_type(gpu, oracle, synth, kz, chain, entropy):
    """every block starts with a magic number: the data type it implies (BIN / MULTIMEDIA / EXE) must reach ROLZ / PACK as in the reference"""
    bs = 1 << 16
    for body_kind in ("text", "dna"):
        blocks = []
        for i, mg in enumerate(MAGICS):
            body = synth.markov_text(bs, seed=i) if body_kind == "text" else _dna(synth, bs, i)
            body = body.copy()
            body[: len(mg)] = np.frombuffer(mg, np.uint8)
            blocks.append(body)
        x = np.concatenate(blocks)
        n = len(x)
        want = oracle.compress(x, chain, entropy, block_size=bs, jobs=8, input_size=n)
        got = gpu.compress(x, chain, entropy, block_size=bs, input_size=n)
        assert len(got) == len(want) and np.array_equal(got, want), (chain, body_kind, len(got), len(want))
        assert np.array_equal(gpu.decompress(want, n + 64), x), (chain, body_kind)
        # the batched block entry point takes the same decision from the host copy of the blocks
        t48, et = kz.transform_type(chain), kz.entropy_type(entropy)
        enc = gpu.encode_blocks(t48, et, blocks)
        for i, b in enumerate(blocks):
            wp, wbits = oracle.encode_block(b, t48, et)
            assert enc[i][1] == wbits and np.array_equal(enc[i][0], wp), (chain, body_kind, i)


# ---------------------------------------------------------------- MM (FSDCodec)
def mm_cases(synth, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    yield "wave8", (128 + 100 * np.sin(t / 40.0) + rng.normal(0, 1.5, n)).astype(np.uint8)  # smooth: delta coding, distance 1
    st = np.empty(n, np.uint8)  # 16-bit little endian samples: distance 2
    v = (np.cumsum(rng.integers(-300, 301, n // 2 + 1)) & 0xFFFF).astype(np.uint16)
    st[0::2] = (v & 0xFF)[: (n + 1) // 2]
    st[1::2] = (v >> 8)[: n // 2]
    yield "pcm16", st
    rgb = np.empty(n, np.uint8)  # three interleaved slowly varying channels: distance 3
    for c in range(3):
        ch = (128 + 90 * np.sin(t[: (n + 2 - c) // 3] / (30.0 + 7 * c)) + rng.normal(0, 1.0, (n + 2 - c) // 3)).astype(np.uint8)
        rgb[c::3] = ch[: len(rgb[c::3])]
    yield "rgb", rgb
    rgba = np.repeat((128 + 60 * np.sin(t[: n // 4 + 1] / 25.0)).astype(np.uint8), 4)[:n].copy()
    rgba[3::4] = 255
    yield "rgba", rgba
    jumps = (t * 37 % 256).astype(np.uint8)  # wrap-around steps: large deltas -> xor coding or escapes
    yield "saw", jumps
    noisy = (128 + 100 * np.sin(t / 40.0)).astype(np.uint8)
    k = rng.integers(0, n, max(1, n // 50))
    noisy[k] = rng.integers(0, 256, len(k)).astype(np.uint8)  # 2 % outliers: escapes inside delta coding
    yield "wave_outliers", noisy
    yield "text", synth.markov_text(n, seed=seed + 1)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 2)
    yield "const", np.full(n, 9, np.uint8)


@pytest.mark.parametrize("n", [500, 1023, 1024, 1030, 4096, 10007, 65536, 300001, 1 << 20])
def test_mm_transform_parity(gpu, oracle, synth, kz, n):
    for cname, x in mm_cases(synth, n, seed=n):
        want, wdt = oracle.transform_forward(T_MM, x)
        got, gdt = gpu.transform_forward(T_MM, x)
        assert gdt == wdt, (cname, n, gdt, wdt)
        if want is None:
            assert got is None, (cname, n)
            continue
        assert got is not None, (cname, n)
        m = min(len(got), len(want))
        assert len(got) == len(want) and np.array_equal(got, want), (cname, n, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
        back = gpu.transform_inverse(T_MM, want, n)
        assert np.array_equal(back, x), (cname, n)


@pytest.mark.parametrize("dt", [1, 2, 3, 6, 7, 8])
def test_mm_respects_incoming_data_type(gpu, oracle, synth, kz, dt):
    for cname, x in mm_cases(synth, 50000, seed=3):
        want, wdt = oracle.transform_forward(T_MM, x, dt)
        got, gdt = gpu.transform_forward(T_MM, x, dt)
        assert (want is None) == (got is None) and gdt == wdt, (cname, dt)
        if want is not None:
            assert np.array_equal(got, want), (cname, dt)


@pytest.mark.parametrize("chain,entropy", [("MM", "ANS0"), ("PACK+MM+LZX", "HUFFMAN"), ("PACK+MM+ROLZ", "NONE"), ("MM+LZ", "NONE")])
@pytest.mark.parametrize("bs", [4096, 1 << 17])
def test_stream_parity_mm_chains(gpu, oracle, synth, kz, chain, entropy, bs):
    parts = [x for _, x in mm_cases(synth, bs, seed=bs)]
    bmp = parts[0].copy()
    bmp[:2] = np.frombuffer(b"BM", np.uint8)  # a BMP magic keeps MM in play (data type MULTIMEDIA); a PNG one rules it out
    png = parts[0].copy()
    png[:4] = np.frombuffer(b"\x89PNG", np.uint8)
    x = np.concatenate(parts + [bmp, png, parts[1][: bs // 2 + 3]])
    n = len(x)
    want = oracle.compress(x, chain, entropy, block_size=bs, jobs=8, input_size=n)
    got = gpu.compress(x, chain, entropy, block_size=bs, input_size=n)
    m = min(len(got), len(want))
    assert len(got) == len(want) and np.array_equal(got, want), (chain, entropy, bs, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
    assert np.array_equal(gpu.decompress(want, n + 64), x), (chain, entropy, bs)
