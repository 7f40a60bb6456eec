"""GPU parity tests for TEXT (TextCodec encoding 2, transform/TextCodec.go:1137-1724): statistics / dictionary set-up kernels around the
one-thread-per-block walk of kz_text_core.cuh (whose logic tests/test_text_core_host.py already checks on the CPU)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T_TEXT = 10


def _words(n_bytes, n_distinct, seed, crlf=False):
    r = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8)
    vocab = [bytes(r.choice(alphabet, int(l))) for l in r.integers(3, 12, n_distinct)]
    common = [b"the", b"and", b"that", b"have", b"with", b"people", b"because", b"The", b"And", b"HTTP", b"don't", b"x", b"ab"]
    seps = [b" ", b" ", b" ", b", ", b". ", b"\r\n" if crlf else b"\n", b"; ", b" (", b") ", b"_", b"\t"]
    out = bytearray()
    while len(out) < n_bytes:
        w = vocab[int(r.integers(0, n_distinct))] if r.random() < 0.7 else common[int(r.integers(0, len(common)))]
        if r.random() < 0.1:
            w = w.capitalize()
        out += w + seps[int(r.integers(0, len(seps)))]
        if r.random() < 0.01:
            out += bytes([0x0F, 0xC3, 0xA9]) + b" "
    return np.frombuffer(bytes(out[:n_bytes]), np.uint8)


def cases(synth, n, seed):
    yield "markov", synth.markov_text(n, seed=seed)
    yield "words50", _words(n, 50, seed + 1)
    yield "words5000_crlf", _words(n, 5000, seed + 2, crlf=True)
    yield "xml", np.resize(np.frombuffer(b"<item id=\"1\">the &amp; and &lt;that&gt; have &quot;with&quot;</item>\n", np.uint8), n)
    yield "uniform", synth.uniform_bytes(n, seed=seed + 3)
    yield "dna", np.frombuffer(b"ACGT", np.uint8)[synth.uniform_bytes(n, seed=seed + 4) & 3]
    lead = synth.markov_text(n, seed=seed + 5).copy()
    lead[: min(n, 37)] = 0x20  # leading spaces are copied before the walk starts
    yield "leading_spaces", lead
    png = synth.markov_text(n, seed=seed + 6).copy()
    png[:4] = np.frombuffer(b"\x89PNG", np.uint8)  # any known magic number: "not text" without looking further
    yield "magic", png


@pytest.mark.parametrize("n,bs", [(1000, 1024), (1024, 1024), (5000, 4096), (70000, 1 << 16), (300001, 1 << 20), (1 << 20, 4 << 20)])
def test_text_transform_parity(gpu, oracle, synth, kz, n, bs):
    gpu.set_stream_block_size(bs)
    try:
        for cname, x in cases(synth, n, seed=n):
            want, wdt = oracle.transform_forward(T_TEXT, x, 0, block_size=bs)
            got, gdt = gpu.transform_forward(T_TEXT, x)
            assert gdt == wdt, (cname, n, gdt, wdt)
            if want is None:
                assert got is None, (cname, n)
                continue
            assert got is not None, (cname, n)
            m = min(len(got), len(want))
            assert len(got) == len(want) and np.array_equal(got, want), (cname, n, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
            back = gpu.transform_inverse(T_TEXT, want, n + 4096)
            assert np.array_equal(back, x), (cname, n)
    finally:
        gpu.set_stream_block_size(0)


@pytest.mark.parametrize("dt", [1, 2, 3, 6, 7, 8])
def test_text_respects_incoming_data_type(gpu, oracle, synth, kz, dt):
    x = synth.markov_text(50000, seed=4)
    gpu.set_stream_block_size(1 << 16)
    try:
        want, wdt = oracle.transform_forward(T_TEXT, x, dt, block_size=1 << 16)
        got, gdt = gpu.transform_forward(T_TEXT, x, dt)
        assert (want is None) == (got is None) and gdt == wdt, dt
        if want is not None:
            assert np.array_equal(got, want), dt
    finally:
        gpu.set_stream_block_size(0)


@pytest.mark.parametrize("chain,entropy", [("TEXT", "ANS0"), ("TEXT+PACK+MM+LZX", "HUFFMAN"), ("TEXT+PACK+MM+ROLZ", "NONE"), ("TEXT+BWT+RANK+ZRLT", "ANS0")])
@pytest.mark.parametrize("bs", [4096, 1 << 17])
def test_stream_parity_text_chains(gpu, oracle, synth, kz, chain, entropy, bs):
    """the level chains of kanzi -l 3 / -l 4 / -l 5 minus UTF (and EXE), whole stream: the block size in the header sizes TEXT's hash map"""
    parts = [x for _, x in cases(synth, bs, seed=bs)] + [synth.markov_text(bs // 2 + 7, seed=1)]
    x = np.concatenate(parts)
    n = len(x)
    want = oracle.compress(x, chain, entropy, block_size=bs, jobs=8, input_size=n)
    got = gpu.compress(x, chain, entropy, block_size=bs, input_size=n)
    m = min(len(got), len(want))
    assert len(got) == len(want) and np.array_equal(got, want), (chain, entropy, bs, len(got), len(want), int(np.argmax(got[:m] != want[:m])))
    assert np.array_equal(gpu.decompress(want, n + 64), x), (chain, entropy, bs)


def test_block_batch_uses_stream_block_size(gpu, oracle, synth, kz):
    """kz_encode_blocks / kz_decode_blocks: the short last block of a stream still hashes with the stream's block size"""
    bs = 1 << 16
    blocks = [synth.markov_text(bs, seed=1), _words(bs, 3000, 2), synth.markov_text(5000, seed=3)]
    t48, et = kz.transform_type("TEXT+LZ"), kz.entropy_type("HUFFMAN")
    gpu.set_stream_block_size(bs)
    try:
        enc = gpu.encode_blocks(t48, et, blocks)
    finally:
        gpu.set_stream_block_size(0)
    stream = oracle.compress(np.concatenate(blocks), "TEXT+LZ", "HUFFMAN", block_size=bs, jobs=4, input_size=sum(len(b) for b in blocks))
    dec = gpu.decode_blocks(t48, et, enc, bs)
    for b, d in zip(blocks, dec):
        assert np.array_equal(b, d)
    assert np.array_equal(gpu.decompress(stream, 3 * bs), np.concatenate(blocks))


def test_text_with_encoding1_codecs_is_refused(gpu, kz, synth):
    """The reference picks the TEXT encoding from the entropy codec (transform/Factory.go:99-119): encoding 2 for NONE / ANS0 / HUFFMAN /
    RANGE, encoding 1 for everything else. Only encoding 2 exists on the GPU path, so `TEXT & ANS1` must be refused (ADVICE r1), both ways."""
    x = synth.markov_text(1 << 16, seed=5)
    for entropy in ("ANS1",):
        with pytest.raises(kz.KanziError):
            gpu.compress(x, "TEXT", entropy, block_size=1 << 16, input_size=len(x))
        with pytest.raises(kz.KanziError):
            gpu.encode_blocks(kz.transform_type("TEXT+UTF"), kz.entropy_type(entropy), [x])
    ok = gpu.compress(x, "TEXT", "ANS0", block_size=1 << 16, input_size=len(x))
    assert np.array_equal(gpu.decompress(ok, len(x) + 64), x)
    # a stream whose header says TEXT & ANS1 (written by the reference with encoding 1) is refused as well, not mis-decoded
    bad = gpu.compress(x, "TEXT", "ANS0", block_size=1 << 16, input_size=len(x)).copy()
    # entropy type lives in header bits 38..42 (after 32 b magic, 4 b version, 2 b checksum): ANS0 = 5 -> ANS1 = 8; the header checksum then
    # no longer matches either, so any error is fine as long as nothing is decoded
    bad[4] ^= 0x01
    with pytest.raises(kz.KanziError):
        gpu.decompress(bad, len(x) + 64)
