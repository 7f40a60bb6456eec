"""GPU parity of the RANK / MTFT inverse (kz_sbrt.cu) on the adversarial rank streams of tests/sbrt_corpus.py, checked byte for byte against
the oracle's inverse, through every route that reaches its two kernels:
  - sbrt_inverse_multi_kernel (blocks of at most 16 MiB): single blocks, block batches with COPY blocks among them, exactly 16 MiB, more
    than 5 blocks per SM, and whole streams;
  - sbrt_inverse_warp_kernel (every block of a batch whose longest block is over 16 MiB): the corpus beside one block of 2^24 + 2^22 ranks,
    whose positions need the kernel's 64-bit entries.
The forward of the decoded data must give the oracle's payloads back. Two contexts on two host threads decode RANK batches of different
sizes side by side: each launch asks for a different dynamic shared memory size, and none may fail."""
import threading

import numpy as np
import pytest

import sbrt_corpus as sc

pytestmark = pytest.mark.gpu

MODES = ["RANK", "MTFT"]


@pytest.fixture(scope="module")
def corpus(oracle, kz):
    """mode -> [(name, R, D)] with D the oracle's inverse of R"""
    out = {}
    for mode in MODES:
        t = kz.TRANSFORM_IDS[mode]
        out[mode] = [(name, r, sc.expected(t, oracle, r)) for name, r in sc.corpus(t, oracle)]
    return out


def payloads(oracle, kz, mode, datas, ranks):
    """the oracle's E_NONE block payloads of datas; every block of 16 bytes or more carries its rank stream after the head"""
    t48 = kz.transform_type(mode)
    out = [oracle.encode_block(d, t48, oracle.E_NONE) for d in datas]
    for (p, _), r in zip(out, ranks):
        if len(r) >= 16:
            assert np.array_equal(p[len(p) - len(r):], r), (mode, len(r))
    return out


def check_blocks(gpu, oracle, kz, mode, names, ranks, datas):
    """decode_blocks on the oracle's payloads == datas; encode_blocks on datas == the oracle's payloads"""
    t48 = kz.transform_type(mode)
    want = payloads(oracle, kz, mode, datas, ranks)
    got = gpu.decode_blocks(t48, kz.E_NONE, want, max(len(d) for d in datas))
    for name, r, g, d in zip(names, ranks, got, datas):
        assert np.array_equal(g, d), sc.first_difference(name, mode, r, g, d)
    enc = gpu.encode_blocks(t48, kz.E_NONE, datas)
    for name, (g, gbits), (w, wbits) in zip(names, enc, want):
        assert gbits == wbits and np.array_equal(g, w), ("forward", name, mode)


@pytest.mark.parametrize("mode", MODES)
def test_single_blocks(gpu, kz, corpus, mode):
    """every case through kz_transform_inverse, n = 1 .. 16 included (the block paths store those as COPY blocks)"""
    t = kz.TRANSFORM_IDS[mode]
    for name, r, d in corpus[mode]:
        got = gpu.transform_inverse(t, r, len(r) + 64)
        assert np.array_equal(got, d), sc.first_difference(name, mode, r, got, d)


@pytest.mark.parametrize("mode", MODES)
def test_block_batch(gpu, oracle, kz, corpus, mode):
    """every case in one batch of blocks up to 16 MiB: the 4-warp kernel, beside the inactive entries of the COPY blocks"""
    names, ranks, datas = zip(*corpus[mode])
    check_blocks(gpu, oracle, kz, mode, names, ranks, datas)


def composite(cases, rng):
    """the cases of one generator in one block, each starting on a 32-rank round (uniform ranks between them)"""
    parts, pos = [], 0
    for _, r, _ in cases:
        pad = (-pos) % 32 + 32
        parts += [rng.integers(0, 256, pad).astype(np.uint8), r]
        pos += pad + len(r)
    return np.concatenate(parts)


@pytest.mark.parametrize("mode", MODES)
def test_block_batch_with_a_block_above_16mib(gpu, oracle, kz, corpus, mode):
    """one block of 2^24 + 2^22 uniform ranks sends every block of the batch to the warp kernel, positions past 2^24 included. A batch gives
    every block a slot of 1.5 x its longest block, so the corpus goes in one block per generator (every case on a round boundary as in
    its own block), with the blocks of under 16 bytes beside them"""
    t = kz.TRANSFORM_IDS[mode]
    rng = np.random.default_rng(7)
    by_gen = {}
    for case in corpus[mode]:
        by_gen.setdefault(case[0].split("/")[0], []).append(case)
    names, ranks = ["uniform_20mib"], [rng.integers(0, 256, (1 << 24) + (1 << 22)).astype(np.uint8)]
    for gen, cases in by_gen.items():
        names.append(gen + "/composite")
        ranks.append(composite(cases, rng))
    for name, r, _ in [c for c in corpus[mode] if len(c[1]) < 16][::50]:
        names.append(name)
        ranks.append(r)
    datas = [sc.expected(t, oracle, r) for r in ranks]
    check_blocks(gpu, oracle, kz, mode, names, ranks, datas)


@pytest.mark.parametrize("mode", MODES)
def test_exactly_16mib(gpu, oracle, kz, mode):
    """2^24 ranks, the longest block of the 4-warp kernel: the largest positions its 32-bit entries (p << 8 | symbol) hold"""
    t = kz.TRANSFORM_IDS[mode]
    r = np.random.default_rng(16).integers(0, 256, 1 << 24).astype(np.uint8)
    r[-100:] = 0  # the last positions through a zero run too
    d = sc.expected(t, oracle, r)
    got = gpu.transform_inverse(t, r, len(r) + 64)
    assert np.array_equal(got, d), sc.first_difference("uniform_16mib", mode, r, got, d)


@pytest.mark.parametrize("mode", MODES)
def test_many_blocks_per_sm(gpu, oracle, kz, corpus, mode):
    """more than 5 blocks per SM: several chains share an SM and no dynamic shared memory is asked for"""
    import torch

    nb = 6 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    short = [c for c in corpus[mode] if 16 <= len(c[1]) <= 4097]
    cases = [short[k % len(short)] for k in range(nb)]
    names, ranks, datas = zip(*cases)
    check_blocks(gpu, oracle, kz, mode, names, ranks, datas)


@pytest.mark.parametrize("mode", MODES)
def test_stream(gpu, oracle, kz, mode):
    """a stream of 64 KiB blocks whose rank streams are the corpus's, through kz_decompress_stream"""
    t = kz.TRANSFORM_IDS[mode]
    streams = sc.rank_streams(1 << 16, t, oracle, seed=3)
    x = np.concatenate([sc.expected(t, oracle, r) for _, r in streams])
    s = oracle.compress(x, mode, "NONE", block_size=1 << 16, input_size=len(x))
    got = gpu.decompress(s, len(x) + 1024)
    assert len(got) == len(x)
    for k, (name, r) in enumerate(streams):
        g, w = got[k << 16: (k + 1) << 16], x[k << 16: (k + 1) << 16]
        assert np.array_equal(g, w), sc.first_difference(name + "/stream", mode, r, g, w)


def test_contexts_with_different_shared_memory_sizes(kz, oracle):
    """RANK batches of 100 and of 300 short blocks on two contexts and two host threads at once: about 1 and 3 chains per SM, so the two
    launches ask for different dynamic shared memory sizes of the same kernel. Every decode must succeed and be exact."""
    t48 = kz.transform_type("RANK")
    rng = np.random.default_rng(11)
    jobs = []
    for nb in (100, 300):
        ranks = [rng.integers(0, 256, 4096).astype(np.uint8) for _ in range(nb)]
        datas = [sc.expected(kz.TRANSFORM_IDS["RANK"], oracle, r) for r in ranks]
        jobs.append((payloads(oracle, kz, "RANK", datas, ranks), datas))
    ctxs = [kz.Context(0) for _ in jobs]
    errors, bad = [], []
    gate = threading.Barrier(len(jobs))

    def worker(k):
        try:
            pl, datas = jobs[k]
            for it in range(20):
                gate.wait()
                got = ctxs[k].decode_blocks(t48, kz.E_NONE, pl, 4096)
                bad.extend((k, it, b) for b, (g, d) in enumerate(zip(got, datas)) if not np.array_equal(g, d))
        except BaseException as e:  # noqa: B902 - re-raised below
            errors.append((k, e))
            gate.abort()

    th = [threading.Thread(target=worker, args=(k,)) for k in range(len(jobs))]
    for x in th:
        x.start()
    for x in th:
        x.join()
    for c in ctxs:
        c.close()
    assert not errors, errors
    assert not bad, bad[:10]
