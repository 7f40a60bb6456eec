"""CPU check of the batched read plan and the index blob (kanzi-go_b200/csrc/kz_read_plan.h) under g++: the plan against a brute-force
Python plan (random requests, duplicates, zero lengths, requests past the end, a request spanning every block, 10^5 requests on a
two-block stream, passes within the budget, one block above the budget alone, slices that tile each request exactly once), and
kz_index_load fuzzed with mutated blobs under ASan / UBSan: it returns an error or a consistent index and never reads outside the blob."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import index_oracle as io_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "read_plan_host.cpp")
HDRS = [os.path.join(ROOT, "kanzi-go_b200", "csrc", h) for h in ("kz_read_plan.h", "kz_stream_plan.h")]
SO = os.path.join(ROOT, "tests", "host", "_build", "libread_plan_host.so")
EXE = os.path.join(ROOT, "tests", "host", "_build", "read_plan_fuzz")
BUDGET = 1 << 30  # STREAM_PASS_BUDGET
u64, u32 = C.c_uint64, C.c_uint32


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(f) for f in [SRC] + HDRS) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    L = C.CDLL(SO)
    L.plan_reads.restype = u32
    L.plan_reads.argtypes = [u64, u32, C.c_int64, u32, C.c_void_p, C.c_void_p, u64]
    L.plan_nblocks.restype = u64
    L.plan_nslices.restype = u64
    L.plan_get.restype = None
    L.plan_get.argtypes = [C.c_void_p] * 5
    L.read_cost.restype = u64
    L.read_cost.argtypes = [u32]
    L.blob_roundtrip.restype = u64
    L.blob_roundtrip.argtypes = [C.c_void_p, u64, C.c_void_p, u64]
    L.xxh64.restype = u64
    L.xxh64.argtypes = [C.c_void_p, u64]
    return L


def check(lib, nblocks, bs, size, reqs, budget=BUDGET):
    """Plans reqs = [(off, len)] and holds the plan against the brute-force one. Returns (passes, blocks)."""
    off = np.array([r[0] for r in reqs] or [0], np.uint64)
    ln = np.array([r[1] for r in reqs] or [0], np.uint64)
    npass = lib.plan_reads(nblocks, bs, size, len(reqs), off.ctypes.data, ln.ctypes.data, budget)
    nk, ns = lib.plan_nblocks(), lib.plan_nslices()
    blocks, first, slice_of = np.zeros(nk + 1, np.uint64), np.zeros(npass + 2, np.uint32), np.zeros(nk + 2, np.uint64)
    want, sl = np.zeros(len(reqs) + 1, np.uint64), np.zeros((ns + 1, 6), np.uint64)
    lib.plan_get(blocks.ctypes.data, first.ctypes.data, slice_of.ctypes.data, want.ctypes.data, sl.ctypes.data)
    blocks, slice_of, want, sl = blocks[:nk], slice_of[: nk + 1], want[: len(reqs)], sl[:ns]
    first = first[: npass + 1] if nk else first[:1]
    total = size if size >= 0 else nblocks * bs
    # the brute-force plan
    exp_want = [min(n, total - o) if o < total else 0 for o, n in reqs]
    assert want.tolist() == exp_want
    exp_blocks = sorted({b for (o, _), w in zip(reqs, exp_want) if w for b in range(o // bs, (o + w - 1) // bs + 1)})
    assert blocks.tolist() == exp_blocks
    # passes: consecutive runs of the sorted blocks, each within the budget unless it is one block
    cost = lib.read_cost(bs)
    per = max(1, budget // cost)
    assert first.tolist() == list(range(0, nk, per)) + [nk] if nk else first.tolist() == [0]
    assert npass == (nk + per - 1) // per
    for p in range(npass):
        k = int(first[p + 1]) - int(first[p])
        assert k >= 1 and (k * cost <= budget or k == 1)
    # slices: grouped by block in slice_of, and they tile every request exactly once
    assert int(slice_of[-1]) == ns and (np.diff(slice_of.astype(np.int64)) >= 1).all() if nk else ns == 0
    if ns:
        req, blk, inb, n, at = (sl[:, c].astype(np.int64) for c in range(5))
        assert (np.diff(blk) >= 0).all()
        assert (np.bincount(blk, minlength=nk) == np.diff(slice_of.astype(np.int64))).all()
        assert (n >= 1).all() and (inb + n <= bs).all()
        o = np.array([r[0] for r in reqs], np.uint64)[req].astype(object)
        # the slice's bytes are where the request says: block * bs + in_block == off + at
        assert all(int(blocks[b]) * bs + int(i) == int(oo) + int(a) for b, i, oo, a in zip(blk, inb, o, at))
        order = np.lexsort((at, req))
        r_, a_, n_ = req[order], at[order], n[order]
        starts = np.r_[True, r_[1:] != r_[:-1]]
        assert (a_[starts] == 0).all()
        assert (a_[1:][~starts[1:]] == (a_ + n_)[:-1][~starts[1:]]).all()
        covered = np.bincount(r_, weights=n_, minlength=len(reqs)).astype(np.int64)
        assert covered.tolist() == exp_want
    else:
        assert sum(exp_want) == 0
    return npass, nk


def test_empty_and_simple(lib):
    assert check(lib, 0, 1024, 0, []) == (0, 0)
    assert check(lib, 0, 1024, 0, [(0, 10), (5, 0)]) == (0, 0)
    assert check(lib, 10, 1024, -1, []) == (0, 0)
    assert check(lib, 10, 1024, -1, [(0, 1)]) == (1, 1)
    assert check(lib, 10, 1024, -1, [(1023, 2)]) == (1, 2)
    assert check(lib, 10, 1024, -1, [(0, 0), (5000, 0)]) == (0, 0)


def test_past_the_end_and_known_size(lib):
    bs, nb = 4096, 7
    size = (nb - 1) * bs + 100
    reqs = [(size - 1, 10), (size, 10), (size + 1, 1), (1 << 63, 1 << 63), ((1 << 64) - 1, (1 << 64) - 1), (0, (1 << 64) - 1), (nb * bs - 1, 5)]
    check(lib, nb, bs, -1, reqs)
    check(lib, nb, bs, size, reqs)
    # with the size known, a request behind the data in the last block touches nothing
    assert check(lib, nb, bs, size, [(size, 50), (size + 10, 1)]) == (0, 0)
    assert check(lib, nb, bs, -1, [(size, 50)]) == (1, 1)


def test_random_requests(lib):
    rng = np.random.default_rng(3)
    for bs, nb in ((1024, 5000), (65536, 300), (4 << 20, 48)):
        total = nb * bs
        reqs = [(int(rng.integers(0, total + bs)), int(rng.integers(0, 3 * bs))) for _ in range(2000)]
        reqs += reqs[:50] + [(0, total), (0, 0), (total, 1)]  # duplicates, one request over every block
        check(lib, nb, bs, -1, reqs)
        check(lib, nb, bs, total - bs + 1, reqs)


def test_many_requests_on_two_blocks(lib):
    rng = np.random.default_rng(4)
    bs = 65536
    reqs = [(int(o), int(n)) for o, n in zip(rng.integers(0, 2 * bs, 100000), rng.integers(0, 4096, 100000))]
    assert check(lib, 2, bs, -1, reqs) == (1, 2)


def test_passes_follow_the_budget(lib):
    bs = 4 << 20
    per = BUDGET // lib.read_cost(bs)
    assert 70 < per < 90  # three slots of a little over 4 MiB per block
    npass, nk = check(lib, 1000, bs, -1, [(0, 1000 * bs)])
    assert nk == 1000 and npass == (1000 + per - 1) // per
    # a small budget: one block above it still runs, alone
    npass, nk = check(lib, 50, bs, -1, [(b * bs + 5, 10) for b in (3, 40, 41)], budget=1 << 20)
    assert (npass, nk) == (3, 3)
    check(lib, 3, 1 << 30, -1, [(0, 3 << 30)])


def model_blob(nb=5, size=-1, headerless=False):
    pos, recs = 0 if headerless else 176, []
    for b in range(nb):
        recs.append((pos + 16, 900 + b))
        pos += 16 + 900 + b
    return {"transform48": 3 << 42, "entropy": 1, "block_size": 2048, "checksum_bits": 32, "input_size": 9000, "header_bits": 0 if headerless else 176,
            "nblocks": nb, "stream_bytes": (pos + 8 + 7) // 8, "size": 0 if nb == 0 else size, "head": bytes(range(32)), "recs": recs}


def roundtrip(lib, blob):
    b = np.frombuffer(bytes(blob), np.uint8).copy()
    out = np.zeros(len(b) + 64, np.uint8)
    n = lib.blob_roundtrip(b.ctypes.data, len(b), out.ctypes.data, out.size)
    return bytes(out[:n]) if n else None


def test_xxh64_and_blob_layout(lib):
    rng = np.random.default_rng(5)
    for n in (0, 1, 3, 4, 7, 8, 31, 32, 33, 100, 1000):
        d = rng.integers(0, 256, n, dtype=np.uint8)
        assert lib.xxh64(d.ctypes.data if n else None, n) == io_.xxh64(d.tobytes())
    assert io_.xxh64(b"") == 0xEF46DB3751D8E999  # the published XXH64 of the empty input, seed 0
    for m in (model_blob(), model_blob(0), model_blob(3, 2 * 2048 + 7), model_blob(4, -1, True)):
        blob = io_.blob(m)
        assert len(blob) == 104 + 16 * m["nblocks"]
        assert roundtrip(lib, blob) == blob


def test_load_rejects_hand_built_blobs(lib):
    good = model_blob(4, 3 * 2048 + 1)
    assert roundtrip(lib, io_.blob(good)) is not None

    def bad(**kw):
        m = dict(good)
        m.update(kw)
        return roundtrip(lib, io_.blob(m)) is None

    recs = good["recs"]
    assert bad(block_size=1023) and bad(block_size=(1 << 30) + 16) and bad(checksum_bits=16) and bad(entropy=32) and bad(transform48=1 << 48)
    assert bad(header_bits=8) and bad(input_size=-1) and bad(input_size=1 << 48)
    assert bad(size=0) and bad(size=3 * 2048) and bad(size=4 * 2048 + 1) and bad(size=-2)
    assert bad(stream_bytes=good["stream_bytes"] - 1)                    # no room for the end marker
    assert bad(recs=[recs[1], recs[0]] + recs[2:])                        # out of order
    assert bad(recs=[(recs[0][0] - 10, recs[0][1])] + recs[1:])           # no room for the prefix
    assert bad(recs=recs[:3] + [(recs[3][0], 1 << 40)])                   # past the end
    assert bad(recs=recs[:3] + [(recs[3][0], 0)])
    assert bad(recs=recs[:3] + [((1 << 64) - 8, 16)])
    blob = io_.blob(good)
    assert roundtrip(lib, blob[:-1]) is None and roundtrip(lib, blob + b"\0") is None and roundtrip(lib, blob[:50]) is None and roundtrip(lib, b"") is None
    for at in (0, 4, 9, 70, 100, len(blob) - 1):
        b = bytearray(blob)
        b[at] ^= 1
        assert roundtrip(lib, b) is None, at
    # a record count that does not match the blob's length, with a good hash
    b = bytearray(blob[:-8])
    b[48:56] = (1 << 60).to_bytes(8, "little")
    assert roundtrip(lib, bytes(b) + io_.xxh64(bytes(b)).to_bytes(8, "little")) is None


def test_blob_load_fuzz_under_sanitizers():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", EXE, SRC],
                       cwd=os.path.dirname(SRC), capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr:
        pytest.skip("sanitizers not available: " + r.stderr[:200])
    assert r.returncode == 0, r.stderr
    r = subprocess.run([EXE, "300"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "fuzz done" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
