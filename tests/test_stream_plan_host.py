"""CPU check of the pass planner of kz_compress_streams / kz_decompress_streams (kanzi-go_b200/csrc/kz_stream_plan.h): every block lands in
exactly one pass and one slot, each pass's stride holds its blocks and is at most twice each member's length plus 16, and the scratch
bound and the pass budget hold, also for adversarial length mixes such as one 1 GiB block among 10^5 one-byte blocks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "stream_plan_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_stream_plan.h")
SO = os.path.join(ROOT, "tests", "host", "_build", "libstream_plan_host.so")
BUDGET = 1 << 30  # STREAM_PASS_BUDGET


@pytest.fixture(scope="module")
def plan():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.plan_compress.restype = C.c_uint32
    lib.plan_compress.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.compress_cost.restype = C.c_uint64
    lib.compress_cost.argtypes = [C.c_uint64]
    lib.plan_decompress.restype = C.c_uint32
    lib.plan_decompress.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.decompress_cost.restype = C.c_uint64
    lib.decompress_cost.argtypes = [C.c_uint32]
    return lib


def check_compress(lib, lens, budget=BUDGET):
    lens = np.ascontiguousarray(lens, np.uint32)
    n = len(lens)
    ps, sl, st = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint64)
    scratch = C.c_uint64(0)
    npass = lib.plan_compress(lens.ctypes.data, n, budget, ps.ctypes.data, sl.ctypes.data, st.ctypes.data, C.byref(scratch))
    ps, sl, st = ps[:n], sl[:n], st[:npass]
    if n == 0:
        assert npass == 0 and scratch.value == 0
        return npass
    # every block in exactly one pass, and the slots of a pass are 0 .. count-1, each taken once
    assert ps.max() < npass
    counts = np.bincount(ps, minlength=npass)
    assert (counts > 0).all()
    for p in range(npass):
        assert sorted(sl[ps == p].tolist()) == list(range(int(counts[p])))
    # each stride holds its blocks and is at most twice each member's length plus 16
    eff = np.maximum(lens.astype(np.uint64), 1)
    assert (st % 16 == 0).all()
    assert (eff <= st[ps]).all()
    assert (st[ps] <= 2 * eff + 16).all()
    # the pass budget holds, except for a pass of one block, and the reported scratch is the largest pass
    cost = np.array([lib.compress_cost(int(s)) for s in st], np.uint64)
    per_pass = counts.astype(np.uint64) * cost
    assert ((per_pass <= budget) | (counts == 1)).all()
    assert scratch.value == int(per_pass.max())
    assert scratch.value <= max(budget, int(lib.compress_cost(int(st.max()))))
    return npass


def test_empty_and_uniform(plan):
    assert check_compress(plan, []) == 0
    assert check_compress(plan, [1]) == 1
    assert check_compress(plan, [65536] * 300) == 1


def test_mixed_lengths(plan):
    rng = np.random.default_rng(1)
    lens = np.exp(rng.normal(np.log(16384), 1.5, 20000)).clip(1, 4 << 20).astype(np.uint32)
    npass = check_compress(plan, lens)
    assert npass < 40


def test_one_huge_block_among_tiny_ones(plan):
    """one 1 GiB block among 10^5 one-byte and fifteen-byte blocks: the huge block runs alone, the tiny ones share small strides"""
    lens = np.ones(100001, np.uint32)
    lens[::2] = 15
    lens[50000] = 1 << 30
    check_compress(plan, lens)
    ps, sl, st = np.zeros(len(lens), np.uint32), np.zeros(len(lens), np.uint32), np.zeros(len(lens), np.uint64)
    scratch = C.c_uint64(0)
    npass = plan.plan_compress(lens.ctypes.data, len(lens), BUDGET, ps.ctypes.data, sl.ctypes.data, st.ctypes.data, C.byref(scratch))
    assert (ps == ps[50000]).sum() == 1
    assert st[:npass][np.arange(npass) != ps[50000]].max() == 16


def test_small_budget_and_geometric_lengths(plan):
    lens = np.array([1 << k for k in range(31)] * 3, np.uint32)
    check_compress(plan, lens)
    check_compress(plan, lens, budget=1 << 20)
    rng = np.random.default_rng(2)
    check_compress(plan, rng.integers(0, 1 << 22, 5000).astype(np.uint32), budget=64 << 20)


@pytest.mark.parametrize("n,bs", [(0, 1024), (1, 1 << 30), (100000, 1024), (5000, 4 << 20), (300, 32 << 20), (7, 1 << 30)])
def test_decompress_passes(plan, n, bs):
    ps, sl = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    scratch = C.c_uint64(0)
    npass = plan.plan_decompress(n, bs, BUDGET, ps.ctypes.data, sl.ctypes.data, C.byref(scratch))
    ps, sl = ps[:n], sl[:n]
    cost = plan.decompress_cost(bs)
    per = max(1, BUDGET // cost)
    assert npass == (n + per - 1) // per
    if n:
        assert (np.diff(ps.astype(np.int64)) >= 0).all()  # blocks keep their order
        counts = np.bincount(ps, minlength=npass)
        assert (counts <= per).all() and counts.sum() == n
        for p in range(npass):
            assert sl[ps == p].tolist() == list(range(int(counts[p])))
        assert scratch.value == int(counts.max()) * cost
        assert scratch.value <= max(BUDGET, cost)
