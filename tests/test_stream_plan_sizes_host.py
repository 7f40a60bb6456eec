"""CPU check of the per-stream block sizes of the many-stream entry points (kanzi-go_b200/csrc/kz_stream_plan.h): streams cut with a block
size each, and the decompression pass plan of a group whose streams differ in block size. Every block lands in exactly one pass and slot,
the blocks of a stream keep their order, each pass's stride holds its blocks and is at most twice each member's slot plus 16, the pass
budget holds (a block over it runs alone), no pass holds more blocks than a grid has rows (65,535), a mix of 1 KiB and 1 GiB streams does
not give the small blocks 1 GiB slots, and one block size for every block gives the uniform plan."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "stream_plan_sizes_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_stream_plan.h")
SO = os.path.join(ROOT, "tests", "host", "_build", "libstream_plan_sizes_host.so")
BUDGET = 1 << 30  # STREAM_PASS_BUDGET
GIB = 1 << 30


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    L = C.CDLL(SO)
    L.cut_blocks_sizes.restype = C.c_uint32
    L.cut_blocks_sizes.argtypes = [C.c_void_p] * 2 + [C.c_uint32] + [C.c_void_p] * 4
    for f in (L.plan_decompress_sizes, L.plan_decompress_uniform):
        f.restype = C.c_uint32
    L.plan_decompress_sizes.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64] + [C.c_void_p] * 5 + [C.POINTER(C.c_uint64)]
    L.plan_decompress_uniform.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64] + [C.c_void_p] * 5 + [C.POINTER(C.c_uint64)]
    L.decompress_slot.restype = C.c_uint64
    L.decompress_slot.argtypes = [C.c_uint32]
    L.decompress_cost.restype = C.c_uint64
    L.decompress_cost.argtypes = [C.c_uint32]
    return L


def cut(lib, lens, sizes):
    lens = np.ascontiguousarray(lens, np.uint64)
    sizes = np.ascontiguousarray(sizes, np.uint32)
    ns = len(lens)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64) if ns else np.zeros(0, np.uint64)
    room = int(sum(-(-int(n) // int(b)) for n, b in zip(lens, sizes))) + 1
    oo, ol, of = np.zeros(room, np.uint64), np.zeros(room, np.uint32), np.zeros(ns + 1, np.uint32)
    nb = lib.cut_blocks_sizes(offs.ctypes.data, lens.ctypes.data, ns, sizes.ctypes.data, oo.ctypes.data, ol.ctypes.data, of.ctypes.data)
    return offs, oo[:nb], ol[:nb], of


def test_cut_blocks_per_stream_sizes(lib):
    rng = np.random.default_rng(5)
    lens = [0, 1, 1023, 1024, 1025, 4096, 5000, 65536 * 3 + 17, 1 << 20, 7, 0, 3 * 1040]
    sizes = [1024, 1024, 1024, 1024, 1024, 4096, 1040, 65536, 1 << 18, 16384, 2048, 1040]
    for _ in range(40):
        lens.append(int(rng.integers(0, 1 << 21)))
        sizes.append(int(rng.integers(64, 1 << 16)) * 16)
    offs, oo, ol, of = cut(lib, lens, sizes)
    assert of[0] == 0 and of[-1] == len(ol)
    for s, (n, bs) in enumerate(zip(lens, sizes)):
        blocks = list(range(of[s], of[s + 1]))
        assert len(blocks) == -(-n // bs)  # an empty stream has no blocks
        for j, b in enumerate(blocks):
            assert oo[b] == offs[s] + j * bs
            assert ol[b] == min(bs, n - j * bs)
        assert sum(int(ol[b]) for b in blocks) == n


def plan(lib, sizes, budget=BUDGET, uniform=None):
    sizes = np.ascontiguousarray(sizes, np.uint32)
    n = len(sizes)
    order, first, stride = np.zeros(max(n, 1), np.uint32), np.zeros(n + 1, np.uint32), np.zeros(max(n, 1), np.uint64)
    ps, sl = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    scratch = C.c_uint64(0)
    if uniform is None:
        np_ = lib.plan_decompress_sizes(sizes.ctypes.data, n, budget, order.ctypes.data, first.ctypes.data, stride.ctypes.data, ps.ctypes.data,
                                        sl.ctypes.data, C.byref(scratch))
    else:
        np_ = lib.plan_decompress_uniform(n, uniform, budget, order.ctypes.data, first.ctypes.data, stride.ctypes.data, ps.ctypes.data,
                                          sl.ctypes.data, C.byref(scratch))
    return dict(n=np_, order=order[:n], first=first[:np_ + 1], stride=stride[:np_], pass_=ps[:n], slot=sl[:n], scratch=scratch.value)


def check(lib, sizes, budget=BUDGET, owner=None):
    """The invariants of a plan over blocks of sizes[b]; owner[b]: the stream of block b (blocks of a stream are listed in order)."""
    P = plan(lib, sizes, budget)
    n = len(sizes)
    if n == 0:
        assert P["n"] == 0 and P["scratch"] == 0
        return P
    assert sorted(P["order"].tolist()) == list(range(n))
    assert P["first"][0] == 0 and P["first"][-1] == n
    slot = np.array([lib.decompress_slot(int(b)) for b in sizes], np.uint64)
    cost = np.array([lib.decompress_cost(int(b)) for b in sizes], np.uint64)
    worst = 0
    for p in range(P["n"]):
        members = P["order"][P["first"][p]:P["first"][p + 1]]
        assert 0 < len(members) <= MAX_PASS_BLOCKS
        assert (P["pass_"][members] == p).all()
        assert sorted(P["slot"][members].tolist()) == list(range(len(members)))
        s = int(P["stride"][p])
        assert s == int(slot[members].max())  # the stride holds every member
        assert (s <= 2 * slot[members] + 16).all()  # and no member gets a slot more than twice its own
        pass_cost = len(members) * int(cost[members].max())
        assert pass_cost <= budget or len(members) == 1
        worst = max(worst, pass_cost)
    assert P["scratch"] == worst
    if owner is not None:  # a stream's blocks are decoded in order: pass by pass, and in order inside a pass
        pos = np.empty(n, np.int64)
        pos[P["order"]] = np.arange(n)
        for s in set(owner):
            idx = [b for b in range(n) if owner[b] == s]
            assert all(pos[a] < pos[b] for a, b in zip(idx, idx[1:]))
    return P


MAX_PASS_BLOCKS = 65535  # the grid rows of a stage launch with one row per block


def test_uniform_sizes_give_the_uniform_plan(lib):
    for bs, n, budget in [(1024, 0, BUDGET), (1024, 1, BUDGET), (4 << 20, 1000, BUDGET), (1 << 30, 3, BUDGET), (65536, 5000, 1 << 26),
                          (1 << 20, 77, 5 << 20), (1024, MAX_PASS_BLOCKS, BUDGET)]:
        got = plan(lib, [bs] * n, budget)
        want = plan(lib, [bs] * n, budget, uniform=bs)
        assert got["n"] == want["n"] and got["scratch"] == want["scratch"]
        for k in ("order", "first", "stride", "pass_", "slot"):
            assert np.array_equal(got[k], want[k]), (bs, n, k)
        assert np.array_equal(got["order"], np.arange(n))


def test_budget_holds_on_random_mixes(lib):
    rng = np.random.default_rng(11)
    for trial in range(30):
        ns = int(rng.integers(1, 60))
        stream_bs = [int(rng.integers(64, 1 << 16)) * 16 if rng.random() < 0.8 else int(rng.integers(1 << 16, 1 << 26)) * 16 for _ in range(ns)]
        sizes, owner = [], []
        for s, bs in enumerate(stream_bs):
            k = int(rng.integers(0, 9))
            sizes += [bs] * k
            owner += [s] * k
        budget = int(rng.choice([BUDGET, 1 << 24, 1 << 22]))
        check(lib, sizes, budget, owner)


def test_oversize_block_runs_alone(lib):
    # a 1 GiB block costs more than the budget: it gets a pass of its own, and the small blocks are not put beside it
    sizes = [1024] * 10 + [GIB] + [1024] * 10
    P = check(lib, sizes, owner=list(range(10)) + [10] + list(range(11, 21)))
    big = [p for p in range(P["n"]) if 10 in P["order"][P["first"][p]:P["first"][p + 1]].tolist()]
    assert len(big) == 1
    members = P["order"][P["first"][big[0]]:P["first"][big[0] + 1]]
    assert members.tolist() == [10]
    assert P["scratch"] == lib.decompress_cost(GIB)


def test_small_and_huge_streams_do_not_share_slots(lib):
    # 1 KiB streams and 1 GiB streams in one group: every small block's stride stays its own slot size
    sizes = [1024, GIB, 1024, 1024, GIB, 1024] * 50
    owner = list(range(len(sizes)))
    P = check(lib, sizes, owner=owner)
    small = lib.decompress_slot(1024)
    for b, bs in enumerate(sizes):
        s = int(P["stride"][P["pass_"][b]])
        assert s == (small if bs == 1024 else lib.decompress_slot(GIB))
    # every 1 KiB block fits in one pass: the 1 GiB ones each take a pass of their own
    assert P["n"] == 1 + sizes.count(GIB)


def test_auto_block_sizes_share_passes(lib):
    # kanzi's `-b auto` over files of nearby sizes: block sizes differ by small steps, and blocks within a factor of two share a pass
    sizes = [max(1024, ((n // 16) + 63) & ~63) for n in range(16 << 10, 48 << 10, 64)]
    P = check(lib, sizes)
    assert P["n"] <= 2


def test_pass_holds_at_most_one_grid_of_rows(lib):
    # 1 KiB blocks fit the budget 335,000 at a time, but a pass holds at most MAX_PASS_BLOCKS of them; blocks keep their order
    n = 2 * MAX_PASS_BLOCKS + 10
    P = check(lib, [1024] * n)
    assert P["n"] == 3 and np.array_equal(P["order"], np.arange(n))
    assert [int(P["first"][p + 1] - P["first"][p]) for p in range(3)] == [MAX_PASS_BLOCKS, MAX_PASS_BLOCKS, 10]
    sizes = [1024] * 70000 + [1040] * 70000
    P = check(lib, sizes)
    assert max(int(P["first"][p + 1] - P["first"][p]) for p in range(P["n"])) <= MAX_PASS_BLOCKS
