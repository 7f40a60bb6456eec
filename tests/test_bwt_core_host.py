"""CPU check of the small-group sort of the BWT forward rounds (kanzi-go_b200/csrc/kz_bwt_core.cuh, the code bwtn_small_kernel runs for every
member of a group of at most BWT_SMALL_GROUP suffixes): for random groups, the place, the new group offset and the new group size of every
member equal those of std::stable_sort by the second key."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "bwt_core_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_bwt_core.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "libbwt_core_host.so")


@pytest.fixture(scope="module")
def core():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.bwt_group_check.restype = C.c_uint32
    lib.bwt_group_check.argtypes = [C.c_void_p, C.c_uint32]
    lib.bwt_group_sort.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.bwt_bits.restype = C.c_uint32
    lib.bwt_bits.argtypes = [C.c_uint64]
    lib.bwt_small_group.restype = C.c_uint32
    return lib


def check(core, key):
    key = np.ascontiguousarray(key, np.uint32)
    return core.bwt_group_check(key.ctypes.data, len(key))


def test_random_groups_match_stable_sort(core):
    r = np.random.default_rng(7)
    g = core.bwt_small_group()
    sizes = [2, 3, 4, 7, 8, 9, 31, 32, 33, 64, 65, 127, g - 1, g]
    for size in sizes:
        for spread in (1, 2, 3, 16, 1 << 23):  # few distinct keys (ties) ... all distinct
            for _ in range(8):
                key = r.integers(0, spread, size)
                assert check(core, key) == 0, (size, spread, key.tolist())


def test_edge_keys(core):
    g = core.bwt_small_group()
    assert check(core, np.zeros(g, np.uint32)) == 0  # every member past the end of its block: one group stays
    assert check(core, np.arange(g, 0, -1)) == 0  # descending
    assert check(core, np.array([(1 << 23) - 1, 0, (1 << 23) - 1, 0])) == 0
    key = np.array([5, 0, 5, 3], np.uint32)
    order, lt, eq = (np.zeros(4, np.uint32) for _ in range(3))
    core.bwt_group_sort(key.ctypes.data, 4, order.ctypes.data, lt.ctypes.data, eq.ctypes.data)
    assert order.tolist() == [1, 3, 0, 2] and lt.tolist() == [2, 0, 2, 1] and eq.tolist() == [2, 1, 2, 1]


def test_key_widths(core):
    assert [core.bwt_bits(v) for v in (0, 1, 2, 3, 4, (1 << 22) - 1, 1 << 22, (1 << 32) - 1)] == [0, 1, 2, 2, 3, 22, 23, 32]
