"""CPU checks of the block range selection that every stream-level decode uses (block_range_records / block_range_slice,
kanzi-go_b200/csrc/kz_common.cuh): the streaming reader numbers the records it walks across batches and decodes exactly the records whose
1-based id the reference keeps, `!(from >= 0 && id < from) && !(to >= 0 && id >= to)` (io/CompressedStream.go:1858-1871), whatever the
batch sizes."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "block_range_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_common.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "libblock_range_host.so")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
NO_END = (1 << 64) - 1


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", CUDA_INC, "-o", SO, SRC])
    L = C.CDLL(SO)
    L.records.argtypes = [C.c_int64, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.records.restype = None
    L.slice.argtypes = [C.c_int64, C.c_int64, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.slice.restype = None
    return L


def kept(block_id, frm, to):
    """the reference's rule for the 1-based block id"""
    return not (frm >= 0 and block_id < frm) and not (to >= 0 and block_id >= to)


def records(lib, frm, to):
    lo, hi = C.c_uint64(0), C.c_uint64(0)
    lib.records(frm, to, C.byref(lo), C.byref(hi))
    return lo.value, hi.value


def session_selection(lib, nrec, batches, frm, to):
    """the record indices a reader session decodes when its walk finds the records in batches of the given sizes"""
    got, first = [], 0
    for size in itertools.cycle(batches):
        if first >= nrec:
            break
        count = min(size, nrec - first)
        lo, hi = C.c_uint32(0), C.c_uint32(0)
        lib.slice(frm, to, first, count, C.byref(lo), C.byref(hi))
        assert 0 <= lo.value <= hi.value <= count
        got += [first + i for i in range(lo.value, hi.value)]
        first += count
    return got


BOUNDS = [-5, -1, 0, 1, 2, 3, 7, 11, 12, 13, 14, 40]


def test_records_follow_the_reference_rule(lib):
    for frm, to in itertools.product(BOUNDS, BOUNDS):
        lo, hi = records(lib, frm, to)
        assert lo <= hi
        for idx in range(50):
            assert (lo <= idx < hi) == kept(idx + 1, frm, to), (frm, to, idx)
    assert records(lib, -1, -1) == (0, NO_END)
    assert records(lib, 0, -1) == records(lib, 1, -1) == (0, NO_END)
    assert records(lib, 5, 1) == (4, 4)
    assert records(lib, -1, 1) == (0, 0)
    assert records(lib, (1 << 62), -1) == ((1 << 62) - 1, NO_END)


@pytest.mark.parametrize("batches", [[1], [4], [3, 1, 5], [1024], [2, 7]], ids=lambda b: "-".join(map(str, b)))
def test_session_batches_decode_the_range(lib, batches):
    nrec = 13
    for frm, to in itertools.product(BOUNDS, BOUNDS):
        want = [i for i in range(nrec) if kept(i + 1, frm, to)]
        assert session_selection(lib, nrec, batches, frm, to) == want, (frm, to)


def test_random_ranges(lib):
    rng = np.random.default_rng(7)
    for _ in range(300):
        nrec = int(rng.integers(0, 300))
        frm, to = (int(v) for v in rng.integers(-3, nrec + 4, 2))
        batches = [int(v) for v in rng.integers(1, 40, int(rng.integers(1, 4)))]
        want = [i for i in range(nrec) if kept(i + 1, frm, to)]
        assert session_selection(lib, nrec, batches, frm, to) == want, (nrec, frm, to, batches)
