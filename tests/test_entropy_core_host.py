"""CPU check of the order-0 entropy core (kanzi-go_b200/csrc/kz_entropy_core.cuh) that skip_decide_kernel and the MM transform's kernels
run: its LOG2_4096 table is the reference's, and Log2ScaledBy1024, ComputeFirstOrderEntropy1024 and the INCOMPRESSIBLE_THRESHOLD test
equal the independent statement in tests/skip_oracle.py, on histograms of 16 bytes to 1 GiB, including the 972 / 973 boundary."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import skip_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "entropy_core_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_entropy_core.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "libentropy_core_host.so")


@pytest.fixture(scope="module")
def core():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.entropy_core_log2_4096.argtypes = [C.c_void_p]
    lib.entropy_core_log2_4096.restype = None
    lib.entropy_core_log2_scaled_1024.argtypes = [C.c_uint32]
    lib.entropy_core_log2_scaled_1024.restype = C.c_uint32
    lib.entropy_core_entropy_1024.argtypes = [C.c_uint32, C.c_void_p]
    lib.entropy_core_incompressible.argtypes = [C.c_uint32, C.c_void_p]
    return lib


def _entropy(core, h):
    h = np.ascontiguousarray(h, np.uint32)
    n = int(h.sum())
    return core.entropy_core_entropy_1024(n, h.ctypes.data), core.entropy_core_incompressible(n, h.ctypes.data), n


def test_log2_table_is_the_reference_table(core):
    t = np.zeros(257, np.uint32)
    core.entropy_core_log2_4096(t.ctypes.data)
    assert t.tolist() == so.LOG2_4096


def test_log2_scaled_1024(core):
    xs = list(range(1, 5000)) + [(1 << k) + d for k in range(12, 31) for d in (-1, 0, 1, 12345)] + [(1 << 30) - 16, 1 << 30]
    for x in xs:
        assert core.entropy_core_log2_scaled_1024(x) == so.log2_scaled_1024(x), x


def test_entropy_and_threshold(core):
    rng = np.random.default_rng(1)
    cases = [np.bincount(np.arange(16) % 256, minlength=256), np.eye(256, dtype=np.int64)[7] * 1000, np.full(256, 1 << 22)]  # 1 GiB uniform
    for n in (16, 100, 4096, 1 << 16, 1 << 22, 1 << 30):
        for alpha in (0.2, 1.0, 4.0):
            p = rng.dirichlet(np.full(256, alpha))
            cases.append(rng.multinomial(n, p))
    for target in (972, 973):
        for n in (1 << 12, 1 << 16):
            cases.append(np.bincount(so.entropy_block(target, n), minlength=256))
    for h in cases:
        e, inc, n = _entropy(core, h)
        assert e == so.entropy_1024(n, h), n
        assert inc == (e >= so.INCOMPRESSIBLE_THRESHOLD)
