"""CPU check of the RANK / MTFT forward's per-segment rule (kanzi-go_b200/csrc/kz_sbrt_core.cuh, what sbrt_rank_kernel runs for every byte):
32-bit keys counted against key(c), tie terms for keys that can tie, 4 KiB segments started from the carried (last, second last) positions.
The output must equal the oracle's SBRT forward byte for byte."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

synth = importlib.import_module("kanzi-go_b200.synth")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "sbrt_core_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_sbrt_core.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "libsbrt_core_host.so")
MODES = [(po.T_MTFT, 1), (po.T_RANK, 2)]


@pytest.fixture(scope="module")
def core():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.sbrt_core_forward.restype = C.c_int
    lib.sbrt_core_forward.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
    return lib


def check(core, x, modes=MODES):
    """core == oracle for every mode; returns the number of bytes that took the tie terms, per mode"""
    x = np.ascontiguousarray(x, np.uint8)
    ties = []
    for ttype, mode in modes:
        want, _ = po.transform_forward(ttype, x)
        got = np.zeros(max(len(x), 1), np.uint8)
        n_ties = C.c_uint64(0)
        assert core.sbrt_core_forward(mode, x.ctypes.data, len(x), got.ctypes.data, C.byref(n_ties)) == 0
        got = got[: len(x)]
        assert np.array_equal(got, want), (mode, len(x), int(np.argmax(got != want)))
        ties.append(n_ties.value)
    return ties


@pytest.mark.parametrize("n", [1, 15, 16, 4095, 4096, 4097, 3 * 4096 + 5, 100003])
def test_segment_boundaries(core, n):
    for x in (synth.markov_text(n, seed=n), synth.uniform_bytes(n, seed=n + 1), synth.zipf_bytes(n, 1.2, seed=n + 2), synth.runs_bytes(n, seed=n + 3),
              np.full(n, 7, np.uint8)):
        check(core, x)


def test_symbols_never_seen(core):
    """symbols that first appear segments after the start, in descending and in random order: t = -1 - d orders them by symbol"""
    r = np.random.default_rng(3)
    head = r.integers(0, 8, 9000).astype(np.uint8)
    for late in (np.arange(255, 7, -1, dtype=np.uint8), r.permutation(np.arange(8, 256)).astype(np.uint8)):
        x = np.concatenate([head, np.repeat(late, 37), head[:5000]])
        ties = check(core, x)
        assert min(ties) >= len(late)  # every first occurrence took the tie terms


def test_equal_q_for_different_symbols(core):
    """RANK q = (l1 + l2) >> 1: sums that collide after the shift, both with small gaps (keys exact) and with gaps above 2 x 254 (keys clipped,
    the tie terms decide)"""
    r = np.random.default_rng(5)
    x = r.integers(0, 3, 50000).astype(np.uint8)  # abba, aabb, ...: equal q all the time
    check(core, x)
    n = 64 * 2048
    x = r.integers(16, 256, n).astype(np.uint8)
    for k in range(64):
        b = 2048 * k
        a, c = 2 * (k % 8), 2 * (k % 8) + 1
        # a at b, b + 1000 (q = b + 500); c at b + 100, b + 900 (q = b + 500) or b + 101, b + 900 (sum one higher, same q after >> 1)
        x[b], x[b + 1000] = a, a
        x[b + 100 + (k & 1)], x[b + 900] = c, c
        x[b + 1001], x[b + 1002], x[b + 1003] = (c, a, c) if k % 3 else (a, c, a)
    ties = check(core, x)
    assert ties[1] > 2 * 64


def test_runs_and_all_symbols(core):
    r = np.random.default_rng(9)
    runs = np.repeat(r.integers(0, 256, 3000).astype(np.uint8), r.integers(1, 300, 3000))
    check(core, runs)
    check(core, (np.arange(70000) % 256).astype(np.uint8))  # every symbol, each at distance 256 (clipped in RANK mode)
    check(core, (255 - np.arange(70000) % 256).astype(np.uint8))
    check(core, np.concatenate([r.permutation(256).astype(np.uint8) for _ in range(300)]))


def test_bwt_of_silesia_shaped_data(core):
    """what RANK sees in kanzi -l 5: the BWT output of the bench's silesia-shaped slab, at 1 MiB"""
    x = synth.silesia_shaped(1 << 20, seed=11)
    bw, _ = po.transform_forward(po.T_BWT, x)
    ties = check(core, bw)
    print("bytes with the tie terms: MTFT %d, RANK %d of %d" % (ties[0], ties[1], len(bw)))
