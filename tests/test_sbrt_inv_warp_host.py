"""CPU only: the warp-resident formulation of the RANK / MTFT inverse (new rank = number of entries above with a larger q,
tests/host/sbrt_inv_warp_host.cpp) reproduces the oracle's serial list walk, on natural data and on the rank streams of tests/sbrt_corpus.py.
The corpus must also keep reaching what sbrt_inverse_warp_kernel (kz_sbrt.cu) treats apart: zero runs across rounds, whole rounds of zeros,
a run at the end of a block, a run of one continued at a round start, and a small rank (lane 0 alone) followed by a deep one."""
import ctypes as C
import importlib
import os
import subprocess
import time

import numpy as np
import pytest

import sbrt_corpus as sc
from oracle import pyoracle as po

synth = importlib.import_module("kanzi-go_b200.synth")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "sbrt_inv_warp_host.cpp")
SO = os.path.join(ROOT, "tests", "host", "_build", "libsbrt_inv_warp_host.so")


@pytest.fixture(scope="module")
def model():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SRC) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.sbrt_inverse_warp_model.restype = C.c_int64
    lib.sbrt_inverse_warp_model.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


@pytest.mark.parametrize("ttype,mode", [(po.T_RANK, 2), (po.T_MTFT, 1)])
@pytest.mark.parametrize("n", [1, 2, 255, 4096, 100003, 1 << 19])
def test_warp_model_matches_oracle(model, ttype, mode, n):
    for x in (synth.markov_text(n, seed=n), synth.uniform_bytes(n, seed=n + 1), synth.zipf_bytes(n, 1.5, seed=n + 2), np.full(n, 200, np.uint8)):
        bw, _ = po.transform_forward(po.T_BWT, x) if n >= 2 else (x, 0)  # BWT output is what RANK sees in the -l 5 chain
        for data in (x, bw):
            enc, _ = po.transform_forward(ttype, data)
            enc = np.ascontiguousarray(enc, np.uint8)
            out = np.zeros(len(enc), np.uint8)
            model.sbrt_inverse_warp_model(mode, enc.ctypes.data, len(enc), out.ctypes.data)
            assert np.array_equal(out, data), (n, mode)


@pytest.mark.parametrize("ttype,mode,name", [(po.T_RANK, 2, "RANK"), (po.T_MTFT, 1, "MTFT")])
def test_warp_model_on_rank_corpus(model, ttype, mode, name):
    t0 = time.time()
    cases = sc.corpus(ttype, po)
    for cname, r in cases:
        want = sc.expected(ttype, po, r)
        got = np.zeros(len(r), np.uint8)
        model.sbrt_inverse_warp_model(mode, r.ctypes.data, len(r), got.ctypes.data)
        assert np.array_equal(got, want), sc.first_difference(cname, name, r, got, want)
    print("%s: %d rank streams, %.1f s" % (name, len(cases), time.time() - t0))


# least count of each event over the corpus (the same in both modes: they depend on the ranks alone)
WARP_MIN = dict(run_crosses_round=1000, round_of_32_zeros=1000, run_ends_block=50, run_of_1_continues=100, small_then_deep=10000)


def test_rank_corpus_reaches_the_warp_kernel_paths():
    tot = dict.fromkeys(WARP_MIN, 0)
    for _, r in sc.corpus(po.T_RANK, po):
        for k, v in sc.warp_events(r).items():
            tot[k] += v
    print("warp kernel events:", tot)
    for k, least in WARP_MIN.items():
        assert tot[k] >= least, (k, tot[k], least)
