"""CPU check of the RANK / MTFT inverse for blocks of at most 16 MiB (sbrt_inverse_multi_kernel, kanzi-go_b200/csrc/kz_sbrt.cu) in the
schedule the kernel runs: ranks staged in shared memory a round ahead and held as words, sentinel slots above position 0 in both mirror
copies. Modelled thread by thread in tests/host/sbrt_inv_multi_staged_host.cpp and run on the adversarial rank streams of
tests/sbrt_corpus.py: the output must equal the oracle's inverse byte for byte, and the corpus must reach every decision of the kernel as
often as test_sbrt_inv_multi_host.py asks of the schedule before it (the same event minimums)."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import sbrt_corpus as sc
from oracle import pyoracle as po
from test_sbrt_inv_multi_host import MTFT_MIN, MTFT_NEVER, RANK_MIN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "sbrt_inv_multi_staged_host.cpp")
SO = os.path.join(ROOT, "tests", "host", "_build", "libsbrt_inv_multi_staged_host.so")


@pytest.fixture(scope="module")
def staged_model():
    po.build()
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SRC) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.sbrt_inverse_multi_model.restype = C.c_int
    lib.sbrt_inverse_multi_model.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.sbrt_inv_multi_event_names.restype = C.c_char_p
    lib.sbrt_inv_multi_event_count.restype = C.c_int
    return lib


@pytest.mark.parametrize("ttype,mode,name", [(po.T_RANK, 2, "RANK"), (po.T_MTFT, 1, "MTFT")])
def test_staged_model_on_rank_corpus(staged_model, ttype, mode, name):
    t0 = time.time()
    names = staged_model.sbrt_inv_multi_event_names().decode().split(",")
    ev = np.zeros(staged_model.sbrt_inv_multi_event_count(), np.uint64)
    assert len(names) == len(ev)
    cases = sc.corpus(ttype, po)
    for cname, r in cases:
        want = sc.expected(ttype, po, r)
        got = np.zeros(len(r), np.uint8)
        assert staged_model.sbrt_inverse_multi_model(mode, r.ctypes.data, len(r), got.ctypes.data, ev.ctypes.data) == 0
        assert np.array_equal(got, want), sc.first_difference(cname, name, r, got, want)
    counts = dict(zip(names, (int(v) for v in ev)))
    print("%s: %d rank streams, %d ranks, %.1f s; events %s" % (name, len(cases), sum(len(r) for _, r in cases), time.time() - t0, counts))
    for ename, least in (RANK_MIN if mode == 2 else MTFT_MIN).items():
        assert counts[ename] >= least, (name, ename, counts[ename], least)
    if mode == 1:
        assert all(counts[e] == 0 for e in MTFT_NEVER), counts
        assert counts["ca_tie"] + counts["cb_tie"] <= 2 * len(cases), counts  # the first step of a stream only
