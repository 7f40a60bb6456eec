"""CPU check of the RANK / MTFT inverse for blocks of at most 16 MiB (sbrt_inverse_multi_kernel, kanzi-go_b200/csrc/kz_sbrt.cu), modelled
thread by thread in tests/host/sbrt_inv_multi_host.cpp, on the adversarial rank streams of tests/sbrt_corpus.py: the output must equal the
oracle's inverse byte for byte, and the corpus must keep reaching every decision of the kernel (event minimums below)."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import sbrt_corpus as sc
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "sbrt_inv_multi_host.cpp")
SO = os.path.join(ROOT, "tests", "host", "_build", "libsbrt_inv_multi_host.so")

# Least count of each event over the corpus. RANK mode: the entry the step leaves at rank r2 (fresh, moved down, stayed; the sentinel
# above rank 0; equal q in either candidate), the fresh entry entering lane 0 of warps 1..3 through the mirror (with and without equal
# q), entries crossing each warp boundary, and every tail length. 100003 uniform ranks alone give some 600 exact warp-boundary insertions.
RANK_MIN = dict(fresh_at_r2=10000, down_to_r2=10000, cand_stays=10000, sentinel_move=10000, ca_tie=1000, cb_tie=1000, insert_64=50,
                insert_128=50, insert_192=50, insert_warp_tie=10, cross_64=10000, cross_128=10000, cross_192=10000,
                **{"tail%d" % t: 1 for t in range(32)})
# MTFT mode: qc = i is above every q in the list (after the first step, where every q and qc are 0), so the new rank is always 0: the
# fresh entry lands at r2 only for r2 == 0 (the sentinel), a candidate never stays when r2 <= r, and there is no insertion at a warp
# boundary. What remains is the move, the sentinel, the boundary crossings and the tails.
MTFT_MIN = dict(fresh_at_r2=10000, down_to_r2=10000, sentinel_move=10000, cross_64=10000, cross_128=10000, cross_192=10000,
                **{"tail%d" % t: 1 for t in range(32)})
MTFT_NEVER = ("cand_stays", "insert_64", "insert_128", "insert_192", "insert_warp_tie")


@pytest.fixture(scope="module")
def model():
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
def test_multi_model_on_rank_corpus(model, ttype, mode, name):
    t0 = time.time()
    names = model.sbrt_inv_multi_event_names().decode().split(",")
    ev = np.zeros(model.sbrt_inv_multi_event_count(), np.uint64)
    assert len(names) == len(ev)
    cases = sc.corpus(ttype, po)
    for cname, r in cases:
        want = sc.expected(ttype, po, r)
        got = np.zeros(len(r), np.uint8)
        assert model.sbrt_inverse_multi_model(mode, r.ctypes.data, len(r), got.ctypes.data, ev.ctypes.data) == 0
        assert np.array_equal(got, want), sc.first_difference(cname, name, r, got, want)
    counts = dict(zip(names, (int(v) for v in ev)))
    print("%s: %d rank streams, %d ranks, %.1f s; events %s" % (name, len(cases), sum(len(r) for _, r in cases), time.time() - t0, counts))
    for ename, least in (RANK_MIN if mode == 2 else MTFT_MIN).items():
        assert counts[ename] >= least, (name, ename, counts[ename], least)
    if mode == 1:
        assert all(counts[e] == 0 for e in MTFT_NEVER), counts
        assert counts["ca_tie"] + counts["cb_tie"] <= 2 * len(cases), counts  # the first step of a stream only
