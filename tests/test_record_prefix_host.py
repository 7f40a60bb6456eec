"""CPU check of write_block_prefix (kanzi-go_b200/csrc/kz_common.cuh), the 5 b | lw b prefix of every block record that the single-stream and
the many-stream assemblies write, against a restatement of the reference's commit (io/CompressedStream.go:951-976): lw = 3 below 8 bits,
else Log2(written >> 3) + 4, then lw - 3 on 5 bits and written on lw bits. Block bit lengths of 2^32 bits and more (lw > 32) are covered
here because no GPU test compresses a block that large."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "record_prefix_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_common.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "librecord_prefix_host.so")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", CUDA_INC, "-o", SO, SRC])
    L = C.CDLL(SO)
    L.record_prefix.restype = C.c_uint32
    L.record_prefix.argtypes = [C.c_uint64, C.c_void_p]
    return L


def reference(written):
    lw = 3 if written < 8 else (written >> 3).bit_length() - 1 + 4
    bits = format(lw - 3, "05b") + format(written, "0%db" % lw)
    padded = bits + "0" * (-len(bits) % 8)
    return len(bits), bytes(int(padded[i: i + 8], 2) for i in range(0, len(padded), 8))


def test_prefix_matches_the_reference_commit(lib):
    # lw - 3 has 5 bits, so lw <= 34: records up to 2^34 - 1 bits (a 1 GiB block writes fewer than 2^33 + 2^30)
    values = list(range(0, 300)) + [(1 << k) + d for k in range(3, 34) for d in (-1, 0, 1)] + [(1 << 33) + 12345, (8 << 30) + 7, (1 << 34) - 1]
    out = np.zeros(8, np.uint8)
    for w in values:
        n = lib.record_prefix(w, out.ctypes.data)
        want_n, want = reference(w)
        assert n == want_n and bytes(out[: len(want)]) == want, (w, n, want_n)
        if w >= 1 << 32:
            assert n - 5 > 32  # the two-part write of lw > 32 bits
