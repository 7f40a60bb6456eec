"""CPU check of the many-stream read plan (plan_reads_streams in kanzi-go_b200/csrc/kz_read_plan.h) under g++ with ASan / UBSan: random
stream sets that mix block sizes and decode groups, streams of zero blocks, sizes known or not, and requests of zero length, past the end
and at 1 << 62, held against a brute-force plan (tests/host/read_plan_streams_host.cpp). A one-stream plan must equal plan_reads."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "read_plan_streams_host.cpp")
EXE = os.path.join(ROOT, "tests", "host", "_build", "read_plan_streams_host")


@pytest.fixture(scope="module")
def exe():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", EXE, SRC],
                       cwd=os.path.dirname(SRC), capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr:
        pytest.skip("sanitizers not available: " + r.stderr[:200])
    assert r.returncode == 0, r.stderr
    return EXE


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_plan_against_brute_force(exe, seed):
    r = subprocess.run([exe, "150", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "plan check done" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
