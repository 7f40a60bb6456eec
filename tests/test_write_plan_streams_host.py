"""CPU check of the many-stream write plan (plan_writes_streams in kanzi-go_b200/csrc/kz_write_plan.h) under g++ with ASan / UBSan: random
stream sets that mix block sizes and groups, empty streams, sizes known or not and streams that take no part, with interleaved writes of
zero length, KZ_WRITE_APPEND, overlaps and offsets near 2^62 (tests/host/write_plan_streams_host.cpp). Each stream's plan must equal
plan_writes over its own writes, every pass must hold one group within the budget, the pair order must be deterministic, and a one-stream
plan must equal the single plan."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "write_plan_streams_host.cpp")
EXE = os.path.join(ROOT, "tests", "host", "_build", "write_plan_streams_host")


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
def test_plan_against_single_plans(exe, seed):
    r = subprocess.run([exe, "200", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "plan check done" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
