"""CPU check of the block cache's bookkeeping (kanzi-go_b200/csrc/kz_block_cache.h) and of the record hash it keys on
(kz_xxh64_core.cuh), under g++: the page allocator and the LRU against a brute-force model on random sequences of lookups and inserts
under small budgets (LRU order, no page owned twice, resident pages never above the budget, blocks larger than the budget refused, budget
0, slices split into page-bounded copies), run under ASan / UBSan; and the record hash of records at every bit offset 0..7 against XXH64
computed in Python over the realigned bytes, independently of the header."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import index_oracle as io_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "block_cache_host.cpp")
HDRS = [os.path.join(ROOT, "kanzi-go_b200", "csrc", h) for h in ("kz_block_cache.h", "kz_xxh64_core.cuh")]
SO = os.path.join(ROOT, "tests", "host", "_build", "libblock_cache_host.so")
EXE = os.path.join(ROOT, "tests", "host", "_build", "block_cache_fuzz")
TILE = 4096
u64 = C.c_uint64


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(f) for f in [SRC] + HDRS) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    L = C.CDLL(SO)
    L.record_hash.restype = u64
    L.record_hash.argtypes = [C.c_void_p, u64, u64]
    L.xxh64.restype = u64
    L.xxh64.argtypes = [C.c_void_p, u64, u64]
    return L


def model_record_hash(rec_bits):
    """The tree hash of a record given as an array of bits: realigned bytes, XXH64 per 4 KiB tile, XXH64 of the digests and the length."""
    nbits = len(rec_bits)
    data = np.packbits(rec_bits).tobytes()  # MSB first, zero padded to a whole byte
    digests = [io_.xxh64(data[t: t + TILE]) for t in range(0, len(data), TILE)]
    return io_.xxh64(b"".join(d.to_bytes(8, "little") for d in digests) + nbits.to_bytes(8, "little"))


def test_xxh64_matches_the_independent_one(lib):
    rng = np.random.default_rng(7)
    for n in (0, 1, 3, 4, 7, 8, 31, 32, 33, 64, 100, 1000, 4096):
        d = rng.integers(0, 256, n, dtype=np.uint8)
        for seed in (0, 0x4B414E5A):
            assert lib.xxh64(d.ctypes.data if n else None, n, seed) == io_.xxh64(d.tobytes(), seed)


@pytest.mark.parametrize("nbits", [1, 7, 8, 9, 100, 8 * TILE - 1, 8 * TILE, 8 * TILE + 1, 8 * 2 * TILE + 5, 8 * 3 * TILE])
def test_record_hash_at_every_bit_offset(lib, nbits):
    rng = np.random.default_rng(nbits)
    rec = rng.integers(0, 2, nbits, dtype=np.uint8)
    want = model_record_hash(rec)
    for lead in range(8):
        for extra in (0, 8):  # a leading byte more: the record starts further into the buffer
            start = lead + extra
            trail = rng.integers(0, 2, 13, dtype=np.uint8)  # noise behind the record's last bit
            bits = np.concatenate([rng.integers(0, 2, start, dtype=np.uint8), rec, trail])
            s = np.packbits(bits)
            assert lib.record_hash(s.ctypes.data, start, nbits) == want, (nbits, start)
    # one bit more or less, or one bit flipped, is another key
    flipped = rec.copy()
    flipped[nbits // 2] ^= 1
    assert model_record_hash(flipped) != want and model_record_hash(np.concatenate([rec, [0]])) != want


def test_cache_against_the_model_under_sanitizers():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", EXE, SRC],
                       cwd=os.path.dirname(SRC), capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr:
        pytest.skip("sanitizers not available: " + r.stderr[:200])
    assert r.returncode == 0, r.stderr
    r = subprocess.run([EXE, "200"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "cache fuzz done" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
