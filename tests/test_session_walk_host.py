"""CPU checks of the streaming reader's resumable record walk (walk_records over read_block_prefix, kanzi-go_b200/csrc/kz_common.cuh) and the
writer's carry rule (batch_bytes_out): oracle streams cut at every byte offset give exactly the records that lie completely before the cut and
never an error, the end marker only when it is inside; a length longer than any block of the stream fails; batches of any bit length, committed
with their carry, concatenate to the stream."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "session_walk_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_common.cuh")
SO = os.path.join(ROOT, "tests", "host", "_build", "libsession_walk_host.so")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
E_PROCESS_BLOCK = 13
NO_LIMIT = 1 << 40


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", CUDA_INC, "-o", SO, SRC])
    L = C.CDLL(SO)
    L.walk.restype = C.c_uint32
    L.walk.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    L.carry_commit.restype = C.c_uint64
    L.carry_commit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


def walk(lib, data, start, max_records=1 << 16, max_bits=NO_LIMIT):
    a = np.ascontiguousarray(np.frombuffer(bytes(data), np.uint8)) if len(data) else np.zeros(1, np.uint8)
    off = np.zeros(max_records + 1, np.uint64)
    bits = np.zeros(max_records + 1, np.uint64)
    res = np.zeros(4, np.int64)
    lib.walk(a.ctypes.data, len(data), start, max_records, max_bits, off.ctypes.data, bits.ctypes.data, res.ctypes.data)
    n = int(res[0])
    return [(int(off[i]), int(bits[i])) for i in range(n)], int(res[1]), bool(res[2]), int(res[3])


def header_bits(stream):
    """Writer.writeHeader (io/CompressedStream.go:429-519): 119 bits of fields, the 2-bit size mask, 0/16/32/48 size bits, 15 + 24 bits"""
    v = int.from_bytes(bytes(stream[:16]), "big")
    mask = (v >> (128 - 121)) & 3
    return 119 + 2 + (0, 16, 32, 48)[mask] + 15 + 24


CHAINS = [("NONE", "NONE", 0), ("NONE", "ANS0", 32), ("LZ", "HUFFMAN", 0), ("BWT+RANK+ZRLT", "ANS0", 64), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 0),
          ("LZ", "RANGE", 32)]


@pytest.mark.parametrize("chain", CHAINS, ids=["%s-%s-x%d" % c for c in CHAINS])
def test_cut_streams_walk_to_the_records_before_the_cut(lib, oracle, kz, chain):
    synth = __import__("importlib").import_module("kanzi-go_b200.synth")
    tr, en, ck = chain
    x = synth.markov_text(9 * 1024 + 333, seed=len(tr) + ck)
    s = oracle.compress(x, tr, en, block_size=1024, checksum_bits=ck, input_size=len(x))
    h = header_bits(s)
    recs, st, ended, nxt = walk(lib, s, h)
    assert st == 0 and ended and len(recs) == 10, (st, ended, len(recs))
    end_marker = recs[-1][0] + recs[-1][1] + 8
    assert nxt == end_marker and (end_marker + 7) // 8 == len(s)
    for cut in range(h // 8 + 1, len(s) + 1):
        got, st, ended, nxt = walk(lib, s[:cut], h)
        want = [r for r in recs if r[0] + r[1] <= 8 * cut]
        assert st == 0 and got == want, (cut, st)
        assert ended == (end_marker <= 8 * cut), cut
        assert nxt == (end_marker if ended else (want[-1][0] + want[-1][1] if want else h)), cut
    # resumable: one record at a time from where the last call stopped
    pos, got = h, []
    while True:
        r, st, ended, pos = walk(lib, s, pos, max_records=1)
        assert st == 0
        got += r
        if ended:
            break
    assert got == recs


def prefix(lw, value):
    bits = format(lw - 3, "05b") + format(value, "0%db" % lw)
    bits += "0" * (-len(bits) % 8)
    return bytes(int(bits[i: i + 8], 2) for i in range(0, len(bits), 8)) + bytes(16)


def test_corrupt_lengths(lib):
    # lw - 3 has 5 bits, so a length has at most 34 bits and never exceeds stream_walk_kernel's 2^34 limit: the largest one the format
    # allows is a record the walk waits for when no bound applies
    _, st, ended, _ = walk(lib, prefix(34, (1 << 34) - 1), 0)
    assert st == 0 and not ended
    # longer than any block of the stream can be: -KZ_E_PROCESS_BLOCK (what the whole-stream walk gives when it runs past the end)
    _, st, _, _ = walk(lib, prefix(20, 600000), 0, max_bits=500000)
    assert st == -E_PROCESS_BLOCK
    recs, st, ended, nxt = walk(lib, prefix(20, 100) + bytes(20), 0, max_bits=500000)
    assert st == 0 and recs == [(25, 100)] and ended and nxt == 125 + 8


def test_carry_commit(lib):
    rng = np.random.default_rng(3)
    for trial in range(200):
        nb = int(rng.integers(1, 8))
        bb = rng.integers(0, 200, nb).astype(np.uint64)
        if trial % 3 == 0:
            bb[:] = 8 * rng.integers(0, 20, nb)  # byte-aligned batches
        total = int(bb.sum())
        stream = rng.integers(0, 256, (total + 7) // 8 + 1).astype(np.uint8)
        if total % 8:
            stream[total // 8] &= (0xFF << (8 - total % 8)) & 0xFF
        stream[(total + 7) // 8:] = 0
        out = np.zeros(total // 8 + 16, np.uint8)
        n = lib.carry_commit(stream.ctypes.data, bb.ctypes.data, nb, out.ctypes.data)
        assert n == (total + 7) // 8
        assert np.array_equal(out[:n], stream[:n]), trial
