"""CPU check of the pass planner of kz_compress_streams / kz_decompress_streams (kanzi-go_b200/csrc/kz_stream_plan.h): every block lands in
exactly one pass and one slot, each pass's stride holds its blocks and is at most twice each member's length plus 16, and the scratch
bound and the pass budget hold, also for adversarial length mixes such as one 1 GiB block among 10^5 one-byte blocks. Also the decode
slot stride and the error order of every stream-level decode (DecodeFailure): the earliest stage wins, then the earliest block. Also what
every encode path decides per block: how streams are cut into blocks, the data type a block's magic number gives, and which blocks
skipBlocks stores, against the statement of tests/skip_oracle.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import skip_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "stream_plan_host.cpp")
HDR = os.path.join(ROOT, "kanzi-go_b200", "csrc", "kz_stream_plan.h")
SO = os.path.join(ROOT, "tests", "host", "_build", "libstream_plan_host.so")
BUDGET = 1 << 30  # STREAM_PASS_BUDGET


@pytest.fixture(scope="module")
def plan():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or max(os.path.getmtime(SRC), os.path.getmtime(HDR)) > os.path.getmtime(SO):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-x", "c++", "-o", SO, SRC])
    lib = C.CDLL(SO)
    lib.plan_compress.restype = C.c_uint32
    lib.plan_compress.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.compress_cost.restype = C.c_uint64
    lib.compress_cost.argtypes = [C.c_uint64]
    lib.plan_decompress.restype = C.c_uint32
    lib.plan_decompress.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.decompress_cost.restype = C.c_uint64
    lib.decompress_cost.argtypes = [C.c_uint32]
    lib.decode_stride.restype = C.c_uint64
    lib.decode_stride.argtypes = [C.c_uint32, C.c_uint32]
    lib.note_failures.restype = C.c_int32
    lib.note_failures.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_int32)]
    lib.cut_blocks.restype = C.c_uint32
    lib.cut_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.magic_data_type.restype = C.c_int32
    lib.magic_data_type.argtypes = [C.c_char_p, C.c_uint32]
    lib.stored_blocks.restype = None
    lib.stored_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return lib


def check_compress(lib, lens, budget=BUDGET):
    lens = np.ascontiguousarray(lens, np.uint32)
    n = len(lens)
    ps, sl, st = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint64)
    scratch = C.c_uint64(0)
    npass = lib.plan_compress(lens.ctypes.data, n, budget, ps.ctypes.data, sl.ctypes.data, st.ctypes.data, C.byref(scratch))
    ps, sl, st = ps[:n], sl[:n], st[:npass]
    if n == 0:
        assert npass == 0 and scratch.value == 0
        return npass
    # every block in exactly one pass, and the slots of a pass are 0 .. count-1, each taken once
    assert ps.max() < npass
    counts = np.bincount(ps, minlength=npass)
    assert (counts > 0).all()
    for p in range(npass):
        assert sorted(sl[ps == p].tolist()) == list(range(int(counts[p])))
    # each stride holds its blocks and is at most twice each member's length plus 16
    eff = np.maximum(lens.astype(np.uint64), 1)
    assert (st % 16 == 0).all()
    assert (eff <= st[ps]).all()
    assert (st[ps] <= 2 * eff + 16).all()
    # the pass budget holds, except for a pass of one block, and the reported scratch is the largest pass
    cost = np.array([lib.compress_cost(int(s)) for s in st], np.uint64)
    per_pass = counts.astype(np.uint64) * cost
    assert ((per_pass <= budget) | (counts == 1)).all()
    assert scratch.value == int(per_pass.max())
    assert scratch.value <= max(budget, int(lib.compress_cost(int(st.max()))))
    return npass


def test_empty_and_uniform(plan):
    assert check_compress(plan, []) == 0
    assert check_compress(plan, [1]) == 1
    assert check_compress(plan, [65536] * 300) == 1


def test_mixed_lengths(plan):
    rng = np.random.default_rng(1)
    lens = np.exp(rng.normal(np.log(16384), 1.5, 20000)).clip(1, 4 << 20).astype(np.uint32)
    npass = check_compress(plan, lens)
    assert npass < 40


def test_one_huge_block_among_tiny_ones(plan):
    """one 1 GiB block among 10^5 one-byte and fifteen-byte blocks: the huge block runs alone, the tiny ones share small strides"""
    lens = np.ones(100001, np.uint32)
    lens[::2] = 15
    lens[50000] = 1 << 30
    check_compress(plan, lens)
    ps, sl, st = np.zeros(len(lens), np.uint32), np.zeros(len(lens), np.uint32), np.zeros(len(lens), np.uint64)
    scratch = C.c_uint64(0)
    npass = plan.plan_compress(lens.ctypes.data, len(lens), BUDGET, ps.ctypes.data, sl.ctypes.data, st.ctypes.data, C.byref(scratch))
    assert (ps == ps[50000]).sum() == 1
    assert st[:npass][np.arange(npass) != ps[50000]].max() == 16


def test_small_budget_and_geometric_lengths(plan):
    lens = np.array([1 << k for k in range(31)] * 3, np.uint32)
    check_compress(plan, lens)
    check_compress(plan, lens, budget=1 << 20)
    rng = np.random.default_rng(2)
    check_compress(plan, rng.integers(0, 1 << 22, 5000).astype(np.uint32), budget=64 << 20)


@pytest.mark.parametrize("n,bs", [(0, 1024), (1, 1 << 30), (100000, 1024), (5000, 4 << 20), (300, 32 << 20), (7, 1 << 30)])
def test_decompress_passes(plan, n, bs):
    ps, sl = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    scratch = C.c_uint64(0)
    npass = plan.plan_decompress(n, bs, BUDGET, ps.ctypes.data, sl.ctypes.data, C.byref(scratch))
    ps, sl = ps[:n], sl[:n]
    cost = plan.decompress_cost(bs)
    per = max(1, BUDGET // cost)
    assert npass == (n + per - 1) // per
    if n:
        assert (np.diff(ps.astype(np.int64)) >= 0).all()  # blocks keep their order
        counts = np.bincount(ps, minlength=npass)
        assert (counts <= per).all() and counts.sum() == n
        for p in range(npass):
            assert sl[ps == p].tolist() == list(range(int(counts[p])))
        assert scratch.value == int(counts.max()) * cost
        assert scratch.value <= max(BUDGET, cost)


@pytest.mark.parametrize("bs", [1024, 65536, 4 << 20, 1 << 30])
def test_decode_stride(plan, bs):
    """Reader.processBlock's buffer plus 64 bytes, rounded to 16, or longer when a block header claims a longer entropy output"""
    for max_pre in (0, 1, bs, bs + max(512, bs >> 4), bs + max(512, bs >> 4) + 1, max(2048, bs + bs // 2)):
        want = (max(max_pre, bs + max(512, bs >> 4)) + 64 + 15) & ~15
        assert plan.decode_stride(bs, max_pre) == want
    assert plan.decode_stride(bs, 0) == plan.decompress_cost(bs) // 2


WALK, HEADER, DECODE, INVERSE, CHECKSUM, DONE = range(6)


def note_failures(lib, notes):
    stage = np.array([s for s, _ in notes] or [0], np.int32)
    code = np.array([c for _, c in notes] or [0], np.int32)
    runs = np.zeros(max(len(notes), 1), np.uint8)
    out_stage = C.c_int32(-1)
    rc = lib.note_failures(stage.ctypes.data, code.ctypes.data, len(notes), runs.ctypes.data, C.byref(out_stage))
    return rc, out_stage.value, runs[: len(notes)].astype(bool).tolist()


def test_failure_none(plan):
    assert note_failures(plan, []) == (0, DONE, [])


def test_failure_earliest_stage_wins(plan):
    """a later block's failure at an earlier stage beats an earlier block's at a later stage"""
    rc, st, runs = note_failures(plan, [(CHECKSUM, -10), (INVERSE, -9), (DECODE, -7), (HEADER, -13)])
    assert (rc, st) == (-13, HEADER)
    assert runs == [True, True, True, True]


def test_failure_earliest_block_within_a_stage(plan):
    rc, st, runs = note_failures(plan, [(DECODE, -7), (DECODE, -13), (DECODE, -10)])
    assert (rc, st) == (-7, DECODE)
    assert runs == [True, False, False]


def test_failure_skips_later_stages(plan):
    """once a stream has failed, its blocks run no stage whose failure could not beat the one it holds"""
    rc, st, runs = note_failures(plan, [(INVERSE, -13), (CHECKSUM, -10), (INVERSE, -9), (DECODE, -7), (INVERSE, -13), (CHECKSUM, -10)])
    assert (rc, st) == (-7, DECODE)
    assert runs == [True, False, False, True, False, False]
    rc, st, runs = note_failures(plan, [(HEADER, -13), (DECODE, -7), (HEADER, -10), (WALK, -9)])
    assert (rc, st) == (-9, WALK)
    assert runs == [True, False, False, True]


def cut(lib, off, lens, bs):
    off, lens = np.ascontiguousarray(off, np.uint64), np.ascontiguousarray(lens, np.uint64)
    ns, room = len(lens), int(sum((int(n) + bs - 1) // bs for n in lens)) + 1
    boff, blen, first = np.zeros(room, np.uint64), np.zeros(room, np.uint32), np.zeros(ns + 1, np.uint32)
    nb = lib.cut_blocks(off.ctypes.data, lens.ctypes.data, ns, bs, boff.ctypes.data, blen.ctypes.data, first.ctypes.data)
    return boff[:nb].tolist(), blen[:nb].tolist(), first.tolist()


@pytest.mark.parametrize("bs", [1024, 4 << 20])
def test_cut_blocks(plan, bs):
    """Writer.Write's cut: blockSize pieces and a shorter last one, stream after stream; an empty stream has none"""
    lens = [0, bs, 3 * bs, 2 * bs + 1, 1, 0, bs - 1, 0]
    off = [7, 7, bs + 16, 5 * bs, 8 * bs + 3, 9 * bs, 9 * bs, 10 * bs]
    boff, blen, first = cut(plan, off, lens, bs)
    want_off, want_len, want_first = [], [], []
    for o, n in zip(off, lens):
        want_first.append(len(want_len))
        for k in range(0, n, bs):
            want_off.append(o + k)
            want_len.append(min(bs, n - k))
    want_first.append(len(want_len))
    assert (boff, blen, first) == (want_off, want_len, want_first)
    assert first == [0, 0, 1, 4, 7, 8, 8, 9, 9]
    # the whole-stream encode is the one-stream case
    assert cut(plan, [0], [3 * bs + 5], bs) == ([0, bs, 2 * bs, 3 * bs], [bs, bs, bs, 5], [0, 4])
    assert cut(plan, [0], [0], bs) == ([], [], [0, 0])
    assert cut(plan, [], [], bs) == ([], [], [0])


# internal/Magic.go:155-206 IsDataMultimedia / IsDataExecutable, over the keys of tests/skip_oracle.py
MULTIMEDIA = {so.JPG, so.GIF, so.PNG, so.RIFF, so.FLAC, so.ID3, so.BMP, so.PBM, so.PGM, so.PPM}
EXECUTABLE = {so.ELF, so.WIN, so.MAC32, so.CIGAM32, so.MAC64, so.CIGAM64}


def data_type(block):
    """encodingTask.encode's initial dataType (io/CompressedStream.go:806-816): DT_BIN 7, DT_MULTIMEDIA 2, DT_EXE 3, else 0"""
    m = so.magic_type(block)
    return 7 if m in so.COMPRESSED else 2 if m in MULTIMEDIA else 3 if m in EXECUTABLE else 0


def magic_heads():
    """every compressed magic number (the 24- and 16-bit ones with every kind of byte behind), JPEG's APP0 key against APP1..APP15, the PDF /
    ELF / Mach-O / RIFF / BMP / MZ heads, PBM / PGM / PPM with and without white space behind, and keys of no format"""
    heads = []
    for k in sorted(so.COMPRESSED):
        if k >> 16 == 0:  # 16-bit key (gzip)
            heads += [(k << 16) | t for t in (0x0000, 0x0800, 0xFFFF)]
        elif k >> 24 == 0:  # 24-bit key (bzip2, ID3)
            heads += [(k << 8) | t for t in (0x00, 0x39, 0xFF)]
        else:
            heads.append(k)
    heads += [0xFFD8FFE0 | i for i in range(16)]
    heads += [so.PDF, so.ELF, so.MAC32, so.CIGAM32, so.MAC64, so.CIGAM64, so.RIFF, (so.BMP << 16) | 0x3604, (so.WIN << 16) | 0x9000]
    heads += [(p << 16) | (ws << 8) | 0x31 for p in (so.PBM, so.PGM, so.PPM) for ws in (0x07, 0x0A, 0x0D, 0x20, 0x09, 0x41)]
    heads += [0x00000000, 0x12345678, 0xFFD8FF00, 0x4B414E5B, 0x1F8A0000]
    return [h.to_bytes(4, "big") for h in heads]


def test_magic_data_type(plan):
    for head in magic_heads():
        for n in (0, 3, 4, 15, 16, 4096):
            block = (head * 1024)[:n]
            padded = bytes(block[:4]).ljust(4, b"\0")
            assert plan.magic_data_type(padded, n) == data_type(block), (head.hex(), n)
    assert plan.magic_data_type(bytes.fromhex("ffd8ffe0"), 16) == 7
    assert all(plan.magic_data_type(bytes.fromhex("ffd8ffe%x" % i), 16) == 0 for i in range(1, 16))


def test_store_rule(plan):
    """stored when longer than 15 bytes and the head is a compressed format's or the entropy test says so: exactly the blocks
    skip_oracle.reason stores for "magic" / "entropy" (the "small" ones are the forward stage's COPY blocks, not this rule's)"""
    rng = np.random.default_rng(3)
    blocks = []
    for head in magic_heads():
        for n in (3, 15, 16, 4096):
            for tail in (np.zeros(n, np.uint8), rng.integers(0, 256, n, dtype=np.uint8)):  # the entropy flag off and on
                b = tail.copy()
                b[: min(4, n)] = np.frombuffer(head, np.uint8)[: min(4, n)]
                blocks.append(b)
    nb = len(blocks)
    heads = np.zeros((nb, 4), np.uint8)
    for i, b in enumerate(blocks):
        heads[i, : min(4, len(b))] = b[:4]
    flags = np.array([so.block_entropy(b) >= so.INCOMPRESSIBLE_THRESHOLD for b in blocks], np.uint8)
    assert flags.any() and not flags.all()
    lens = np.array([len(b) for b in blocks], np.uint32)
    store, counts = np.zeros(nb, np.uint8), np.zeros(4, np.uint64)
    plan.stored_blocks(heads.ctypes.data, flags.ctypes.data, lens.ctypes.data, nb, store.ctypes.data, counts.ctypes.data)
    reasons = [so.reason(b) for b in blocks]
    assert store.tolist() == [int(r in ("magic", "entropy")) for r in reasons]
    for i, r in enumerate(reasons):  # both states of the flag on blocks the magic number stores
        if r == "magic":
            assert data_type(blocks[i]) == 7
    by = {r: [len(b) for b, q in zip(blocks, reasons) if q == r] for r in ("magic", "entropy")}
    assert by["magic"] and by["entropy"]
    assert counts.tolist() == [len(by["magic"]), sum(by["magic"]), len(by["entropy"]), sum(by["entropy"])]
    # the flag alone decides a block whose head is no compressed format's
    assert {(int(f), int(s)) for f, s, r, b in zip(flags, store, reasons, blocks) if len(b) > 15 and data_type(b) != 7} == {(0, 0), (1, 1)}
