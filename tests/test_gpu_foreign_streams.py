"""The data-parallel inverses of LZ / LZX, ZRLT, MM, PACK / DNA and TEXT on stage streams that no encoder here writes
(tests/foreign_streams.py), against the oracle's inverse. Every case obeys one rule: the oracle decodes it -> the GPU decodes it to the
same bytes; the oracle rejects it -> the GPU rejects it with the same code. Routes: kz_transform_inverse over a sweep of caps around the
output length, kz_decode_blocks on batches of one-stage E_NONE block records (status per block), and whole streams.

The LZ cases also check where they ran: a stream lzi_parse_kernel can take never reaches lz_inverse_serial, every other one does.
"""
import numpy as np
import pytest

import foreign_streams as fs

pytestmark = pytest.mark.gpu

PROBE = 40 << 20  # the cap at which the oracle gives a case's output length
BS = 1 << 16      # block size of the batches: every stage gets bs + max(512, bs >> 4) bytes on both sides (see block_batch)


def oracle_inverse(oracle, t, s, cap, block_size=0):
    """-> (bytes or None, error code or 0, exact): exact is False when the output depends on what the destination held before (the
    reference copies bytes it never wrote); then only the verdict and the length can be compared"""
    try:
        a = oracle.transform_inverse(t, s, cap, block_size=block_size, fill=0)
    except oracle.OracleError as e:
        return None, e.code, True
    b = oracle.transform_inverse(t, s, cap, block_size=block_size, fill=0xA5)
    return a, 0, np.array_equal(a, b)


def gpu_inverse(gpu, kz, t, s, cap):
    try:
        return gpu.transform_inverse(t, s, cap), 0
    except kz.KanziError as e:
        return None, e.code


def check_one(gpu, kz, oracle, t, name, s, cap, block_size=0):
    want, wcode, exact = oracle_inverse(oracle, t, s, cap, block_size)
    got, gcode = gpu_inverse(gpu, kz, t, s, cap)
    where = "%s (n=%d, cap=%d)" % (name, len(s), cap)
    if want is None:
        assert got is None, "%s: the oracle rejects it (code %d), the GPU decoded %d bytes" % (where, wcode, len(got))
        assert gcode == wcode, "%s: codes %d (GPU) and %d (oracle)" % (where, gcode, wcode)
        return None
    assert got is not None, "%s: the oracle decodes %d bytes, the GPU fails with code %d" % (where, len(want), gcode)
    assert len(got) == len(want), "%s: %d bytes decoded, %d expected" % (where, len(got), len(want))
    if exact and not np.array_equal(got, want):
        k = int(np.argmax(got != want))
        raise AssertionError("%s: first difference at %d (got %d, want %d)" % (where, k, got[k], want[k]))
    return want


def out_len(oracle, t, s, block_size=0):
    try:
        return len(oracle.transform_inverse(t, s, PROBE, block_size=block_size))
    except oracle.OracleError:
        return None


def caps(L, n, lz=False):
    """the cap sweep around the output length L (around the stream length n when the oracle rejects the case at any cap)"""
    L = n if L is None else L
    c = [L - 1, L, L + 1, L + 64] + ([L + 15, L + 16] if lz else [])
    return [x for x in c if x >= 0]


def sweep(gpu, kz, oracle, t, cases, lz=False, block_size=0):
    for case in cases:
        name, s = case[0], case[1]
        cap = case[2] if len(case) > 2 and isinstance(case[2], int) else None
        for c in [cap] if cap is not None else caps(out_len(oracle, t, s, block_size), len(s), lz):
            check_one(gpu, kz, oracle, t, name, s, c, block_size)


# ---- block batches ------------------------------------------------------------------------------------------------------------------

def decode_raw(gpu, t48, payloads, block_size, out_stride):
    """kz_decode_blocks -> (status, out_len, blocks); status is per block, the call's own return code is not looked at"""
    nb = len(payloads)
    blob = np.concatenate([p for p, _ in payloads])
    offs = np.cumsum([0] + [p.size for p, _ in payloads[:-1]]).astype(np.uint64)
    bits = np.array([b for _, b in payloads], np.uint64)
    out = np.zeros(out_stride * nb, np.uint8)
    lens = np.zeros(nb, np.uint32)
    status = np.zeros(nb, np.int32)
    gpu.lib.kz_decode_blocks(gpu.h, t48, 0, 0, blob.ctypes.data, offs.ctypes.data, bits.ctypes.data, nb, block_size, out.ctypes.data, out_stride,
                             lens.ctypes.data, status.ctypes.data)
    return status, lens, [out[b * out_stride: b * out_stride + int(lens[b])] for b in range(nb)]


def block_batch(gpu, kz, oracle, t, cases, block_size=BS, out_stride=None):
    """every case as a one-stage E_NONE record, all in one kz_decode_blocks call, against oracle.decode_block at the same block size.
    Both give the stage len(dst) = bs + max(512, bs >> 4) (Reader.processBlock, CompressedStream.go:1649-1653) as long as no record is
    longer: cases are kept below that, so that the verdicts do not depend on the batch's longest record."""
    room = block_size + max(512, block_size >> 4)
    cases = [c for c in cases if 1 <= len(c[1]) <= room - 64]
    recs = [fs.block_record(c[1]) for c in cases]
    t48 = t << 42
    out_stride = out_stride or block_size + block_size // 2 + 2048
    status, lens, got = decode_raw(gpu, t48, recs, block_size, out_stride)
    verdicts = set()
    for c, (p, bits), st, g in zip(cases, recs, status, got):
        name, s = c[0], c[1]
        try:
            want = oracle.decode_block(p, bits, t48, 0, 0, block_size)
        except oracle.OracleError as e:
            assert st == -e.code, "%s (n=%d): block status %d, the oracle fails with code %d" % (name, len(s), st, e.code)
            verdicts.add(False)
            continue
        verdicts.add(True)
        assert st == 0, "%s (n=%d): block status %d, the oracle decodes %d bytes" % (name, len(s), st, len(want))
        assert len(g) == len(want), "%s: %d bytes decoded, %d expected" % (name, len(g), len(want))
        _, _, exact = oracle_inverse(oracle, t, s, room, block_size)
        assert not exact or np.array_equal(g, want), name
    return verdicts


# ---- ZRLT -------------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def zrlt_cases():
    return fs.zrlt_cases()


def test_zrlt_group_of_23_digits_across_a_tile(gpu, kz, oracle):
    """8,170 ones, then a 23-digit group split 22 | 1 by the first 8 KiB tile boundary: 2^23 - 1 zeros, a valid run in any block above
    8 MiB. The group's head carried into the next tile must not be bounded by a constant"""
    s = fs.zrlt_repro()
    want = np.concatenate([np.ones(8170, np.uint8), np.zeros((1 << 23) - 1, np.uint8)])
    assert np.array_equal(oracle.transform_inverse(fs.T_ZRLT, s, len(want)), want)
    got = gpu.transform_inverse(fs.T_ZRLT, s, len(want) + 64)
    assert len(got) == len(want) and np.array_equal(got, want)


def test_zrlt_16mib_stream_of_a_long_run(gpu, oracle):
    """the same data through -t ZRLT -e NONE at -b 16m: the forward gives the stream above, GPU compress == oracle compress, and the GPU
    decodes the oracle's stream"""
    x = np.concatenate([np.ones(8170, np.uint8), np.zeros((1 << 23) - 1, np.uint8)])
    assert np.array_equal(oracle.transform_forward(fs.T_ZRLT, x)[0], fs.zrlt_repro())
    want = oracle.compress(x, "ZRLT", "NONE", block_size=16 << 20, input_size=len(x))
    got = gpu.compress(x, "ZRLT", "NONE", block_size=16 << 20, input_size=len(x))
    assert np.array_equal(got, want)
    y = gpu.decompress(want, len(x) + 1024)
    assert len(y) == len(x) and np.array_equal(y, x)


def test_zrlt_large_groups(gpu, kz, oracle):
    for name, s, cap in fs.zrlt_large_cases():
        for c in (cap - 65, cap - 64, cap):
            check_one(gpu, kz, oracle, fs.T_ZRLT, name, s, c)


def test_zrlt_cap_sweep(gpu, kz, oracle, zrlt_cases):
    sweep(gpu, kz, oracle, fs.T_ZRLT, zrlt_cases)


def test_zrlt_mutations(gpu, kz, oracle, zrlt_cases):
    sweep(gpu, kz, oracle, fs.T_ZRLT, fs.mutations([c[:2] for c in zrlt_cases if len(c[1]) < 100000], 200, seed=61, head=2))


def test_zrlt_block_batch(gpu, kz, oracle, zrlt_cases):
    assert block_batch(gpu, kz, oracle, fs.T_ZRLT, zrlt_cases[:300]) == {True, False}


def test_zrlt_block_batch_long_block_beside_short_ones(gpu, kz, oracle, zrlt_cases):
    """the 8 MiB run beside short blocks at -b 16m: tiles of every block run at once"""
    cases = [("repro", fs.zrlt_repro())] + [c for c in zrlt_cases if len(c[1]) < 20000][::25]
    block_batch(gpu, kz, oracle, fs.T_ZRLT, cases, block_size=16 << 20, out_stride=9 << 20)


# ---- MM ---------------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def mm_cases():
    return fs.mm_cases()


def test_mm_cap_sweep(gpu, kz, oracle, mm_cases):
    sweep(gpu, kz, oracle, fs.T_MM, mm_cases)


def test_mm_mutations(gpu, kz, oracle, mm_cases):
    sweep(gpu, kz, oracle, fs.T_MM, fs.mutations([c for c in mm_cases if len(c[1]) < 100000], 200, seed=62, head=2))


def test_mm_block_batch(gpu, kz, oracle, mm_cases):
    """every header and escape shape in one batch"""
    assert block_batch(gpu, kz, oracle, fs.T_MM, [c for c in mm_cases if len(c[1]) < 5000]) == {True, False}


# ---- PACK / DNA -------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def alias_cases():
    return fs.alias_cases()


@pytest.mark.parametrize("t", [fs.T_PACK, fs.T_DNA], ids=["PACK", "DNA"])
def test_alias_cap_sweep(gpu, kz, oracle, alias_cases, t):
    sweep(gpu, kz, oracle, t, alias_cases)


@pytest.mark.parametrize("t", [fs.T_PACK, fs.T_DNA], ids=["PACK", "DNA"])
def test_alias_mutations(gpu, kz, oracle, alias_cases, t):
    sweep(gpu, kz, oracle, t, fs.mutations([c[:2] for c in alias_cases if len(c[1]) < 100000], 200, seed=63, head=6))


@pytest.mark.parametrize("t", [fs.T_PACK, fs.T_DNA], ids=["PACK", "DNA"])
def test_alias_block_batch(gpu, kz, oracle, alias_cases, t):
    assert block_batch(gpu, kz, oracle, t, alias_cases) == {True, False}


# ---- LZ / LZX ---------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lz_cases():
    return fs.lz_cases()


def serial_launches(gpu, fn):
    gpu.profile(True)
    gpu.profile_reset()
    try:
        fn()
        return gpu.kernel_time("lz_inverse_serial")[0]
    finally:
        gpu.profile(False)


@pytest.mark.parametrize("t", [fs.T_LZ, fs.T_LZX], ids=["LZ", "LZX"])
def test_lz_cap_sweep(gpu, kz, oracle, lz_cases, t):
    sweep(gpu, kz, oracle, t, lz_cases, lz=True)


def test_lz_parallel_parse_takes_every_encoder_shaped_stream(gpu, kz, oracle, lz_cases):
    """at a generous cap, a stream the parse can take (fs.lz_parallel_shape, and the oracle accepts it) runs without lz_inverse_serial;
    every other stream, every "odd" case among them, goes through it"""
    kept = serial = 0
    for name, s, label in lz_cases:
        L = out_len(oracle, fs.T_LZ, s)
        cap = (L if L is not None else len(s)) + 64
        parallel = L is not None and fs.lz_parallel_shape(s)
        assert label != "shaped" or parallel, name
        assert label != "odd" or not parallel, name
        n = serial_launches(gpu, lambda: check_one(gpu, kz, oracle, fs.T_LZ, name, s, cap))
        assert (n == 0) == parallel, "%s: %d lz_inverse_serial launches, the parse %s take it" % (name, n, "should" if parallel else "cannot")
        kept += parallel
        serial += not parallel
    assert kept >= 30 and serial >= 10


def test_lz_mutations(gpu, kz, oracle, lz_cases):
    sweep(gpu, kz, oracle, fs.T_LZ, fs.mutations([c[:2] for c in lz_cases if len(c[1]) < 100000], 200, seed=64, head=13), lz=True)


def test_lz_block_batch(gpu, kz, oracle, lz_cases):
    mutants = fs.mutations([c[:2] for c in lz_cases if len(c[1]) < 60000], 100, seed=65)
    assert block_batch(gpu, kz, oracle, fs.T_LZ, [c[:2] for c in lz_cases] + mutants) == {True, False}


# ---- TEXT -------------------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def text_cases(oracle):
    return fs.text_cases(oracle)


def test_text_mutations_cap_sweep(gpu, kz, oracle, text_cases):
    """valid TEXT streams and their mutants; some mutants must stay on the parallel path"""
    gpu.set_stream_block_size(fs.TEXT_BS)
    kept = []
    try:
        for name, s in text_cases + fs.mutations(text_cases, 200, seed=66, head=4):
            for c in caps(out_len(oracle, fs.T_TEXT, s, fs.TEXT_BS), len(s)):
                gpu.profile(True)
                gpu.profile_reset()
                try:
                    want = check_one(gpu, kz, oracle, fs.T_TEXT, name, s, c, fs.TEXT_BS)
                    if want is not None and gpu.kernel_time("text_inverse_serial")[0] == 0 and not name.startswith("fwd_"):
                        kept.append(name)
                finally:
                    gpu.profile(False)
    finally:
        gpu.set_stream_block_size(0)
    assert kept, "no mutated TEXT stream stayed on the parallel path"


# ---- whole streams ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tr", ["LZ", "LZX", "MM", "PACK", "DNA", "TEXT"])
def test_whole_stream(gpu, oracle, lz_cases, tr):
    """one stream per stage, from data whose blocks go through the stage: the GPU decodes the oracle's stream"""
    rng = np.random.default_rng(7)
    if tr in ("LZ", "LZX"):
        x = oracle.transform_inverse(fs.T_LZ, dict((c[0], c[1]) for c in lz_cases)["reps_mixed_2000"], PROBE)
    elif tr == "MM":
        ramp = (np.arange(300000) // 3 % 256).astype(np.int64)
        x = ((ramp + rng.integers(-3, 4, ramp.size)) % 256).astype(np.uint8)
    elif tr == "PACK":
        x = rng.choice(np.array([7, 9, 200], np.uint8), 300000)
    elif tr == "DNA":
        x = rng.choice(np.frombuffer(b"ACGT", np.uint8), 300000)
    else:
        x = fs.synth.markov_text(300000, seed=9)
    if tr in ("MM", "PACK", "DNA"):
        assert oracle.transform_forward(fs.TRANSFORMS[tr], x[: 1 << 17])[0] is not None, "the stage declines the data"
    s = oracle.compress(x, tr, "NONE", block_size=1 << 17, input_size=len(x))
    y = gpu.decompress(s, len(x) + 1024)
    assert len(y) == len(x) and np.array_equal(y, x)
