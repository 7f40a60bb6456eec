"""kz_decode_blocks on batches with corrupt blocks. The call goes through ctypes, so that status / out_len can be read after a failure.
Every block's fixture is the oracle's record (oracle.encode_block); a fault is one corrupted field of it, or an out_stride too small."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BS = 1 << 16
N = 20000  # bytes per block
SENTINEL = 0x5A5A5A5A


def _fields(p):
    """(offset of the length bytes, their count, offset of the checksum) of a block record (encodingTask.encode :836-887)"""
    mode = int(p[0])
    at = 2 if not mode & 0x80 and mode & 0x10 else 1
    size = ((mode >> 5) & 3) + 1
    return at, size, at + size


def corrupt(p, bits, fault, ck):
    """-> (payload, bits) with the fault applied"""
    p = p.copy()
    at, size, ck_at = _fields(p)
    if fault == "header":  # a block length of 0
        p[at: at + size] = 0
    elif fault == "entropy":  # the record ends 64 bits early: the NONE codec runs out of data
        bits -= 64
    elif fault == "inverse":  # every primary index of the BWT header (behind the block header, NONE codec) past the block's end
        d = ck_at + ck // 8
        p[d + 1: d + 1 + 8 * ((int(p[d]) & 3) + 1)] = 0xFF
    elif fault == "checksum":
        p[ck_at] ^= 0x01
    return p, bits


def decode_raw(gpu, t48, et, ck, payloads, out_stride):
    """kz_decode_blocks -> (return code, status, out_len, decoded blocks); status and out_len start as a sentinel"""
    nb = len(payloads)
    blob = np.concatenate([p for p, _ in payloads])
    offs = np.cumsum([0] + [p.size for p, _ in payloads[:-1]]).astype(np.uint64)
    bits = np.array([b for _, b in payloads], np.uint64)
    out = np.zeros(out_stride * nb, np.uint8)
    out_len = np.full(nb, SENTINEL, np.uint32)
    status = np.full(nb, SENTINEL, np.int32)
    rc = gpu.lib.kz_decode_blocks(gpu.h, t48, et, ck, blob.ctypes.data, offs.ctypes.data, bits.ctypes.data, nb, BS, out.ctypes.data,
                                  out_stride, out_len.ctypes.data, status.ctypes.data)
    return rc, status, out_len, [out[b * out_stride: b * out_stride + int(out_len[b])] for b in range(nb)]


def batch(oracle, synth, chain, lens, seed):
    """blocks of lens[i] bytes and their records"""
    tr, en, ck = chain
    xs = [synth.markov_text(n, seed=seed + i) for i, n in enumerate(lens)]
    return xs, [oracle.encode_block(x, oracle.parse_transform(tr), oracle.parse_entropy(en), checksum_bits=ck) for x in xs]


# (fault, chain, expected code): one of each failure of a block; "out_stride" is a good block in too small an output slot
FAULTS = [
    ("header", ("BWT", "ANS0", 32), 2),  # ERR_BLOCK_SIZE
    ("header", ("NONE", "ANS0", 0), 2),
    ("entropy", ("BWT", "NONE", 0), 13),  # ERR_PROCESS_BLOCK
    ("inverse", ("BWT", "NONE", 0), 13),
    ("checksum", ("BWT", "ANS0", 32), 19),  # ERR_CRC_CHECK
    ("checksum", ("NONE", "NONE", 64), 19),
    ("out_stride", ("BWT", "ANS0", 0), 12),  # ERR_WRITE_FILE
    ("out_stride", ("NONE", "ANS0", 32), 12),
]
IDS = ["%s-%s-%s-%d" % (f, *c) for f, c, _ in FAULTS]


def faulty_batch(oracle, synth, fault, chain):
    """good, faulty, good, the good blocks shorter: (blocks, records, out_stride)"""
    tr, en, ck = chain
    xs, recs = batch(oracle, synth, chain, [N // 4, N, N // 4], seed=70)
    out_stride = N // 2 if fault == "out_stride" else BS + BS // 2 + 2048
    recs[1] = corrupt(*recs[1], fault, ck)
    t48, et = oracle.parse_transform(tr), oracle.parse_entropy(en)
    if fault == "out_stride":
        assert len(oracle.decode_block(*recs[1], t48, et, ck, BS)) > out_stride
    else:
        with pytest.raises(oracle.OracleError):
            oracle.decode_block(*recs[1], t48, et, ck, BS)
    return xs, recs, out_stride


@pytest.mark.parametrize("fault,chain,code", FAULTS, ids=IDS)
def test_one_failing_block_gives_its_code(gpu, oracle, synth, fault, chain, code):
    tr, en, ck = chain
    _, recs, out_stride = faulty_batch(oracle, synth, fault, chain)
    rc, _, _, _ = decode_raw(gpu, oracle.parse_transform(tr), oracle.parse_entropy(en), ck, recs, out_stride)
    assert rc == -code


@pytest.mark.parametrize("fault,chain,code", FAULTS, ids=IDS)
def test_every_status_is_written_and_good_blocks_decode(gpu, oracle, synth, fault, chain, code):
    tr, en, ck = chain
    xs, recs, out_stride = faulty_batch(oracle, synth, fault, chain)
    rc, status, out_len, got = decode_raw(gpu, oracle.parse_transform(tr), oracle.parse_entropy(en), ck, recs, out_stride)
    assert rc == -code
    assert list(status) == [0, -code, 0]
    assert out_len[1] == 0
    for b in (0, 2):
        assert out_len[b] == N // 4 and np.array_equal(got[b], xs[b]), b


def test_mixed_batch_reports_the_first_failing_block(gpu, oracle, synth):
    """good, checksum mismatch, good, bad header, good on BWT+ANS0: every status is the code of that block decoded alone, the good blocks
    decode to the oracle's bytes, and the call returns the first failing block's code"""
    chain = ("BWT", "ANS0", 32)
    tr, en, ck = chain
    t48, et = oracle.parse_transform(tr), oracle.parse_entropy(en)
    xs, recs = batch(oracle, synth, chain, [N] * 5, seed=90)
    recs[1] = corrupt(*recs[1], "checksum", ck)
    recs[3] = corrupt(*recs[3], "header", ck)
    out_stride = BS + BS // 2 + 2048
    rc, status, out_len, got = decode_raw(gpu, t48, et, ck, recs, out_stride)
    assert rc == -19
    alone = [decode_raw(gpu, t48, et, ck, [r], out_stride)[0] for r in recs]
    assert alone == [0, -19, 0, -2, 0]
    assert list(status) == alone
    for b in (0, 2, 4):
        want = oracle.decode_block(*recs[b], t48, et, ck, BS)
        assert np.array_equal(want, xs[b]) and out_len[b] == N and np.array_equal(got[b], want), b
    assert out_len[1] == 0 and out_len[3] == 0
