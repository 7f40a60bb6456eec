"""CPU checks of the range decode restated in tests/range_oracle.py (kanzi d --from / --to), against the oracle's full decode: a range is
the matching slice of the full decode for every (from, to) of the grid; a defect inside a skipped block (its header, payload or checksum) is
not an error, the same defect inside the range gives the full decode's code, and a walk error behind the range (truncation) still fails."""
import itertools

import numpy as np
import pytest

import range_oracle as ro

BS = 1024
NBLK = 12
CHAINS = [("DNA+LZ", "HUFFMAN", 0), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN", 0), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE", 0),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0", 0), ("LZ", "HUFFMAN", 0), ("NONE", "NONE", 32), ("NONE", "NONE", 64)]
IDS = ["%s-%s-x%d" % c for c in CHAINS]
GRID = [-1, 0, 1, 2, NBLK - 1, NBLK, NBLK + 1]


def stream_of(oracle, synth, chain, seed=5):
    tr, en, ck = chain
    x = np.ascontiguousarray(synth.markov_text(NBLK * BS - 300, seed=seed), np.uint8)
    return x, oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=len(x))


def expected_slice(x, frm, to):
    blocks = [x[i: i + BS] for i in range(0, len(x), BS)]
    keep = [b for i, b in enumerate(blocks) if ro.in_range(i + 1, frm, to)]
    return np.concatenate(keep) if keep else np.zeros(0, np.uint8)


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_range_is_the_slice_of_the_full_decode(oracle, synth, chain):
    x, s = stream_of(oracle, synth, chain)
    full = oracle.decompress(s, len(x) + 64)
    assert np.array_equal(full, x)
    assert np.array_equal(ro.decompress_range(oracle, s), x)
    assert len(ro.walk(s, ro.header_bits(s))) == NBLK
    for frm, to in itertools.product(GRID, GRID):
        got = ro.decompress_range(oracle, s, frm, to)
        assert np.array_equal(got, expected_slice(x, frm, to)), (frm, to)
    assert len(ro.decompress_range(oracle, s, -1, 1)) == 0
    assert len(ro.decompress_range(oracle, s, 7, 3)) == 0


@pytest.mark.parametrize("chain", [CHAINS[3], CHAINS[5]], ids=[IDS[3], IDS[5]])
def test_defects_in_skipped_blocks_are_not_errors(oracle, synth, chain):
    x, s = stream_of(oracle, synth, chain, seed=9)
    recs = ro.walk(s, ro.header_bits(s))
    kinds = ["header", "payload"] + (["checksum"] if chain[2] else [])
    for kind, victim in itertools.product(kinds, (0, 5, NBLK - 1)):
        bad = ro.corrupt(s, recs[victim], kind)
        full = ro.outcome(oracle.decompress, bad, len(x) + 64)
        if kind != "payload":
            assert full[0] == "err", (kind, victim)
        vid = victim + 1
        # the defective block outside the range: the range decodes
        for frm, to in ((vid + 1, -1), (-1, vid), (vid + 1, vid + 3), (1, vid)):
            if ro.in_range(vid, frm, to):
                continue
            assert np.array_equal(ro.decompress_range(oracle, bad, frm, to), expected_slice(x, frm, to)), (kind, victim, frm, to)
        # inside the range: the full decode's outcome (for a payload defect without checksums that may be wrong bytes, not an error)
        got = ro.outcome(ro.decompress_range, oracle, bad, vid, vid + 1)
        if full[0] == "err":
            assert got == full, (kind, victim, got, full)
        else:
            assert got[0] == "ok"


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_walk_errors_behind_the_range_still_fail(oracle, synth, chain):
    x, s = stream_of(oracle, synth, chain, seed=11)
    recs = ro.walk(s, ro.header_bits(s))
    for cut in (len(s) - 1, (recs[-1][0] + recs[-1][1] // 2) // 8, (recs[6][0] + 3) // 8):
        t = s[:cut]
        full = ro.outcome(oracle.decompress, t, len(x) + 64)
        assert full[0] == "err"
        for frm, to in ((1, 2), (2, 4), (-1, 1), (NBLK + 1, -1)):
            assert ro.outcome(ro.decompress_range, oracle, t, frm, to) == full, (cut, frm, to)
    # the end marker's 5-bit lw rewritten to 34 bits: the length it announces runs past the end of the stream
    big = ro.flip(s, recs[-1][0] + recs[-1][1], 5)
    full = ro.outcome(oracle.decompress, big, len(x) + 64)
    assert full[0] == "err"
    assert ro.outcome(ro.decompress_range, oracle, big, 1, 2) == full
