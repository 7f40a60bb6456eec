"""TEST INFRASTRUCTURE ONLY. Rank streams for the RANK / MTFT inverse (kz_sbrt.cu), shared by the CPU model tests and the GPU tests.

SBRT is a bijection on byte strings: every byte string R is the forward of exactly one D, D = oracle.transform_inverse(T, R, n). So the
inverse can be driven with the rank sequences that stress its kernels instead of the ones natural data happens to produce: deep ranks, moves
across the warp boundaries of sbrt_inverse_multi_kernel (list entries 64 / 128 / 192; 2 entries per lane) and the lane boundaries of
sbrt_inverse_warp_kernel (8 entries per lane), equal q in RANK mode, and zero runs at every offset of a 32-rank round.
"""
import importlib

import numpy as np

synth = importlib.import_module("kanzi-go_b200.synth")

MIB = 1 << 20
CONST_RANKS = (0, 1, 2, 7, 8, 31, 32, 63, 64, 65, 127, 128, 191, 192, 254, 255)
# r, r + 1 alternating: the warp boundaries of the 4-warp kernel (63/64, 127/128, 191/192), its lane boundaries (2 entries per lane: 1/2,
# 31/32) and those of the warp kernel (8 entries per lane: 7/8, 15/16)
ALT_PAIRS = ((63, 64), (127, 128), (191, 192), (1, 2), (31, 32), (7, 8), (15, 16))
LENGTHS = tuple(range(1, 41)) + (63, 64, 65, 95, 96, 97, 4095, 4096, 4097, 100003)


def _zero_runs(n, rng):
    """zero runs of every length 1 .. 70, each starting at every offset mod 32 in turn, between nonzero ranks (small and deep)"""
    r = rng.integers(1, 256, n).astype(np.uint8)
    pos, k = 1, 0
    while pos < n:
        length, off = 1 + k % 70, (k // 70 + k) % 32
        start = pos + (off - pos) % 32
        if start >= n:
            break
        r[start: start + length] = 0
        pos, k = start + length + 1, k + 1
    return r


def _aligned_32(n, rng):
    """runs of exactly 32 zeros on round boundaries, one nonzero rank between them every other round"""
    r = np.zeros(n, np.uint8)
    i = np.arange(n)
    r[(i // 32) % 2 == 1] = rng.integers(1, 256, int(np.count_nonzero((i // 32) % 2 == 1)))
    return r


def _run_to_end(n, rng):
    r = rng.integers(1, 256, n).astype(np.uint8)
    r[n - min(n, 45 + n % 32):] = 0
    return r


def _forward(ttype, oracle, x):
    if len(x) == 0:
        return x
    f, _ = oracle.transform_forward(ttype, x)
    return f


def rank_streams(n, ttype, oracle, seed=0):
    """-> [(name, R)] of n ranks each. ttype selects the forward used by the cases taken from real data (R depends on the mode there)."""
    rng = np.random.default_rng(seed * 1000003 + n)
    i = np.arange(n)
    out = [("const%d" % c, np.full(n, c, np.uint8)) for c in CONST_RANKS]
    out += [("alt%d_%d" % (a, b), np.where(i % 2 == 0, a, b).astype(np.uint8)) for a, b in ALT_PAIRS]
    out += [
        ("ramp_up", (i % 256).astype(np.uint8)),                    # r2 == r + 1
        ("ramp_down", (255 - i % 256).astype(np.uint8)),            # r2 == r - 1
        ("ramp_pairs", ((i // 2) % 256).astype(np.uint8)),          # r2 == r, then r2 == r + 1
        ("sawtooth", np.abs((i * 7) % 140 - 70).astype(np.uint8) * 3 + (i % 3).astype(np.uint8)),  # triangle of step 21 with jitter
        ("uniform", rng.integers(0, 256, n).astype(np.uint8)),
        ("below3", rng.integers(0, 3, n).astype(np.uint8)),
        ("small_deep", np.where(rng.random(n) < 0.85, rng.integers(0, 8, n), rng.integers(8, 256, n)).astype(np.uint8)),
        ("zero_runs", _zero_runs(n, rng)),
        ("zero_32", _aligned_32(n, rng)),
        ("zero_to_end", _run_to_end(n, rng)),
        ("bwt_text", _forward(ttype, oracle, oracle.bwt_forward_raw(synth.markov_text(n, seed=n))[0])),  # what RANK sees in kanzi -l 5
        ("abc", _forward(ttype, oracle, rng.integers(0, 3, n).astype(np.uint8))),  # 3 symbols: equal q all the time in RANK mode
    ]
    assert all(len(r) == n for _, r in out)
    return [(name, np.ascontiguousarray(r, np.uint8)) for name, r in out]


def corpus(ttype, oracle, lengths=LENGTHS):
    """[(name, R)] over every length; name carries the length"""
    return [("%s/n=%d" % (name, n), r) for n in lengths for name, r in rank_streams(n, ttype, oracle)]


def expected(ttype, oracle, r):
    """the data whose forward is r; up to 1 MiB the forward is checked to give r back"""
    d = oracle.transform_inverse(ttype, r, len(r))
    assert len(d) == len(r)
    if len(r) <= MIB:
        f = _forward(ttype, oracle, d)
        assert np.array_equal(f, r), "the oracle's forward does not give the rank stream back"
    return d


def first_difference(name, mode, r, got, want):
    """the message of a mismatch: case, mode, the first differing position and the ranks just before it"""
    got = np.asarray(got)
    if len(got) != len(want):
        return "%s %s: %d bytes decoded, %d expected" % (name, mode, len(got), len(want))
    k = int(np.argmax(got != want))
    return "%s %s: first difference at %d of %d (got %d, want %d), ranks %d..%d: %s" % (
        name, mode, k, len(want), got[k], want[k], max(0, k - 8), k, np.asarray(r[max(0, k - 8): k + 1]).tolist())


def warp_events(r):
    """what sbrt_inverse_warp_kernel (rounds of 32 ranks, zero runs in one step, ranks < 8 on lane 0) meets in r, counted from r alone"""
    r = np.asarray(r)
    n = len(r)
    ev = dict(run_crosses_round=0, round_of_32_zeros=0, run_ends_block=0, run_of_1_continues=0, small_then_deep=0)
    if n == 0:
        return ev
    z = r == 0
    starts = np.flatnonzero(z & ~np.concatenate(([False], z[:-1])))
    ends = np.flatnonzero(z & ~np.concatenate((z[1:], [False]))) + 1  # exclusive
    ev["run_crosses_round"] = int(np.count_nonzero(starts // 32 != (ends - 1) // 32))
    full = n // 32
    ev["round_of_32_zeros"] = int(np.count_nonzero(z[: 32 * full].reshape(full, 32).all(axis=1))) if full else 0
    ev["run_ends_block"] = int(z[-1])
    # a round opening with a zero that continues the previous round's run, and the next rank nonzero (or the end): L == 1 at j == 0
    k = np.arange(32, n, 32)
    nxt = np.append(z, False)[k + 1]
    ev["run_of_1_continues"] = int(np.count_nonzero(z[k] & z[k - 1] & ~nxt))
    ev["small_then_deep"] = int(np.count_nonzero((r[:-1] > 0) & (r[:-1] < 8) & (r[1:] >= 8)))
    return ev
