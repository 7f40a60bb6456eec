"""Round profile of the BWT forward's prefix doubling on the input the BWT stage sees in bench.py's -l 5 encode.

The silesia-shaped slab of bench.py (same size and seed) is cut into 4 MiB blocks and every block goes through the oracle's TEXT and UTF
forward (the stages in front of BWT at -l 5). Then:

  CPU (always): a numpy model of the rounds exactly as bwt_forward_batch runs them (first key = block index + 6 symbols, h = 6, 12, 24, ...,
      second key 0 past the end of the block, stop when no group is left or h >= 2 x the largest block). Per round: m (members of
      unresolved groups), the number of groups, a histogram of group sizes, the members in groups of at most BWT_SMALL_GROUP, and the width of
      the narrow key of the large groups.
  --gpu: bwt_forward over the same batch on cuda:0 with every round timed by CUDA events (kz_bwt_profile), once with the rounds of the
      build (small groups on chip, narrow keys) and once forced onto the 56-bit global sort of every round; per round the sort, the
      small-group pass, the bookkeeping around the global sort, the selects and the host synchronisation gaps, in ms per call.

    python tools/bwt_rounds.py [--mb 200] [--gpu] [--reps 5]
"""
import argparse
import importlib
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

synth = importlib.import_module("kanzi-go_b200.synth")
SMALL_GROUP = 256  # BWT_SMALL_GROUP of kanzi-go_b200/csrc/kz_bwt_core.cuh
BINS = [(2, 2), (3, 8), (9, 64), (65, 2048), (2049, None)]


def stage_input(mb, block=4 << 20):
    from oracle import pyoracle as po

    po.build()
    x = synth.silesia_shaped(int(mb * 1_000_000), seed=synth.SEED + 1)  # bench.py: make_data(kind, n, synth.SEED + 1)
    blocks = []
    for o in range(0, len(x), block):
        b = x[o: o + block]
        dt = 0
        for t in (po.T_TEXT, po.T_UTF):
            out, dt = po.transform_forward(t, b, dt, block_size=block)
            if out is not None:
                b = out
        blocks.append(np.ascontiguousarray(b, np.uint8))
    return blocks


def bits_for(v):
    return int(v).bit_length()


def model(blocks):
    """numpy restatement of bwt_forward_batch's rounds; returns one dict per round"""
    n = np.array([len(b) for b in blocks], np.int64)
    base = np.concatenate([[0], np.cumsum(n)[:-1]])
    total, max_n = int(n.sum()), int(n.max())
    data = np.concatenate(blocks).astype(np.uint64)
    blk = np.repeat(np.arange(len(blocks)), n)
    end = (base + n)[blk]
    idx = np.arange(total, dtype=np.int64)
    key = blk.astype(np.uint64)
    for j in range(6):
        p = idx + j
        ok = p < end
        sym = np.zeros(total, np.uint64)
        sym[ok] = data[p[ok]] + 1
        key = (key << np.uint64(9)) | sym
    sa = np.argsort(key, kind="stable")
    sk = key[sa]
    start = np.ones(total, bool)
    start[1:] = sk[1:] != sk[:-1]
    g = np.maximum.accumulate(np.where(start, idx, 0))
    rank = np.empty(total, np.int64)
    rank[sa] = g
    rounds = [dict(round=0, h=0, m=total, groups=int(start.sum()), hist=None, small=0, bits=64)]
    if (g == idx).all() or 6 >= max_n:
        return rounds
    nxt = np.append(g[1:], -1)
    cpos = np.nonzero((g != idx) | (nxt == g))[0]
    h = 6
    for r in range(1, 48):
        m = len(cpos)
        if m == 0:
            break
        v = sa[cpos]
        hd = rank[v]
        b = blk[v]
        ok = v + h < end[v]
        r2 = np.zeros(m, np.int64)
        r2[ok] = rank[v[ok] + h] - base[b[ok]] + 1
        st = np.nonzero(cpos == hd)[0]
        sizes = np.diff(np.append(st, m))
        hist = [int(((sizes >= a) & (True if z is None else sizes <= z)).sum()) for a, z in BINS]
        small = int(sizes[sizes <= SMALL_GROUP].sum())
        nlarge = int((sizes > SMALL_GROUP).sum())
        ml = m - small
        bits = (bits_for(ml // (SMALL_GROUP + 1) - 1) if ml else 0) + bits_for(max_n)
        rounds.append(dict(round=r, h=h, m=m, groups=len(st), hist=hist, small=small, large_groups=nlarge, bits=bits))
        k2 = (hd << 32) | r2
        o = np.argsort(k2, kind="stable")
        ks = k2[o]
        ns = np.ones(m, bool)
        ns[1:] = ks[1:] != ks[:-1]
        gg = np.maximum.accumulate(np.where(ns, cpos, 0))
        sv = v[o]
        sa[cpos] = sv
        rank[sv] = gg
        h *= 2
        if h >= 2 * max_n:
            break
        nx = np.append(gg[1:], -1)
        cpos = cpos[(gg != cpos) | (nx == gg)]
    return rounds


def print_model(rounds, blocks):
    sizes = [len(b) for b in blocks]
    print(f"stage input: {len(blocks)} blocks, {sum(sizes):,} bytes, largest {max(sizes):,}")
    print("round      h            m     groups        2      3-8     9-64  65-2048    >2048   in <=G (%)  large  key bits")
    for d in rounds:
        if d["hist"] is None:
            print(f"{d['round']:5d} {d['h']:6d} {d['m']:12,d} {d['groups']:10,d}   (first sort: every position, 64-bit key)")
            continue
        hs = " ".join(f"{c:8,d}" for c in d["hist"])
        pct = 100.0 * d["small"] / d["m"]
        print(f"{d['round']:5d} {d['h']:6d} {d['m']:12,d} {d['groups']:10,d} {hs}   {pct:9.1f}  {d['large_groups']:5d}  {d['bits']:8d}")


def gpu_profile(blocks, reps):
    kz = importlib.import_module("kanzi-go_b200")
    ctx = kz.Context(0)
    t48 = kz.transform_type("BWT")
    out = {}
    for label, wide in (("small groups on chip + narrow keys", False), ("56-bit global sort every round", True)):
        ctx.bwt_profile(time_rounds=True, wide_rounds=wide)
        ctx.profile(True)
        ctx.encode_blocks(t48, kz.E_NONE, blocks)  # warm-up
        ctx.profile_reset()
        launches0 = ctx.launch_count()
        for _ in range(reps):
            ctx.encode_blocks(t48, kz.E_NONE, blocks)
        launches = (ctx.launch_count() - launches0) / reps
        names = ctx.profile_names()
        per = {}
        for nm in names:
            if nm.startswith("bwt_round:"):
                _, r, part = nm.split(":")
                per.setdefault(int(r), {})[part] = ctx.kernel_time(nm)[1] / reps
        total = ctx.kernel_time("bwt_forward")[1] / reps
        out[label] = (total, per, launches)
        ctx.profile(False)
    ctx.bwt_profile()
    for label, (total, per, launches) in out.items():
        print(f"\nbwt_forward {total:.2f} ms per call ({label}; launches per call incl. the timing scopes: {launches:.0f})")
        print("round    sort   small   large  select     gap    (ms per call)")
        sums = {}
        for r in sorted(per):
            p = per[r]
            row = [p.get(k, 0.0) for k in ("sort", "small", "large", "select", "gap")]
            for k, x in zip(("sort", "small", "large", "select", "gap"), row):
                sums[k] = sums.get(k, 0.0) + x
            print(f"{r:5d} " + " ".join(f"{x:7.2f}" for x in row))
        print("  sum " + " ".join(f"{sums.get(k, 0.0):7.2f}" for k in ("sort", "small", "large", "select", "gap")))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--mb", type=float, default=200.0, help="slab size in MB (bench.py: 200)")
    ap.add_argument("--gpu", action="store_true", help="time the rounds on cuda:0 as well")
    ap.add_argument("--no-model", action="store_true", help="skip the CPU model")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    t0 = time.time()
    blocks = stage_input(a.mb)
    print(f"# TEXT + UTF forward (oracle): {time.time() - t0:.1f} s", flush=True)
    if not a.no_model:
        t0 = time.time()
        print_model(model(blocks), blocks)
        print(f"# model: {time.time() - t0:.1f} s", flush=True)
    if a.gpu:
        gpu_profile(blocks, a.reps)


if __name__ == "__main__":
    main()
