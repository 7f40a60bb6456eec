"""Cost of kanzi's `-b auto` over many files: one call per block size against one call for all files.

With `-b auto` BlockCompressor gives every file the block size size / jobs, rounded up to 64 and clamped to [1 KiB, 1 GiB]
(app/BlockCompressor.go:574-580; kz.auto_block_size). Takes the corpus of tools/streams_bench.py (its corpus(nfiles, seed)), gives each
file its auto block size for --jobs, and for each level times two arms on one context:
  per-size = what a caller of kz_compress_streams has to do: one call per distinct block size, and one kz_decompress_streams call over the
             streams of each block size;
  one-call = one kz_compress_streams_bs call and one kz_decompress_streams call over all files.
Both go through the host-buffer entry points and their Python wrappers. Each arm is first run once over all files, so that both time
their steady state (module loads, scratch and staging grown to full size); then the arms run --reps times each, alternating. It checks
that both arms give identical streams and that both decode to the input, and prints one JSON line per level with the number of distinct
block sizes, and per arm the median and the range over the repeats of files/s and MB/s (input bytes over wall time, ending in a device
synchronise) and the kernel launches, next to the card's name and power limit read in the same run.

    python tools/auto_block_bench.py [--files 20000] [--jobs 16] [--levels l3,l5] [--reps 3] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
kz = importlib.import_module("kanzi-go_b200")
from streams_bench import LEVELS, card, corpus  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=20000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--jobs", type=int, default=16)
    ap.add_argument("--levels", default="l3,l5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    files = corpus(a.files, a.seed)
    bs = [kz.auto_block_size(len(f), a.jobs) for f in files]
    by_size = defaultdict(list)
    for i, b in enumerate(bs):
        by_size[b].append(i)
    total = sum(len(f) for f in files)
    caps = [len(f) for f in files]
    name, pl = card()
    ctx = kz.Context(0)
    lines = []
    for lv in a.levels.split(","):
        tr, en = LEVELS[lv]

        def per_size():
            per, dec = [None] * len(files), [None] * len(files)
            t0 = time.perf_counter()
            for b, idx in by_size.items():
                outs, st = ctx.compress_streams([files[i] for i in idx], tr, en, b)
                assert (st == 0).all()
                for i, o in zip(idx, outs):
                    per[i] = o
            t1 = time.perf_counter()
            for b, idx in by_size.items():
                ys, st = ctx.decompress_streams([per[i] for i in idx], [caps[i] for i in idx])
                assert (st == 0).all()
                for i, y in zip(idx, ys):
                    dec[i] = y
            return per, dec, t1 - t0, time.perf_counter() - t1

        def one_call():
            t0 = time.perf_counter()
            one, st = ctx.compress_streams(files, tr, en, bs)
            t1 = time.perf_counter()
            dec, st2 = ctx.decompress_streams(one, caps)
            assert (st == 0).all() and (st2 == 0).all()
            return one, dec, t1 - t0, time.perf_counter() - t1

        arms = {"per_size": per_size, "one_call": one_call}
        res = {k: {"compress_s": [], "decompress_s": [], "launches": 0} for k in arms}
        got = {k: f() for k, f in arms.items()}  # warm-up at full size
        for _ in range(a.reps):
            for k, f in arms.items():
                ctx.launch_count(reset=True)
                got[k] = f()
                res[k]["launches"] = ctx.launch_count(reset=True)
                res[k]["compress_s"].append(got[k][2])
                res[k]["decompress_s"].append(got[k][3])
        same = all(np.array_equal(x, y) for x, y in zip(got["per_size"][0], got["one_call"][0]))
        decoded = all(np.array_equal(x, f) and np.array_equal(y, f) for x, y, f in zip(got["per_size"][1], got["one_call"][1], files))

        def arm(r):
            out = {"launches": int(r["launches"])}
            for d in ("compress", "decompress"):
                t = sorted(r[d + "_s"])
                out[d + "_s"] = t
                out[d + "_files_per_s"] = {"median": len(files) / t[len(t) // 2], "min": len(files) / t[-1], "max": len(files) / t[0]}
                out[d + "_MB_per_s"] = {"median": total / t[len(t) // 2] / 1e6, "min": total / t[-1] / 1e6, "max": total / t[0] / 1e6}
            return out

        line = {"tool": "auto_block_bench", "level": lv, "transform": tr, "entropy": en, "jobs": a.jobs, "files": len(files),
                "distinct_block_sizes": len(by_size), "input_bytes": total, "compressed_bytes": sum(len(s) for s in got["one_call"][0]),
                "median_file_bytes": int(np.median(caps)), "largest_file_bytes": max(caps), "reps": a.reps,
                "per_size": arm(res["per_size"]), "one_call": arm(res["one_call"]), "identical_streams": same, "round_trip_ok": decoded,
                "gpu": name, "power_limit": pl}
        print(json.dumps(line), flush=True)
        lines.append(line)
        assert same and decoded
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
