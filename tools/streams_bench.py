"""Cost of one stream call versus one batched call over many small files.

Builds a seeded corpus by cutting synth.silesia_shaped into --files files with log-normal sizes (median 16 KiB, clipped at 4 MiB), and for
each level times two arms on one context:
  single  = one kz_compress_stream + one kz_decompress_stream per file (Context.compress / Context.decompress);
  batched = one kz_compress_streams + one kz_decompress_streams call over all files (Context.compress_streams / decompress_streams).
Both arms go through the host-buffer entry points and their Python wrappers. It checks that both arms produce identical streams and that
both decode to the input, and prints one JSON line per level with files/s, MB/s (input bytes over wall time, ending in a device
synchronise) and kernel launches per arm, next to the card's name and power limit read in the same run.

    python tools/streams_bench.py [--files 20000] [--levels l3,l5] [--out FILE]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
kz = importlib.import_module("kanzi-go_b200")
synth = importlib.import_module("kanzi-go_b200.synth")

LEVELS = {"l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")}
BLOCK = 4 << 20  # kanzi's default block size


def corpus(nfiles, seed):
    rng = np.random.default_rng(seed)
    sizes = np.exp(rng.normal(np.log(16384), 1.3, nfiles)).clip(0, 4 << 20).astype(np.int64)
    slab = synth.silesia_shaped(int(sizes.sum()), seed=seed)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    return [slab[offs[i]: offs[i + 1]] for i in range(nfiles)]


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "not read"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=20000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--levels", default="l3,l5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    files = corpus(a.files, a.seed)
    total = sum(len(f) for f in files)
    name, pl = card()
    ctx = kz.Context(0)
    lines = []
    for lv in a.levels.split(","):
        tr, en = LEVELS[lv]
        caps = [len(f) for f in files]
        # warm-up of both arms (module loads, scratch growth)
        for f in files[:32]:
            ctx.decompress(ctx.compress(f, tr, en, BLOCK), len(f) + 1)
        w, _ = ctx.compress_streams(files[:256], tr, en, BLOCK)
        ctx.decompress_streams(w, caps[:256])
        ctx.launch_count(reset=True)
        t0 = time.perf_counter()
        single = [ctx.compress(f, tr, en, BLOCK) for f in files]
        t1 = time.perf_counter()
        single_dec = [ctx.decompress(s, c) for s, c in zip(single, caps)]
        t2 = time.perf_counter()
        l_single = ctx.launch_count(reset=True)
        batched, st = ctx.compress_streams(files, tr, en, BLOCK)
        t3 = time.perf_counter()
        batched_dec, st2 = ctx.decompress_streams(batched, caps)
        t4 = time.perf_counter()
        l_batched = ctx.launch_count(reset=True)
        assert (st == 0).all() and (st2 == 0).all()
        same = all(np.array_equal(x, y) for x, y in zip(single, batched))
        decoded = all(np.array_equal(x, f) and np.array_equal(y, f) for x, y, f in zip(single_dec, batched_dec, files))
        cbytes = sum(len(s) for s in batched)

        def arm(tc, td, launches):
            return {"compress_s": tc, "decompress_s": td, "compress_files_per_s": len(files) / tc, "decompress_files_per_s": len(files) / td,
                    "compress_MB_per_s": total / tc / 1e6, "decompress_MB_per_s": total / td / 1e6, "launches": int(launches)}

        line = {"tool": "streams_bench", "level": lv, "transform": tr, "entropy": en, "block_size": BLOCK, "files": len(files), "input_bytes": total,
                "compressed_bytes": cbytes, "median_file_bytes": int(np.median([len(f) for f in files])), "largest_file_bytes": max(len(f) for f in files),
                "single": arm(t1 - t0, t2 - t1, l_single), "batched": arm(t3 - t2, t4 - t3, l_batched), "identical_streams": same,
                "round_trip_ok": decoded, "gpu": name, "power_limit": pl}
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
