"""Bytes and files/s of the many-small-files call with and without stream headers (kz_set_headerless_writer / kz_set_headerless_reader).

Uses the corpus of tools/streams_bench.py (--files files with log-normal sizes, median 16 KiB, clipped at 4 MiB, cut from
synth.silesia_shaped) and, for each level, compresses every file as a stream of its own with its size given (fileSize, as
BlockCompressor passes it), so that every header is 160 bits plus 16 / 32 / 48 size bits: whole bytes, and a headerless stream is its
headered stream without its first header-length bytes.

    python tools/headerless_bytes.py [--files 20000] [--levels l3,l5] [--out FILE]           # on a GPU: bytes and files/s
    python tools/headerless_bytes.py --oracle [--jobs 8] [--files 20000] [--levels l3,l5]   # no GPU: bytes from the CPU oracle

GPU mode times one kz_compress_streams and one kz_decompress_streams call over all files each way (headered, then headerless; median of
--reps runs after a warm-up, wall time ending in a device synchronise), checks that every headerless stream is its headered stream without
the header and that both decode to the input, and prints one JSON line per level next to the card's name and power limit read in the same
run. Oracle mode prints the byte counts only; its rates are null.
"""
import argparse
import importlib
import json
import os
import statistics
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
kz = importlib.import_module("kanzi-go_b200")
from streams_bench import BLOCK, LEVELS, card, corpus  # noqa: E402


def header_bytes(n):
    """Writer.writeHeader's length for a stream with fileSize n: 160 bits and 0 / 16 / 32 / 48 size bits (io/CompressedStream.go:429-519)"""
    return (160 + (0 if n <= 0 or n >= 1 << 48 else 48 if n >= 1 << 32 else 32 if n >= 1 << 16 else 16)) // 8


def _oracle_len(args):
    f, tr, en = args
    from oracle import pyoracle

    return len(pyoracle.compress(f, tr, en, BLOCK, 0, input_size=len(f)))


def oracle_level(files, tr, en, jobs):
    from oracle import pyoracle

    pyoracle.build()
    with ProcessPoolExecutor(jobs) as ex:
        return list(ex.map(_oracle_len, [(f, tr, en) for f in files], chunksize=16))


def timed(ctx, fn, reps):
    import torch

    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, statistics.median(ts)


def gpu_level(ctx, files, tr, en, reps):
    caps = [len(f) for f in files]
    sizes = np.array(caps, np.int64)
    hl = dict(transform=tr, entropy=en, block_size=BLOCK, checksum_bits=0)
    for headerless in (False, True):  # warm-up (module loads, scratch growth)
        w, _ = ctx.compress_streams(files[:256], tr, en, BLOCK, input_sizes=sizes[:256], headerless=headerless)
        ctx.decompress_streams(w, caps[:256], headerless=hl if headerless else None)
    (h, st1), tc_h = timed(ctx, lambda: ctx.compress_streams(files, tr, en, BLOCK, input_sizes=sizes), reps)
    (d_h, st2), td_h = timed(ctx, lambda: ctx.decompress_streams(h, caps), reps)
    (n, st3), tc_n = timed(ctx, lambda: ctx.compress_streams(files, tr, en, BLOCK, input_sizes=sizes, headerless=True), reps)
    (d_n, st4), td_n = timed(ctx, lambda: ctx.decompress_streams(n, caps, headerless=hl), reps)
    assert all((s == 0).all() for s in (st1, st2, st3, st4))
    stripped = all(np.array_equal(a[header_bytes(len(f)):], b) for a, b, f in zip(h, n, files))
    decoded = all(np.array_equal(x, f) and np.array_equal(y, f) for x, y, f in zip(d_h, d_n, files))
    rates = {"headered": {"compress_files_per_s": len(files) / tc_h, "decompress_files_per_s": len(files) / td_h},
             "headerless": {"compress_files_per_s": len(files) / tc_n, "decompress_files_per_s": len(files) / td_n}}
    return [len(s) for s in h], [len(s) for s in n], rates, stripped and decoded


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=20000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--levels", default="l3,l5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle", action="store_true", help="byte counts from the CPU oracle, without a GPU")
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    files = corpus(a.files, a.seed)
    total = sum(len(f) for f in files)
    hdr = sum(header_bytes(len(f)) for f in files)
    ctx, name, pl = None, "none (CPU oracle)", None
    if not a.oracle:
        name, pl = card()
        ctx = kz.Context(0)
    lines = []
    for lv in a.levels.split(","):
        tr, en = LEVELS[lv]
        if a.oracle:
            with_h, rates, ok = oracle_level(files, tr, en, a.jobs), None, True
            without_h = [m - header_bytes(len(f)) for m, f in zip(with_h, files)]
        else:
            with_h, without_h, rates, ok = gpu_level(ctx, files, tr, en, a.reps)
        line = {"tool": "headerless_bytes", "level": lv, "transform": tr, "entropy": en, "block_size": BLOCK, "files": len(files),
                "input_bytes": total, "bytes_with_headers": sum(with_h), "bytes_without_headers": sum(without_h), "header_bytes": hdr,
                "saved_fraction": hdr / sum(with_h), "source": "oracle" if a.oracle else "gpu", "rates": rates, "checked": ok, "gpu": name,
                "power_limit": pl}
        assert sum(with_h) - sum(without_h) == hdr
        print(json.dumps(line), flush=True)
        lines.append(line)
        assert ok
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
