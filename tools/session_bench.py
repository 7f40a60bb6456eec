"""Throughput of the streaming sessions (kz_writer_* / kz_reader_*) on one long stream, next to the whole-stream calls.

Generates a silesia-shaped input of --gib GiB piecewise from a seed (one synth.silesia_shaped slab of 64 MiB, each piece a rotation of it
taken as two views of the slab, so the input is never held twice and the pieces cost nothing inside the timed loops) and, for each chain, feeds it in 1 MiB pieces from pinned memory through a writer (4 MiB blocks, batch_blocks
for about 256 MiB per batch), then feeds the stream it wrote in 1 MiB pieces through a reader. MB/s is input bytes over wall time per
direction (the copies into the pinned input buffer are the caller's I/O and are counted). It records kz_device_bytes of the sessions'
context at its highest (one fresh context per chain), checks that the reader gives the input back (by hash), and in the same run times
kz_compress_stream / kz_decompress_stream on a 200 MB slab, alternated with the sessions. One JSON line per chain, with the card's name and
power limit read in the same run. The effect of the overlap alone (the same sessions without it) is not measured here.

    python tools/session_bench.py [--gib 4] [--chains l3,l5,configs1] [--out FILE]
"""
import argparse
import ctypes as C
import hashlib
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

CHAINS = {"l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0"), "configs1": ("NONE", "ANS0")}
BLOCK = 4 << 20
PIECE = 1 << 20
SLAB = 64 << 20


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "not read"
    return name, pl


class Pump:
    """one session driven through the C ABI from a pinned 1 MiB input buffer into a 64 MiB output buffer; tracks kz_device_bytes"""

    def __init__(self, ctx, step, fin, free, h, sink):
        self.ctx, self.step, self.fin, self.free, self.h, self.sink = ctx, step, fin, free, h, sink
        self.pin = ctx.lib.kz_alloc_pinned(PIECE)
        self.pin_view = np.ctypeslib.as_array((C.c_uint8 * PIECE).from_address(self.pin))
        self.out = np.empty(64 << 20, np.uint8)
        self.peak = 0

    def feed(self, data):
        used, made = C.c_size_t(0), C.c_size_t(0)
        for o in range(0, data.size, PIECE):
            n = min(PIECE, data.size - o)
            self.pin_view[:n] = data[o: o + n]
            pos = 0
            while pos < n:
                self.ctx._check(self.step(self.h, self.pin + pos, n - pos, C.byref(used), self.out.ctypes.data, self.out.size, C.byref(made)))
                pos += used.value
                if made.value:
                    self.sink(self.out[: made.value])
            self.peak = max(self.peak, self.ctx.device_bytes())

    def finish(self):
        made = C.c_size_t(0)
        while True:
            rc = self.ctx._check(self.fin(self.h, self.out.ctypes.data, self.out.size, C.byref(made)))
            if made.value:
                self.sink(self.out[: made.value])
            if rc == 0:
                break
        self.peak = max(self.peak, self.ctx.device_bytes())
        self.free(self.h)
        self.ctx.lib.kz_free_pinned(self.pin)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--chains", default="l3,l5,configs1")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    slab = np.ascontiguousarray(synth.silesia_shaped(SLAB, seed=a.seed), np.uint8)
    npieces = max(1, int(a.gib * (1 << 30)) // SLAB)
    def piece(i):  # np.roll(slab, 7919 * i) as two views: the pieces cost no copy inside the timed loops
        k = (-7919 * i) % SLAB
        return (slab[k:], slab[:k])

    total = npieces * SLAB
    want = hashlib.sha256()
    for i in range(npieces):
        for v in piece(i):
            want.update(v)
    small = np.concatenate([v for i in range(200_000_000 // SLAB + 1) for v in piece(i)])[:200_000_000]
    name, pl = card()
    ref = kz.Context(0)  # the whole-stream calls', so that their scratch is not counted for the sessions
    bb = kz.default_batch_blocks(BLOCK)
    for key in a.chains.split(","):
        ctx = kz.Context(0)  # this chain's sessions alone: kz_device_bytes reports its scratch and the open session's buffers
        tr, en = CHAINS[key]
        t48, et = kz.transform_type(tr), kz.entropy_type(en)
        # whole-stream calls on 200 MB (warm-up, then timed), alternated with the sessions
        s_small = ref.compress(small, tr, en, BLOCK, 0, small.size)
        ref.decompress(s_small, small.size + 64)
        t0 = time.perf_counter()
        s_small = ref.compress(small, tr, en, BLOCK, 0, small.size)
        t_wc = time.perf_counter() - t0
        # writer
        parts = []
        h = C.c_void_p()
        ctx._check(ctx.lib.kz_writer_open(ctx.h, t48, et, BLOCK, 0, bb, total, C.byref(h)))
        w = Pump(ctx, ctx.lib.kz_writer_write, ctx.lib.kz_writer_finish, ctx.lib.kz_writer_free, h, lambda b: parts.append(b.copy()))
        t0 = time.perf_counter()
        for i in range(npieces):
            for v in piece(i):
                w.feed(v)
        w.finish()
        t_w = time.perf_counter() - t0
        stream_bytes = sum(p.size for p in parts)
        t0 = time.perf_counter()
        y = ref.decompress(s_small, small.size + 64)
        t_wd = time.perf_counter() - t0
        assert np.array_equal(y, small)
        # reader
        got = hashlib.sha256()
        h = C.c_void_p()
        ctx._check(ctx.lib.kz_reader_open(ctx.h, bb, C.byref(h)))
        r = Pump(ctx, ctx.lib.kz_reader_read, ctx.lib.kz_reader_finish, ctx.lib.kz_reader_free, h, got.update)
        t0 = time.perf_counter()
        for p in parts:
            r.feed(p)
        r.finish()
        t_r = time.perf_counter() - t0
        assert got.digest() == want.digest(), "the reader did not give the input back"
        res = {"chain": key, "transform": tr, "entropy": en, "block_size": BLOCK, "batch_blocks": bb, "input_bytes": total,
               "stream_bytes": stream_bytes, "writer_MBps": round(total / t_w / 1e6, 1), "reader_MBps": round(total / t_r / 1e6, 1),
               "device_bytes_max": max(w.peak, r.peak), "whole_stream_200MB_compress_MBps": round(small.size / t_wc / 1e6, 1),
               "whole_stream_200MB_decompress_MBps": round(small.size / t_wd / 1e6, 1), "gpu": name, "power_limit": pl}
        line = json.dumps(res)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
        del parts
        ctx.close()
    ref.close()


if __name__ == "__main__":
    main()
