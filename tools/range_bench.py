"""Cost of a block range decode (kz_set_block_range, kanzi d --from / --to) next to the full decode of the same stream.

Compresses the 200 MB silesia-shaped slab (seed 0, 4 MiB blocks: 48 blocks) at -l 3 and -l 5 with the GPU and then, on the device-resident
path (kz_decompress_stream_device, stream and output in HBM), times with CUDA events on the context's stream:
  - the full decode;
  - one block at the front (block 1), in the middle (block 25) and at the end (block 48);
  - the first half of the stream (blocks 1 .. 24).
Each case is warmed up once and timed --reps times; the median is reported, with the decoded bytes (checked against the matching slice of
the input) and kz_stage_bytes of every inverse stage from a separate profiled run. One JSON line per (level, case), with the card's name and
power limit read in the same run.

    python tools/range_bench.py [--reps 5] [--out FILE]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
kz = importlib.import_module("kanzi-go_b200")
synth = importlib.import_module("kanzi-go_b200.synth")

LEVELS = {"l3": ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), "l5": ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")}
BLOCK = 4 << 20
N = 200_000_000


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
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    x = np.ascontiguousarray(synth.silesia_shaped(N, seed=0), np.uint8)
    nblocks = (N + BLOCK - 1) // BLOCK
    cases = {"full": (-1, -1), "block_front": (1, 2), "block_middle": (nblocks // 2 + 1, nblocks // 2 + 2),
             "block_end": (nblocks, nblocks + 1), "first_half": (1, nblocks // 2 + 1)}
    name, pl = card()
    ctx = kz.Context(0)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream())
    cap = N + 64
    d_dst = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    for level, (tr, en) in LEVELS.items():
        s = ctx.compress(x, tr, en, BLOCK, 0, N)
        d_src = torch.zeros(s.size + 64, dtype=torch.uint8, device="cuda")
        d_src[: s.size] = torch.from_numpy(s).cuda()
        torch.cuda.synchronize()
        for case, (frm, to) in cases.items():
            lo = 0 if frm < 0 else frm - 1
            hi = nblocks if to < 0 else to - 1
            want = x[lo * BLOCK: min(hi * BLOCK, N)]

            def run():
                return ctx.decompress_device(d_src.data_ptr(), s.size, d_dst.data_ptr(), cap, frm, to)

            n = run()  # warm-up
            assert n == want.size and np.array_equal(d_dst[:n].cpu().numpy(), want), (level, case)
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run()
                e1.record(stream)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            ctx.profile(True)
            ctx.profile_reset()
            run()
            stages = {}
            for t in (kz.T_TEXT, kz.T_UTF, kz.T_PACK, kz.T_MM, kz.T_LZX, kz.T_BWT, kz.T_RANK, kz.T_ZRLT):
                k, b_in, b_out = ctx.stage_bytes("stage:inv:%d" % t)
                if k:
                    stages["inv:%d" % t] = [b_in, b_out]
            ctx.profile(False)
            ctx.profile_reset()
            res = {"level": level, "transform": tr, "entropy": en, "case": case, "from": frm, "to": to, "stream_bytes": int(s.size),
                   "decoded_bytes": int(n), "ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3), "reps": a.reps,
                   "stage_bytes": stages, "gpu": name, "power_limit": pl}
            line = json.dumps(res)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
        del d_src
    ctx.close()


if __name__ == "__main__":
    main()
