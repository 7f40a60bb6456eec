"""What a stream index and batched range reads (kz_index_build, kz_read_ranges) cost next to the calls a caller had before them.

Compresses the 200 MB silesia-shaped slab (seed 0, 4 MiB blocks: 48 blocks) at -l 3 and -l 5 with the GPU and then, for the device-resident
variant (stream and destination in HBM) and the host variant (both in host memory), times with a host clock around calls that end in a
device synchronise:
  - full:          one full decode (kz_decompress_stream[_device]);
  - index_build:   kz_index_build[_device];
  - one_read:      one 4 KiB read through the index, against one_range: kz_set_block_range(k, k + 1) + a decode of that block + a slice;
  - batch_1000:    1,000 uniformly random 4 KiB reads in one call, against single_calls: the same reads one call each (--singles of them are
                   timed and the sum scaled to 1,000; the JSON says how many were timed);
  - batch_4blocks: 1,000 random 4 KiB reads confined to 4 blocks, in one call.
Every arm is warmed up once; then the arms alternate --reps times and the median is reported. Every read is checked against the input.
One JSON line per (level, variant), with the card's name and power limit read in the same run. Fails without a GPU.

    python tools/read_bench.py [--reps 3] [--singles 1000] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
kz = importlib.import_module("kanzi-go_b200")
synth = importlib.import_module("kanzi-go_b200.synth")
from range_bench import BLOCK, LEVELS, N, card  # noqa: E402

READ = 4096
NREQ = 1000


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--singles", type=int, default=NREQ, help="how many of the 1,000 single-request calls are timed")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    name, pl = card()
    x = np.ascontiguousarray(synth.silesia_shaped(N, seed=0), np.uint8)
    nblocks = (N + BLOCK - 1) // BLOCK
    rng = np.random.default_rng(0)
    uniform = [(int(o), READ) for o in rng.integers(0, N - READ, NREQ)]
    four = [(int(b) * BLOCK + int(o), READ) for b, o in zip(rng.choice([3, 17, 30, 40], NREQ), rng.integers(0, BLOCK - READ, NREQ))]
    one = uniform[0]
    ctx = kz.Context(0)

    def timed(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    for level, (tr, en) in LEVELS.items():
        s = ctx.compress(x, tr, en, block_size=BLOCK, input_size=N)
        d_src = torch.zeros(len(s) + 64, dtype=torch.uint8, device="cuda")
        d_src[: len(s)] = torch.from_numpy(s).cuda()
        d_full = torch.empty(N + 128, dtype=torch.uint8, device="cuda")
        d_dst = torch.empty(NREQ * READ + 64, dtype=torch.uint8, device="cuda")
        for variant in ("device", "host"):
            dev = variant == "device"
            ix = ctx.index_device(d_src, len(s)) if dev else ctx.index(s)

            def reads(reqs):
                """one call -> the delivered bytes, request after request"""
                if not dev:
                    outs, st = ix.read_many(s, reqs)
                    assert not any(st)
                    return b"".join(outs)
                out_len, st = ix.read_many_device(d_src, len(s), [r[0] for r in reqs], [r[1] for r in reqs], d_dst, [READ * i for i in range(len(reqs))])
                assert not st.any() and (out_len == READ).all()
                return d_dst[: READ * len(reqs)]

            def check(got, reqs):
                want = b"".join(x[o: o + n].tobytes() for o, n in reqs)
                got = got if isinstance(got, bytes) else got.cpu().numpy().tobytes()
                assert got == want

            def one_range():
                k = one[0] // BLOCK
                if dev:
                    n = ctx.decompress_device(d_src.data_ptr(), len(s), d_full.data_ptr(), N + 64, k + 1, k + 2)
                    return d_full[one[0] - k * BLOCK: one[0] - k * BLOCK + READ], n
                blk = ctx.decompress(s, BLOCK + 64, k + 1, k + 2)
                return blk[one[0] - k * BLOCK: one[0] - k * BLOCK + READ].tobytes(), len(blk)

            def singles():
                for r in uniform[: a.singles]:
                    reads([r])

            arms = {
                "full": (lambda: ctx.decompress_device(d_src.data_ptr(), len(s), d_full.data_ptr(), N + 64)) if dev else (lambda: ctx.decompress(s, N + 64)),
                "index_build": (lambda: ctx.index_device(d_src, len(s))) if dev else (lambda: ctx.index(s)),
                "one_read": lambda: reads([one]),
                "one_range": one_range,
                "batch_1000": lambda: reads(uniform),
                "batch_4blocks": lambda: reads(four),
                "single_calls": singles,
            }
            check(reads(uniform), uniform)  # warm-up of every arm, and the checks
            check(reads(four), four)
            check(reads([one]), [one])
            got = one_range()[0]
            check(got if isinstance(got, bytes) else got, [one])
            arms["full"]()
            arms["index_build"]()
            ms = {k: [] for k in arms}
            for rep in range(a.reps):
                for k, f in arms.items():
                    if k == "single_calls" and rep:
                        continue  # the longest arm by far: timed once
                    ms[k].append(timed(f)[1])
            med = {k: round(float(np.median(v)), 2) for k, v in ms.items()}
            med["single_calls_scaled_to_1000"] = round(med.pop("single_calls") * NREQ / max(a.singles, 1), 1)
            ctx.profile(True)
            ctx.profile_reset()
            reads(uniform)
            blocks = ctx.stage_bytes("read:blocks")[1]
            h2d = ctx.stage_bytes("read:h2d")[2]
            ctx.profile(False)
            ctx.profile_reset()
            line = json.dumps({"level": level, "transform": tr, "entropy": en, "variant": variant, "input_bytes": N, "stream_bytes": int(len(s)),
                               "blocks": nblocks, "read_bytes": READ, "requests": NREQ, "ms_median": med, "reps": a.reps, "singles_timed": a.singles,
                               "batch_1000_blocks_decoded": blocks, "batch_1000_h2d_bytes": h2d, "gpu": name, "power_limit": pl})
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
