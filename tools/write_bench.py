"""What a write into a compressed stream (kz_write_ranges[_device]) costs against what an object store pays today: decompress the whole
stream, edit it, compress it again.

Compresses the 200 MB silesia-shaped slab (seed 0, 4 MiB blocks: 48 blocks) at -l 3 and -l 5 and, for the host variant (stream, writes and
tail in host memory) and the device variant (all in HBM), times with a host clock around calls that end in a device synchronise:
  (a) w1:      4 KiB overwrites at random offsets, one per call (--calls calls, median);
  (b) w256:    256 such overwrites in one call (median of --calls // 4 calls);
  (c) a64k:    64 KiB appends, one per call (median);
  (d) a4m:     4 MiB appends, one per call (median);
  (e) rebuild: decompress the slab, change 4 KiB, compress it again (the host API, median of 3).
Every call starts from the original stream and an index whose size is known, so each one re-encodes only what it touches. The first call's
new stream is checked against a compress of the edited data. One JSON line per (level, variant), with the card's name and power limit read
in the same run. Fails without a GPU.

    python tools/write_bench.py [--calls 8] [--out FILE]
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

W = 4096


def timed(f):
    import torch

    torch.cuda.synchronize()
    t = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    ctx = kz.Context(0)
    x = np.ascontiguousarray(synth.silesia_shaped(N, seed=0), np.uint8)
    rng = np.random.default_rng(1)
    lines = []
    for lv, (tr, en) in LEVELS.items():
        s = ctx.compress(x, tr, en, block_size=BLOCK, input_size=N)
        d_src = torch.zeros(len(s) + 64, dtype=torch.uint8, device="cuda")
        d_src[: len(s)] = torch.from_numpy(s).cuda()
        base = kz.StreamIndex.load(ctx.index(s).save(), ctx)
        base.read(s, N - 1, 1)  # the size is known
        blob = base.save()
        cases = {
            "w1": lambda: [(int(rng.integers(0, N - W)), rng.integers(0, 256, W, dtype=np.uint8).tobytes())],
            "w256": lambda: [(int(o), rng.integers(0, 256, W, dtype=np.uint8).tobytes()) for o in rng.integers(0, N - W, 256)],
            "a64k": lambda: [(kz.WRITE_APPEND, synth.markov_text(64 << 10, seed=int(rng.integers(1 << 30))).tobytes())],
            "a4m": lambda: [(kz.WRITE_APPEND, synth.markov_text(4 << 20, seed=int(rng.integers(1 << 30))).tobytes())],
        }
        for variant in ("host", "device"):
            res = {"level": lv, "variant": variant, "card": name, "power_limit": power, "stream_bytes": len(s), "ms": {}}
            for cname, make in cases.items():
                times = []
                for c in range(max(1, a.calls // 4) if cname == "w256" else a.calls):
                    writes = make()
                    ix = kz.StreamIndex.load(blob, ctx)
                    if variant == "host":
                        ms, (keep, tail) = timed(lambda: ix.write_many(s, writes))
                        new_tail = tail
                    else:
                        bufs = [np.frombuffer(d, np.uint8) for _, d in writes]
                        data = np.concatenate(bufs)
                        ln = [b.size for b in bufs]
                        doff = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
                        d_data = torch.from_numpy(data).cuda()
                        cap = len(s) + sum(n // BLOCK + 2 for n in ln) * ctx.lib.kz_max_block_output(BLOCK) + 16
                        d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
                        ms, (keep, nd) = timed(lambda: ix.write_many_device(d_src, len(s), [o for o, _ in writes], ln, d_data, doff, d_dst, cap))
                        new_tail = d_dst[:nd].cpu().numpy().tobytes()
                    if c == 0:
                        y = bytearray(x.tobytes())
                        for o, d in writes:
                            o = len(y) if o == kz.WRITE_APPEND else o
                            y[o:o + len(d)] = d
                        want = ctx.compress(np.frombuffer(bytes(y), np.uint8), tr, en, block_size=BLOCK, input_size=N)
                        assert s[:keep].tobytes() + new_tail == want.tobytes(), (lv, variant, cname)
                    times.append(ms)
                res["ms"][cname] = float(np.median(times))
            reb = []
            for _ in range(3):
                def rebuild():
                    y = ctx.decompress(s, N + 64).copy()
                    o = int(rng.integers(0, N - W))
                    y[o:o + W] = 0
                    return ctx.compress(y, tr, en, block_size=BLOCK, input_size=N)
                reb.append(timed(rebuild)[0])
            res["ms"]["rebuild"] = float(np.median(reb))
            print(json.dumps(res), flush=True)
            lines.append(res)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
