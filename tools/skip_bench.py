"""What kanzi's skipBlocks option (kz_set_skip_blocks, kanzi c --skip) costs and gains, setting off against on, at -l 3 and -l 5.

Workloads (4 MiB blocks, on the device-resident paths kz_compress_stream_device / kz_decompress_stream_device):
  a) the 200 MB silesia-shaped slab (seed 0), compressible almost everywhere: what the decision pass costs;
  b) the same slab with every fourth 4 MiB block (blocks 3, 7, 11, ...) replaced by members that Python's standard library compressed
     (gzip, bz2 and xz in turn) from seeded pieces of the slab: real magic numbers and real high entropy, as in archives of media,
     packages and already-compressed files.
For every (workload, level) the two settings alternate, --runs times each; encode and decode are timed with CUDA events on the context's
stream and the medians reported as MB/s of input. A separate profiled run gives the blocks stored by magic number and by entropy
(kz_stage_bytes "skip:magic" / "skip:entropy") and the decision kernels' time (kz_kernel_time "skip_hist" / "skip_decide"). Every stream
is checked to decode to its input. One JSON line per (workload, level, setting), with the card's name and power limit read in the same run.

    python tools/skip_bench.py [--runs 3] [--out FILE]
"""
import argparse
import bz2
import gzip
import importlib
import json
import lzma
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
kz = importlib.import_module("kanzi-go_b200")
synth = importlib.import_module("kanzi-go_b200.synth")
from range_bench import BLOCK, LEVELS, N, card  # noqa: E402


def mixed(x):
    """x with every fourth block (3, 7, 11, ...) replaced by stdlib-compressed members (gzip, bz2, xz in turn): members of consecutive
    2 MiB pieces of the slab from a seeded start, concatenated until the block is full, so that no block repeats itself"""
    rng = np.random.default_rng(1)
    y = x.copy()
    coders = [lambda b: gzip.compress(b, mtime=0), bz2.compress, lambda b: lzma.compress(b, format=lzma.FORMAT_XZ, preset=1)]
    for k, b in enumerate(range(3, (N + BLOCK - 1) // BLOCK, 4)):
        n = min(BLOCK, N - b * BLOCK)
        o, fill = int(rng.integers(0, N)), bytearray()
        while len(fill) < n:
            piece = np.roll(x, -o)[: 2 << 20] if o + (2 << 20) > N else x[o: o + (2 << 20)]
            fill += coders[k % 3](piece.tobytes())
            o = (o + (2 << 20)) % N
        y[b * BLOCK: b * BLOCK + n] = np.frombuffer(bytes(fill[:n]), np.uint8)
    return y


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    name, pl = card()
    base = np.ascontiguousarray(synth.silesia_shaped(N, seed=0), np.uint8)
    ctx = kz.Context(0)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream())
    cap = int(ctx.lib.kz_max_stream_output(N, BLOCK))
    d_src = torch.empty(N + 64, dtype=torch.uint8, device="cuda")
    d_cmp = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(N + 64, dtype=torch.uint8, device="cuda")

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = f()
        e1.record(stream)
        e1.synchronize()
        return r, e0.elapsed_time(e1)

    for wl, x in (("a_silesia", base), ("b_mixed", mixed(base))):
        d_src[:N] = torch.from_numpy(x).cuda()
        torch.cuda.synchronize()
        for level, (tr, en) in LEVELS.items():
            t48, et = kz.transform_type(tr), kz.entropy_type(en)

            def enc(skip):
                return ctx.compress_device(d_src.data_ptr(), N, d_cmp.data_ptr(), cap, t48, et, BLOCK, 0, N, skip_blocks=skip)

            def dec(n):
                return ctx.decompress_device(d_cmp.data_ptr(), n, d_out.data_ptr(), N + 64)

            res = {False: {"enc": [], "dec": []}, True: {"enc": [], "dec": []}}
            for skip in (False, True):  # warm-up of both settings, and the check
                n = enc(skip)
                assert dec(n) == N and torch.equal(d_out[:N], d_src[:N]), (wl, level, skip)
            for _ in range(a.runs):
                for skip in (False, True):
                    n, ms_e = timed(lambda: enc(skip))
                    _, ms_d = timed(lambda: dec(n))
                    res[skip]["enc"].append(ms_e)
                    res[skip]["dec"].append(ms_d)
                    res[skip]["bytes"] = int(n)
            for skip in (False, True):
                ctx.profile(True)
                ctx.profile_reset()
                enc(skip)
                prof = {"skip_hist_ms": round(ctx.kernel_time("skip_hist")[1], 3), "skip_decide_ms": round(ctx.kernel_time("skip_decide")[1], 3)}
                for r in ("magic", "entropy"):
                    _, nb, nbytes = ctx.stage_bytes("skip:" + r)
                    prof["stored_" + r] = [nb, nbytes]
                ctx.profile(False)
                ctx.profile_reset()
                me, md = float(np.median(res[skip]["enc"])), float(np.median(res[skip]["dec"]))
                line = json.dumps({"workload": wl, "level": level, "transform": tr, "entropy": en, "skip_blocks": skip, "input_bytes": N,
                                   "compressed_bytes": res[skip]["bytes"], "enc_ms_median": round(me, 2), "dec_ms_median": round(md, 2),
                                   "enc_MBps": round(N / me / 1e3, 1), "dec_MBps": round(N / md / 1e3, 1), "runs": a.runs,
                                   "enc_ms": [round(v, 2) for v in res[skip]["enc"]], "dec_ms": [round(v, 2) for v in res[skip]["dec"]], **prof,
                                   "gpu": name, "power_limit": pl})
                print(line, flush=True)
                if a.out:
                    with open(a.out, "a") as f:
                        f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
