"""Parts of the BWT inverse on the blocks the -l 5 decode of bench.py hands it, and of the stages after it.

The silesia-shaped slab of bench.py (same size and seed) is cut into 4 MiB blocks and encoded on cuda:0 with TEXT+UTF+BWT and no entropy
coder (the stages in front of RANK at -l 5), so the decode of those blocks runs the BWT inverse of the benchmark's 48 blocks in one batch
and then the UTF and TEXT inverses. With kz_bwt_profile bit 0 every part of bwt_inverse_batch is timed by CUDA events under
"bwt_inverse:<part>"; the table gives ms per decode for each part, the whole BWT inverse and the UTF / TEXT inverses after it.

    python tools/bwt_inverse_parts.py [--mb 200] [--reps 5] [--variants]

--variants also times the whole BWT inverse for other shapes of its walk: sub-list stride and staging bytes per sub-list
(kz_bwt_profile bits 8-19; the output never depends on them, which the script checks).
"""
import argparse
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BLOCK = 4 << 20
# (stride, staging bytes per sub-list); 0 = the default of the build
VARIANTS = [(0, 0), (64, 128), (64, 256), (32, 64), (32, 256), (16, 64), (16, 128)]


def encoded_blocks(ctx, kz, mb):
    synth = importlib.import_module("kanzi-go_b200.synth")
    x = synth.silesia_shaped(int(mb * 1_000_000), seed=synth.SEED + 1)  # bench.py: make_data(kind, n, synth.SEED + 1)
    blocks = [x[o: o + BLOCK] for o in range(0, len(x), BLOCK)]
    t = kz.transform_type("TEXT+UTF+BWT")
    return blocks, t, ctx.encode_blocks(t, kz.E_NONE, blocks)


def timed_decode(ctx, kz, t, payloads, reps, **shape):
    try:
        ctx.bwt_profile(time_rounds=True, **shape)
    except TypeError:  # an older build: no walk shape (and no parts of the inverse timed)
        if shape:
            return None
        ctx.bwt_profile(time_rounds=True)
    ctx.profile(True)
    out = ctx.decode_blocks(t, kz.E_NONE, payloads, block_size=BLOCK)  # warm-up (and the bytes)
    ctx.profile_reset()
    for _ in range(reps):
        ctx.decode_blocks(t, kz.E_NONE, payloads, block_size=BLOCK)
    res = {nm: ctx.kernel_time(nm)[1] / reps for nm in ctx.profile_names()}
    ctx.profile(False)
    return res, out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--mb", type=float, default=200.0, help="slab size in MB (bench.py: 200)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--variants", action="store_true", help="time the BWT inverse for other walk shapes as well")
    a = ap.parse_args()
    kz = importlib.import_module("kanzi-go_b200")
    ctx = kz.Context(0)
    blocks, t, payloads = encoded_blocks(ctx, kz, a.mb)
    print(f"{len(blocks)} blocks, {sum(len(b) for b in blocks):,} input bytes, {sum(len(p[0]) for p in payloads):,} bytes into the decode")
    res, out = timed_decode(ctx, kz, t, payloads, a.reps)
    for b, d in zip(blocks, out):
        assert np.array_equal(b, d), "decode differs from the input"
    print("part                     ms per decode")
    for nm in sorted(res):
        if nm.startswith("bwt_inverse") or nm in ("utf_inverse", "text_inverse"):
            print(f"{nm:24s} {res[nm]:8.2f}")
    if a.variants:
        print("\nstride  stage   bwt_inverse ms   walk   doubling   copy")
        for st, sg in VARIANTS:
            r = timed_decode(ctx, kz, t, payloads, a.reps, inverse_stride=st, inverse_stage=sg)
            if r is None:
                print(f"{st:6d} {sg:6d}   (not in this build)")
                continue
            rv, ov = r
            for b, d in zip(blocks, ov):
                assert np.array_equal(b, d), ("decode differs from the input", st, sg)
            print(f"{st:6d} {sg:6d}   {rv.get('bwt_inverse', 0):14.2f} {rv.get('bwt_inverse:walk', 0):6.2f} {rv.get('bwt_inverse:doubling', 0):10.2f}"
                  f" {rv.get('bwt_inverse:copy', 0):6.2f}")
        ctx.bwt_profile()


if __name__ == "__main__":
    main()
