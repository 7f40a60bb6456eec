"""Cost of range reads over many small compressed objects: one call per object against one call over all of them.

Builds the corpus of tools/streams_bench.py (--files objects cut from synth.silesia_shaped, log-normal sizes of median 16 KiB, 4 MiB
blocks, so most objects are one block), compresses it with one kz_compress_streams call per level, and times with a host clock around
calls that end in a device synchronise:
  index:  one kz_index_build per object (Context.index) against one kz_index_build_streams call (Context.index_streams); the blobs of
          both arms must be identical.
  reads:  batches of --batch reads of 4 KiB (shorter where the object is), objects drawn uniformly or Zipf(1.2) over a shuffled order,
          offsets uniform inside the object. single = one kz_read_ranges[_device] per touched object (StreamIndex.read_many /
          read_many_device); batched = one kz_read_ranges_streams[_device] call (Context.read_streams / read_streams_device). Host
          variant (streams and destinations in host memory) and device variant (both in HBM), without a cache and with a cache of 100 %
          of the decoded corpus that one read of every object filled first (each arm has its own cache, filled the same way).
Every arm is warmed up, the arms alternate --reps times with a fresh batch each time, and the medians are reported. Both arms must return
identical bytes, equal to the input. One JSON line per case with ms per batch, reads/s and kernel launches per arm, next to the card's
name and power limit read in the same run. Fails without a GPU.

    python tools/read_streams_bench.py [--files 20000] [--levels l3,l5] [--reps 3] [--batch 1000] [--out FILE]
"""
import argparse
import ctypes as C
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
from streams_bench import BLOCK, LEVELS, card, corpus  # noqa: E402

READ = 4096
PAGE = 64 << 10


def batch(rng, sizes, n, zipf, perm):
    """n requests (object, off, len) over objects of the given decoded sizes (all > 0)"""
    if zipf:
        obj = perm[np.minimum(rng.zipf(1.2, n) - 1, len(sizes) - 1)]
    else:
        obj = rng.integers(0, len(sizes), n)
    out = []
    for k in obj:
        sz = int(sizes[k])
        o = int(rng.integers(0, max(sz - READ, 0) + 1))
        out.append((int(k), o, min(READ, sz - o)))
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=20000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--levels", default="l3,l5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    files = [f for f in corpus(a.files, a.seed) if len(f)]
    sizes = np.array([len(f) for f in files], np.int64)
    name, pl = card()
    ctx = kz.Context(0)
    lines = []

    def emit(line):
        line.update({"gpu": name, "power_limit": pl})
        print(json.dumps(line), flush=True)
        lines.append(line)

    for lv in a.levels.split(","):
        tr, en = LEVELS[lv]
        streams, st = ctx.compress_streams(files, tr, en, BLOCK)
        assert not st.any()
        # ---- index: one build per object against one build over all objects
        ctx.index_streams(streams[:64])
        [ctx.index(s) for s in streams[:64]]
        t_single, t_batched, l_single, l_batched = [], [], 0, 0
        for _ in range(a.reps):
            ctx.launch_count(reset=True)
            t0 = time.perf_counter()
            single = [ctx.index(s) for s in streams]
            t_single.append(time.perf_counter() - t0)
            l_single = ctx.launch_count(reset=True)
            t0 = time.perf_counter()
            batched, st = ctx.index_streams(streams)
            t_batched.append(time.perf_counter() - t0)
            l_batched = ctx.launch_count(reset=True)
            assert not st.any()
        same = all(x.save() == y.save() for x, y in zip(single, batched))
        emit({"tool": "read_streams_bench", "case": "index", "level": lv, "transform": tr, "entropy": en, "objects": len(streams),
              "single_ms": 1e3 * float(np.median(t_single)), "batched_ms": 1e3 * float(np.median(t_batched)), "single_launches": int(l_single),
              "batched_launches": int(l_batched), "identical_blobs": same})
        assert same
        del single, batched
        # ---- reads
        so = np.zeros(len(streams), np.uint64)
        at = 0
        for i, s in enumerate(streams):
            so[i] = at
            at = (at + len(s) + 64 + 15) & ~15
        sl = np.array([len(s) for s in streams], np.uint64)
        buf = np.zeros(at + 64, np.uint8)
        for o, s in zip(so, streams):
            buf[int(o): int(o) + len(s)] = s
        d_src = torch.from_numpy(buf).cuda()
        pages = int(sum((min(int(n), BLOCK) + PAGE - 1) // PAGE * ((int(n) + BLOCK - 1) // BLOCK) for n in sizes))
        rng = np.random.default_rng(a.seed)
        perm = rng.permutation(len(streams))
        for device in (False, True):
            for cached in (False, True):
                ixs = {arm: ctx.index_streams(streams)[0] for arm in ("single", "batched")}
                slots_of = {arm: (C.c_void_p * len(streams))(*[x.h for x in ixs[arm]]) for arm in ixs}
                caches = {arm: ctx.block_cache(pages * PAGE) for arm in ("single", "batched")} if cached else {"single": None, "batched": None}
                if cached:  # one read of every object fills each arm's cache
                    every = [(k, 0, int(sizes[k])) for k in range(len(streams))]
                    for arm in ("single", "batched"):
                        for i in range(0, len(every), 2000):
                            ctx.read_streams(streams, ixs[arm], every[i: i + 2000], cache=caches[arm])
                d_dst = torch.zeros(a.batch * READ + 64, dtype=torch.uint8, device="cuda")

                def run(arm, reqs):
                    """-> list of bytes per request"""
                    ix, cache = ixs[arm], caches[arm]
                    slots = slots_of[arm]
                    ln = [r[2] for r in reqs]
                    dst_off = np.concatenate([[0], np.cumsum(ln[:-1])]).astype(np.uint64)
                    if arm == "batched":
                        # the ABI straight from the packed object table (the wrappers would pack it again on every call)
                        rs = np.array([r[0] for r in reqs], np.uint32)
                        off = np.array([r[1] for r in reqs], np.uint64)
                        n = np.array(ln, np.uint64)
                        out_len, st = np.zeros(len(reqs), np.uint64), np.zeros(len(reqs), np.int32)
                        fn = ctx.lib.kz_read_ranges_streams_device if device else ctx.lib.kz_read_ranges_streams
                        h_dst = None if device else np.empty(int(n.sum()) + 1, np.uint8)
                        fn(ctx.h, None if cache is None else cache.h, len(streams), C.addressof(slots), d_src.data_ptr() if device else buf.ctypes.data,
                           so.ctypes.data, sl.ctypes.data, len(reqs), rs.ctypes.data, off.ctypes.data, n.ctypes.data,
                           d_dst.data_ptr() if device else h_dst.ctypes.data, dst_off.ctypes.data, out_len.ctypes.data, st.ctypes.data)
                        assert not st.any()
                        if not device:
                            return [h_dst[int(o): int(o) + k].tobytes() for o, k in zip(dst_off, ln)]
                    else:
                        by_obj = {}
                        for i, r in enumerate(reqs):
                            by_obj.setdefault(r[0], []).append(i)
                        outs = [None] * len(reqs)
                        for k, idx in by_obj.items():
                            if device:
                                out_len, st = ix[k].read_many_device(d_src.data_ptr() + int(so[k]), int(sl[k]), [reqs[i][1] for i in idx],
                                                                     [ln[i] for i in idx], d_dst.data_ptr(), dst_off[idx], ctx, cache)
                                assert not st.any()
                            else:
                                got, st = ix[k].read_many(streams[k], [reqs[i][1:] for i in idx], ctx, cache)
                                assert not any(st)
                                for i, g in zip(idx, got):
                                    outs[i] = g
                        if not device:
                            return outs
                    torch.cuda.synchronize()
                    h = d_dst[: int(sum(ln))].cpu().numpy()
                    return [h[int(o): int(o) + n].tobytes() for o, n in zip(dst_off, ln)]

                for pattern in ("uniform", "zipf"):
                    warm = batch(rng, sizes, a.batch, pattern == "zipf", perm)
                    run("single", warm), run("batched", warm)
                    t = {"single": [], "batched": []}
                    launches = {}
                    identical = True
                    touched = []
                    for rep in range(a.reps):
                        reqs = batch(rng, sizes, a.batch, pattern == "zipf", perm)
                        touched.append(len({r[0] for r in reqs}))
                        got = {}
                        for arm in (("single", "batched") if rep % 2 == 0 else ("batched", "single")):
                            ctx.launch_count(reset=True)
                            t0 = time.perf_counter()
                            got[arm] = run(arm, reqs)
                            t[arm].append(time.perf_counter() - t0)
                            launches[arm] = int(ctx.launch_count(reset=True))
                        want = [files[k][o: o + n].tobytes() for k, o, n in reqs]
                        identical &= got["single"] == got["batched"] == want
                    ms = {arm: 1e3 * float(np.median(v)) for arm, v in t.items()}
                    emit({"tool": "read_streams_bench", "case": "read", "level": lv, "transform": tr, "entropy": en, "objects": len(streams),
                          "variant": "device" if device else "host", "pattern": pattern, "cache": "100%" if cached else "none",
                          "reads_per_batch": a.batch, "objects_touched": int(np.median(touched)), "single_ms": ms["single"],
                          "batched_ms": ms["batched"], "single_reads_per_s": a.batch / ms["single"] * 1e3,
                          "batched_reads_per_s": a.batch / ms["batched"] * 1e3, "single_launches": launches["single"],
                          "batched_launches": launches["batched"], "identical": identical})
                    assert identical
                for c in caches.values():
                    if c is not None:
                        c.close()
        del d_src
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
