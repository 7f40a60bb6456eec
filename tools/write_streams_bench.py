"""Cost of writes into many small compressed objects: one call per touched object against one call over all of them.

Builds the corpus of tools/streams_bench.py (--files objects cut from synth.silesia_shaped, log-normal sizes of median 16 KiB, 4 MiB
blocks, so most objects are one block), compresses it with one kz_compress_streams call per level, and times, with a host clock around
calls that end in a device synchronise, batches of --batch writes:
  overwrite-uniform / overwrite-zipf: 4 KiB overwrites at uniform offsets inside the object, objects drawn uniformly or Zipf(1.2) over a
          shuffled order;
  append: 1 KiB appends (KZ_WRITE_APPEND), objects drawn uniformly.
single = one kz_write_ranges[_device] per touched object (StreamIndex.write_many / write_many_device); batched = one
kz_write_ranges_streams[_device] call (Context.write_streams / the device ABI on the packed object table). Host variant (streams, data
and tails in host memory) and device variant (all in HBM). Every batch starts from the compressed corpus with fresh indexes
(kz_index_build_streams, outside the timed window), so appends learn each object's size. Every arm is warmed up, the arms alternate
--reps times with a fresh batch each time, and the medians are reported. Both arms must return identical keeps and tails. One JSON line
per case with ms per batch and kernel launches per arm, next to the card's name and power limit read in the same run. Fails without a GPU.

    python tools/write_streams_bench.py [--files 20000] [--levels l3,l5] [--reps 3] [--batch 1000] [--out FILE]
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

OVERWRITE, APPEND = 4096, 1024


def batch(rng, sizes, n, pattern, perm):
    """n writes (object, off, data) over objects of the given decoded sizes (all > 0)"""
    if pattern == "overwrite-zipf":
        obj = perm[np.minimum(rng.zipf(1.2, n) - 1, len(sizes) - 1)]
    else:
        obj = rng.integers(0, len(sizes), n)
    out = []
    for k in obj:
        if pattern == "append":
            out.append((int(k), kz.WRITE_APPEND, rng.integers(0, 256, APPEND, dtype=np.uint8).tobytes()))
        else:
            sz = int(sizes[k])
            out.append((int(k), int(rng.integers(0, max(sz - OVERWRITE, 0) + 1)), rng.integers(0, 256, OVERWRITE, dtype=np.uint8).tobytes()))
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
    mbo = ctx.lib.kz_max_block_output(BLOCK)
    lines = []

    def emit(line):
        line.update({"gpu": name, "power_limit": pl})
        print(json.dumps(line), flush=True)
        lines.append(line)

    for lv in a.levels.split(","):
        tr, en = LEVELS[lv]
        streams, st = ctx.compress_streams(files, tr, en, BLOCK)
        assert not st.any()
        ns = len(streams)
        so = np.zeros(ns, np.uint64)
        at = 0
        for i, s in enumerate(streams):
            so[i] = at
            at = (at + len(s) + 64 + 15) & ~15
        sl = np.array([len(s) for s in streams], np.uint64)
        buf = np.zeros(at + 64, np.uint8)
        for o, s in zip(so, streams):
            buf[int(o): int(o) + len(s)] = s
        d_src = torch.from_numpy(buf).cuda()
        rng = np.random.default_rng(a.seed)
        perm = rng.permutation(ns)
        for device in (False, True):

            def run(arm, writes):
                """-> {object: (keep, tail)} over the touched objects, from fresh indexes"""
                ixs, st = ctx.index_streams(streams)
                assert not st.any()
                torch.cuda.synchronize()
                by_obj, by_idx = {}, {}
                for i, w in enumerate(writes):
                    by_obj.setdefault(w[0], []).append(w[1:])
                    by_idx.setdefault(w[0], []).append(i)
                cap = {k: int(sl[k]) + sum(len(d) // BLOCK + 2 for _, d in v) * mbo + 16 for k, v in by_obj.items()}
                if device:
                    bufs = [np.frombuffer(w[2], np.uint8) for w in writes]
                    ln = np.array([b.size for b in bufs], np.uint64)
                    data_off = np.concatenate([[0], np.cumsum(ln[:-1])]).astype(np.uint64)
                    d_data = torch.from_numpy(np.concatenate(bufs)).cuda()
                    dst_off = np.zeros(ns, np.uint64)
                    dst_cap = np.zeros(ns, np.uint64)
                    pos = 0
                    for k in sorted(by_obj):
                        dst_off[k], dst_cap[k] = pos, cap[k]
                        pos += (cap[k] + 15) & ~15
                    d_dst = torch.empty(pos + 64, dtype=torch.uint8, device="cuda")
                    torch.cuda.synchronize()
                ctx.launch_count(reset=True)
                t0 = time.perf_counter()
                res = {}
                if arm == "batched" and device:
                    slots = (C.c_void_p * ns)(*[x.h for x in ixs])
                    ws = np.array([w[0] for w in writes], np.uint32)
                    off = np.array([w[1] for w in writes], np.uint64)
                    keep, out_n, st = np.zeros(ns, np.uint64), np.zeros(ns, np.uint64), np.zeros(ns, np.int32)
                    rc = ctx.lib.kz_write_ranges_streams_device(ctx.h, ns, C.addressof(slots), d_src.data_ptr(), so.ctypes.data, sl.ctypes.data, len(writes),
                                                                ws.ctypes.data, off.ctypes.data, ln.ctypes.data, d_data.data_ptr(), data_off.ctypes.data,
                                                                d_dst.data_ptr(), dst_off.ctypes.data, dst_cap.ctypes.data, keep.ctypes.data,
                                                                out_n.ctypes.data, st.ctypes.data)
                    assert rc == 0
                    ms = 1e3 * (time.perf_counter() - t0)
                    for k in by_obj:
                        res[k] = (int(keep[k]), int(dst_off[k]), int(out_n[k]))
                elif arm == "batched":
                    keeps, tails, st = ctx.write_streams(streams, ixs, writes)
                    ms = 1e3 * (time.perf_counter() - t0)
                    assert not any(st)
                    res = {k: (keeps[k], tails[k]) for k in by_obj}
                else:
                    for k, v in by_obj.items():
                        if device:
                            idx = by_idx[k]
                            kp, n = ixs[k].write_many_device(d_src.data_ptr() + int(so[k]), int(sl[k]), [writes[i][1] for i in idx], ln[idx],
                                                             d_data.data_ptr(), data_off[idx], d_dst.data_ptr() + int(dst_off[k]), cap[k], ctx)
                            res[k] = (kp, int(dst_off[k]), n)
                        else:
                            res[k] = ixs[k].write_many(streams[k], v, ctx)
                    torch.cuda.synchronize()
                    ms = 1e3 * (time.perf_counter() - t0)
                nl = int(ctx.launch_count(reset=True))
                if device:
                    h = d_dst.cpu().numpy()
                    res = {k: (r[0], h[r[1]: r[1] + r[2]].tobytes()) for k, r in res.items()}
                return ms, nl, res

            for pattern in ("overwrite-uniform", "overwrite-zipf", "append"):
                warm = batch(rng, sizes, a.batch, pattern, perm)
                run("single", warm), run("batched", warm)
                t = {"single": [], "batched": []}
                launches = {}
                identical = True
                touched = []
                for rep in range(a.reps):
                    writes = batch(rng, sizes, a.batch, pattern, perm)
                    touched.append(len({w[0] for w in writes}))
                    got = {}
                    for arm in (("single", "batched") if rep % 2 == 0 else ("batched", "single")):
                        ms, launches[arm], got[arm] = run(arm, writes)
                        t[arm].append(ms)
                    identical &= got["single"] == got["batched"]
                med = {arm: float(np.median(v)) for arm, v in t.items()}
                emit({"tool": "write_streams_bench", "level": lv, "transform": tr, "entropy": en, "objects": ns, "variant": "device" if device else "host",
                      "pattern": pattern, "writes_per_batch": a.batch, "write_bytes": APPEND if pattern == "append" else OVERWRITE,
                      "objects_touched": int(np.median(touched)), "single_ms": med["single"], "batched_ms": med["batched"],
                      "speedup": med["single"] / med["batched"], "single_launches": launches["single"], "batched_launches": launches["batched"],
                      "identical": identical})
                assert identical
        del d_src
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
