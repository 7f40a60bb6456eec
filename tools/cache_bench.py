"""What the block cache (kz_cache_*, kz_read_ranges_cached[_device]) saves on repeated range reads, and what it costs when it saves nothing.

Compresses the 200 MB silesia-shaped slab (seed 0, 4 MiB blocks: 48 blocks) at -l 3 and -l 5 and, for the device-resident variant (stream
and destination in HBM) and the host variant (both in host memory), times with a host clock around calls that end in a device synchronise:
  (a) reader_at:  4 KiB reads in order over 8 blocks, one call each (an io.ReaderAt's pattern: 8,192 calls). Cached: every call, from an
                  empty cache (one decode per block, then copies). Uncached: --singles calls spread evenly over the 8 blocks (the
                  same number in each) are timed and the sum scaled to 8,192.
  (b) zipf:       10 calls of 1,000 4 KiB reads each, blocks drawn Zipf(1.2) over a shuffled block order, offsets uniform inside the
                  block; budgets of 25 %, 50 % and 100 % of the decoded size, each from an empty cache, against the uncached calls:
                  ms per call (median of the 10 calls, and the first call alone) and the hit rate over the 10 calls.
  (c) no_hits:    1,000 uniformly random 4 KiB reads in one call on an empty cache (every block a miss: hashing, lookups and inserts),
                  against the same call uncached; plus the hashing alone, from kz_profile (device kernel time or host wall time).
The arms alternate --reps times and the medians are reported. Every read is checked against the input. One JSON line per (level,
variant), with the card's name and power limit read in the same run. Fails without a GPU.

    python tools/cache_bench.py [--reps 3] [--singles 32] [--out FILE]
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
CALLS = 10
SEQ_BLOCKS = 8


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--singles", type=int, default=32, help="how many of the uncached reader_at calls are timed (a multiple of 8)")
    ap.add_argument("--levels", default="l3,l5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    name, pl = card()
    x = np.ascontiguousarray(synth.silesia_shaped(N, seed=0), np.uint8)
    nblocks = (N + BLOCK - 1) // BLOCK
    rng = np.random.default_rng(0)
    seq = [(k * READ + 20 * BLOCK, READ) for k in range(SEQ_BLOCKS * BLOCK // READ)]  # blocks 20 .. 27
    perm = rng.permutation(nblocks)
    zipf_sets = []
    for _ in range(CALLS):
        b = perm[np.minimum(rng.zipf(1.2, NREQ) - 1, nblocks - 1)]
        o = b * BLOCK + rng.integers(0, BLOCK - READ, NREQ)
        zipf_sets.append([(int(v), READ) for v in np.minimum(o, N - READ)])
    uniform = [(int(o), READ) for o in rng.integers(0, N - READ, NREQ)]
    ctx = kz.Context(0)

    def timed(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    for level in a.levels.split(","):
        tr, en = LEVELS[level]
        s = ctx.compress(x, tr, en, block_size=BLOCK, input_size=N)
        d_src = torch.zeros(len(s) + 64, dtype=torch.uint8, device="cuda")
        d_src[: len(s)] = torch.from_numpy(s).cuda()
        d_dst = torch.empty(NREQ * READ + 64, dtype=torch.uint8, device="cuda")
        for variant in ("device", "host"):
            dev = variant == "device"
            ix = ctx.index_device(d_src, len(s)) if dev else ctx.index(s)

            def reads(reqs, cache=None, check=False):
                if dev:
                    out_len, st = ix.read_many_device(d_src, len(s), [r[0] for r in reqs], [r[1] for r in reqs], d_dst,
                                                      [READ * i for i in range(len(reqs))], cache=cache)
                    assert not st.any() and (out_len == READ).all()
                    got = d_dst[: READ * len(reqs)].cpu().numpy().tobytes() if check else None
                else:
                    outs, st = ix.read_many(s, reqs, cache=cache)
                    assert not any(st)
                    got = b"".join(outs)
                if check:
                    assert got == b"".join(x[o: o + n].tobytes() for o, n in reqs)

            caches = {f: ctx.block_cache(int(f * N)) for f in (0.25, 0.5, 1.0)}
            full = caches[1.0]

            def reader_at_cached():
                full.clear()
                for r in seq:
                    reads([r], full)

            spread = seq[:: len(seq) // a.singles][: a.singles]  # every block of the 8 alike, since their decode times differ

            def reader_at_uncached():
                for r in spread:
                    reads([r])

            def zipf(cache):
                """the 10 calls -> (ms per call, hit rate)"""
                if cache is not None:
                    cache.clear()
                    h0, m0 = cache.stats["hits"], cache.stats["misses"]
                per = [timed(lambda: reads(z, cache))[1] for z in zipf_sets]
                rate = None
                if cache is not None:
                    h, m = cache.stats["hits"] - h0, cache.stats["misses"] - m0
                    rate = h / max(h + m, 1)
                return per, rate

            def no_hits():
                full.clear()
                reads(uniform, full)

            # warm-up and checks of every arm
            for r in seq[:3] + seq[-2:]:
                reads([r], full, check=True)
            reads(zipf_sets[0], check=True)
            reads(zipf_sets[0], full, check=True)
            reads(zipf_sets[0], full, check=True)
            no_hits()
            reads(uniform, check=True)
            ms = {k: [] for k in ("reader_at_cached", "reader_at_uncached_scaled", "no_hits_cached", "no_hits_uncached")}
            zms = {k: [] for k in ("uncached", "0.25", "0.5", "1.0")}
            zfirst = {k: [] for k in zms}
            rates = {}
            for rep in range(a.reps):
                ms["reader_at_cached"].append(timed(reader_at_cached)[1])
                ms["reader_at_uncached_scaled"].append(timed(reader_at_uncached)[1] * len(seq) / a.singles)
                ms["no_hits_cached"].append(timed(no_hits)[1])
                ms["no_hits_uncached"].append(timed(lambda: reads(uniform))[1])
                for k, c in (("uncached", None), ("0.25", caches[0.25]), ("0.5", caches[0.5]), ("1.0", full)):
                    per, rate = zipf(c)
                    zms[k].append(float(np.median(per)))
                    zfirst[k].append(per[0])
                    rates[k] = rate
            med = {k: round(float(np.median(v)), 2) for k, v in ms.items()}
            # hashing alone, and what a miss-only call inserts
            ctx.profile(True)
            ctx.profile_reset()
            no_hits()
            hash_ms = ctx.kernel_time("record_hash")[1] if dev else ctx.kernel_time("host:record_hash")[1]
            ins = ctx.stage_bytes("read:cache_insert")[1:]
            ctx.profile(False)
            ctx.profile_reset()
            for c in caches.values():
                c.close()
            line = json.dumps({
                "level": level, "transform": tr, "entropy": en, "variant": variant, "input_bytes": N, "stream_bytes": int(len(s)), "blocks": nblocks,
                "read_bytes": READ,
                "reader_at": {"calls": len(seq), "blocks": SEQ_BLOCKS, "cached_ms_total": med["reader_at_cached"],
                              "uncached_ms_total_scaled": med["reader_at_uncached_scaled"], "uncached_calls_timed": a.singles,
                              "cached_ms_per_read": round(med["reader_at_cached"] / len(seq), 3),
                              "uncached_ms_per_read": round(med["reader_at_uncached_scaled"] / len(seq), 3)},
                "zipf": {"requests_per_call": NREQ, "calls": CALLS,
                         "ms_per_call_median": {k: round(float(np.median(v)), 2) for k, v in zms.items()},
                         "first_call_ms": {k: round(float(np.median(v)), 2) for k, v in zfirst.items()},
                         "hit_rate": {k: round(v, 3) for k, v in rates.items() if v is not None}},
                "no_hits": {"requests": NREQ, "cached_ms": med["no_hits_cached"], "uncached_ms": med["no_hits_uncached"],
                            "record_hash_ms": round(hash_ms, 2), "inserted_blocks": ins[0], "inserted_bytes": ins[1]},
                "reps": a.reps, "gpu": name, "power_limit": pl})
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
