"""knn_combined and flat KNN for mixed query batches: one lb2_index_search_combined_batch call against one
lb2_index_search_combined call per distinct parameter set, and one lb2_flat_search_batch call against one
lb2_flat_search call per distinct parameter set, at the C1 shape (synth.sift_like: 1 M x 128 f32, IVF_PQ(256, 16)).

    python tools/combined_batch_timing.py [--n 1000000] [--nq 2000] [--flat-nq 1000] [--reps 1] [--out FILE]

The mixed batch: k in 1..100, refine factor 0..10, nprobes in {5, 10, 20, 50} with a quarter of the queries at
minimum 1 / maximum None instead, and 30 % of the queries under one of 64 allow lists of ~50 % of the indexed rows,
each with its own bitmap of ~50 % of the unindexed rows.  On top of the index, 10 000 and 100 000 appended unindexed
rows (device-resident).  Cases, each timed in this run with CUDA events around the whole blocking call (host outputs
included), median of --reps after a warm-up:
  combined_batch / combined_per_set   per unindexed size: one search_combined_batch call / one search_combined call
                                      per distinct (k, nprobes, refine factor, filter) set;
  flat_batch / flat_per_set           flat KNN over the 1 M rows (device-resident) for the first --flat-nq queries,
                                      each with its own k, filter (64 bitmaps of ~50 %) and, for 20 %, a range.
The kernel launches of every case (lb2_launch_count) and the card's name and power limit are recorded.  Results go to
FILE as JSON (default combined_batch_timing.json)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lance_b200 as lb  # noqa: E402
from lance_b200 import synth  # noqa: E402


def timed(call, reps):
    call()
    ts = []
    for _ in range(reps):
        lb.timer_start()
        call()
        ts.append(lb.timer_stop())
    lb.launch_count(reset=True)
    call()
    return float(np.median(ts)), lb.launch_count(reset=True)


def bits(mask):
    b = np.zeros((len(mask) + 63) // 64 * 64, np.uint8)
    b[:len(mask)] = mask
    return np.packbits(b.reshape(-1, 8)[:, ::-1]).view(np.uint64).copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=2000)
    ap.add_argument("--flat-nq", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--out", default="combined_batch_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("combined_batch_timing: no CUDA device (nothing is measured without one)")
    d, K, extra = 128, 256, (10_000, 100_000)
    x = synth.sift_like(a.n + max(extra), d)
    q = synth.sift_like_queries(a.nq, d)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    xd = lb.DeviceArray.from_numpy(x[:a.n])
    ix = lb.IvfPqIndex.build(xd, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, seed=0))
    rid = ix.export()["row_ids"]
    rng = np.random.default_rng(0)
    nq = a.nq
    k = rng.integers(1, 101, nq)
    rf = rng.integers(0, 11, nq)
    nprobes = np.where(rng.random(nq) < 0.25, 0, rng.choice([5, 10, 20, 50], nq))  # 0: minimum 1 / maximum None
    filters = [lb.DeviceArray.from_numpy(ix.row_mask(rng.choice(rid, len(rid) // 2, replace=False), None))
               for _ in range(64)]
    fof = np.where(rng.random(nq) < 0.3, rng.integers(0, 64, nq), -1)
    res = {"card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "nq": nq,
           "mix": "k 1..100, refine 0..10, nprobes {5,10,20,50} or (25%) min 1 / max None, "
                  "30% under one of 64 ~50% allow lists (and ~50% of the unindexed rows)",
           "cases": {}}

    def record(name, ms, queries, launches, **more):
        res["cases"][name] = {"ms": ms, "queries": queries, "qps": queries / (ms / 1e3), "launches": launches, **more}
        print(name, res["cases"][name], flush=True)

    sets = {}
    for i in range(nq):
        sets.setdefault((int(k[i]), int(nprobes[i]), int(rf[i]), int(fof[i])), []).append(i)
    groups = [(key, np.ascontiguousarray(q[v])) for key, v in sets.items()]
    for m in extra:
        ux = lb.DeviceArray.from_numpy(x[a.n:a.n + m])
        urid = lb.DeviceArray.from_numpy(np.arange(a.n, a.n + m, dtype=np.uint64))
        uf = [lb.DeviceArray.from_numpy(bits(rng.random(m) < 0.5)) for _ in range(64)]
        kw = dict(vectors=xd, unindexed_vectors=ux, unindexed_row_ids=urid)
        ms, launches = timed(lambda: ix.search_combined_batch(q, k, nprobes=nprobes, refine_factor=rf, filters=filters,
                                                              filter_of=fof, unindexed_filters=uf, **kw), a.reps)
        record(f"combined_batch_{m}", ms, nq, launches, unindexed=m)

        def per_set():
            for (kk, p, r, f), qs in groups:
                ix.search_combined(qs, kk, nprobes=p if p else None, refine_factor=r,
                                   allow_bitmap=filters[f] if f >= 0 else None,
                                   unindexed_allow_bitmap=uf[f] if f >= 0 else None, **kw)
        ms, launches = timed(per_set, a.reps)
        record(f"combined_per_set_{m}", ms, nq, launches, unindexed=m, calls=len(groups))
    fq = min(a.flat_nq, nq)
    qf = np.ascontiguousarray(q[:fq])
    fk = k[:fq]
    ff = [lb.DeviceArray.from_numpy(bits(rng.random(a.n) < 0.5)) for _ in range(64)]
    ffof = np.where(rng.random(fq) < 0.3, rng.integers(0, 64, fq), -1)
    hi = np.where(rng.random(fq) < 0.2, np.float32(2e5), np.nan).astype(np.float32)
    ms, launches = timed(lambda: lb.flat_search_batch(xd, qf, fk, "l2", filters=ff, filter_of=ffof, upper_bound=hi),
                         a.reps)
    record("flat_batch", ms, fq, launches, rows=a.n)
    fsets = {}
    for i in range(fq):
        fsets.setdefault((int(fk[i]), int(ffof[i]), float(hi[i])), []).append(i)
    fgroups = [(key, np.ascontiguousarray(qf[v])) for key, v in fsets.items()]

    def flat_per_set():
        for (kk, f, h), qs in fgroups:
            lb.flat_search(xd, qs, kk, "l2", allow_bitmap=ff[f] if f >= 0 else None,
                           upper_bound=None if np.isnan(h) else h)
    ms, launches = timed(flat_per_set, a.reps)
    record("flat_per_set", ms, fq, launches, rows=a.n, calls=len(fgroups))
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
