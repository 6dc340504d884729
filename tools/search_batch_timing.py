"""One lb2_index_search_batch call over queries with mixed parameters, against what the single-parameter calls need
for the same work, at the C1 shape (synth.sift_like: 1 M x 128 f32, IVF_PQ(256, 16)).

    python tools/search_batch_timing.py [--n 1000000] [--nq 10000] [--per-query 1000] [--reps 3] [--out FILE]

The mixed batch: k in {10, 50, 100}, nprobes in {5, 10, 20, 50} with a quarter of the queries at minimum 1 / maximum
None instead, refine factor 0 or 10, and 30 % of the queries under one of 64 allow lists of ~50 % of the rows (bitmaps
staged on the device once).  Cases, each timed in this run with
CUDA events around the whole blocking call (host outputs included), median of --reps after a warm-up:
  batch            one search_batch call;
  per_param_set    one search_ex (search_probed for the minimum / maximum queries) call per distinct
                   (k, nprobes, refine factor, filter) set;
  per_query        one such call per query, over the first --per-query queries (QPS over those);
  uniform_search / uniform_batch   the plain C1 batch (k = 10, nprobes = 10) through search and search_batch.
The kernel launches of the batch call (lb2_launch_count) and the card's name and power limit are recorded; so is the
fixed-probe part of the mix alone through search_batch (fixed_only).  Results go to FILE as JSON (default
search_batch_timing.json)."""
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
    out = call()
    ts = []
    for _ in range(reps):
        lb.timer_start()
        out = call()
        ts.append(lb.timer_stop())
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--per-query", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="search_batch_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("search_batch_timing: no CUDA device (nothing is measured without one)")
    d, K = 128, 256
    x = synth.sift_like(a.n, d)
    q = synth.sift_like_queries(a.nq, d)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    xd = lb.DeviceArray.from_numpy(x)
    ix = lb.IvfPqIndex.build(xd, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, seed=0))
    rid = ix.export()["row_ids"]
    rng = np.random.default_rng(0)
    nq = a.nq
    k = rng.choice([10, 50, 100], nq)
    nprobes = np.where(rng.random(nq) < 0.25, 0, rng.choice([5, 10, 20, 50], nq))  # 0: minimum 1 / maximum None
    rf = rng.choice([0, 10], nq)
    rf[k * np.maximum(rf, 1) > 1024] = 0  # k' <= 1024
    filters = [lb.DeviceArray.from_numpy(ix.row_mask(rng.choice(rid, len(rid) // 2, replace=False), None))
               for _ in range(64)]
    fof = np.where(rng.random(nq) < 0.3, rng.integers(0, 64, nq), -1)
    res = {"card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "nq": nq,
           "mix": "k {10,50,100}, nprobes {5,10,20,50} or (25%) min 1 / max None, refine 0/10, "
                  "30% under one of 64 ~50% allow lists",
           "cases": {}}

    def record(name, ms, queries, **extra):
        res["cases"][name] = {"ms": ms, "queries": queries, "qps": queries / (ms / 1e3), **extra}
        print(name, res["cases"][name], flush=True)

    batch = lambda: ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=xd, filters=filters,  # noqa
                                    filter_of=fof)
    ms, _ = timed(batch, a.reps)
    lb.launch_count(reset=True)
    batch()
    launches = lb.launch_count(reset=True)
    record("batch", ms, nq, launches=launches)
    fx = np.nonzero(nprobes > 0)[0]
    qf = np.ascontiguousarray(q[fx])
    ms, _ = timed(lambda: ix.search_batch(qf, k[fx], nprobes=nprobes[fx], refine_factor=rf[fx], vectors=xd,
                                          filters=filters, filter_of=fof[fx]), a.reps)
    record("fixed_only_batch", ms, len(fx))

    def one(qs, kk, p, r, f):
        kw = dict(refine_factor=r, vectors=xd if r else None, allow_bitmap=filters[f] if f >= 0 else None)
        if p:
            ix.search_ex(qs, k=kk, nprobes=p, **kw)
        else:
            ix.search_probed(qs, kk, **kw)

    sets = {}
    for i in range(nq):
        sets.setdefault((int(k[i]), int(nprobes[i]), int(rf[i]), int(fof[i])), []).append(i)
    groups = [(key, np.array(v), np.ascontiguousarray(q[v])) for key, v in sets.items()]

    def per_set():
        for (kk, p, r, f), _, qs in groups:
            one(qs, kk, p, r, f)
    ms, _ = timed(per_set, a.reps)
    record("per_param_set", ms, nq, calls=len(groups))

    m = min(a.per_query, nq)

    def per_query():
        for i in range(m):
            one(q[i:i + 1], int(k[i]), int(nprobes[i]), int(rf[i]), int(fof[i]))
    ms, _ = timed(per_query, a.reps)
    record("per_query", ms, m, calls=m)

    ms, _ = timed(lambda: ix.search(q, k=10, nprobes=10), a.reps)
    record("uniform_search", ms, nq)
    ms, _ = timed(lambda: ix.search_batch(q, 10, nprobes=10), a.reps)
    record("uniform_batch", ms, nq)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
