"""IVF_HNSW_SQ next to IVF_SQ on SIFT-shaped data (synth.sift_like: 1 M x 128 f32, K = 256).

    python tools/hnsw_timing.py [--n 1000000] [--nq 1000] [--reps 3] [--out FILE]

Records the build time of each index (host wall clock around the blocking build; for IVF_HNSW_SQ also the graph
stage alone, the difference of the two), and for nprobes 1 / 10 at k = 10 the search time (CUDA events around the
whole batched call, median of --reps after a warm-up) as QPS and recall@10 against the exact top-10 (lb.flat_search),
IVF_HNSW_SQ at ef 15 / 50 / 150.  The CPU restatement of the graph build (tests/hnsw_reference.py) is pure Python
and precomputes an n_p x n_p distance matrix per partition, so no CPU build time at this size is recorded.  The
card's name and power limit are recorded.  Results go to FILE as JSON (default hnsw_timing.json)."""
import argparse
import json
import os
import subprocess
import sys
import time

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
    return float(np.median(ts))


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / truth.shape[1] for a, b in zip(ids, truth)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="hnsw_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("hnsw_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    data = synth.sift_like(a.n, a.d)
    queries = synth.sift_like_queries(a.nq, a.d)
    k = 10
    truth, _, _ = lb.flat_search(data, queries, k)
    out = dict(card=card, shape=dict(n=a.n, d=a.d, K=a.K, nq=a.nq, k=k, data="synth.sift_like"),
               cpu_restatement_build="not measured: the restatement is pure Python with an n_p x n_p distance matrix"
                                     " per partition, not sized for 1 M rows")
    t0 = time.perf_counter()
    sq = lb.IvfSqIndex.build(data, "l2", num_partitions=a.K)
    lb.synchronize()
    sq_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    hn = lb.IvfHnswSqIndex.build(data, "l2", num_partitions=a.K)
    lb.synchronize()
    hn_s = time.perf_counter() - t0
    sizes = np.diff(hn.export()["part_offsets"].astype(np.int64))
    out["build_s"] = dict(ivf_sq=sq_s, ivf_hnsw_sq=hn_s, graph_stage=hn_s - sq_s,
                          hnsw_params=dict(max_level=7, m=20, ef_construction=150),
                          partition_rows=dict(min=int(sizes.min()), median=float(np.median(sizes)),
                                              max=int(sizes.max())))
    rows = []
    for nprobes in (1, 10):
        ms = timed(lambda: sq.search(queries, k=k, nprobes=nprobes), a.reps)
        ids, _ = sq.search(queries, k=k, nprobes=nprobes)
        rows.append(dict(index="ivf_sq", nprobes=nprobes, ef=None, ms=ms, qps=a.nq / ms * 1e3,
                         recall_at_10=recall(ids, truth)))
        for ef in (15, 50, 150):
            ms = timed(lambda: hn.search(queries, k=k, nprobes=nprobes, ef=ef), a.reps)
            ids, _ = hn.search(queries, k=k, nprobes=nprobes, ef=ef)
            rows.append(dict(index="ivf_hnsw_sq", nprobes=nprobes, ef=ef, ms=ms, qps=a.nq / ms * 1e3,
                             recall_at_10=recall(ids, truth)))
        print(json.dumps(rows[-4:]), flush=True)
    out["search"] = rows
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["build_s"]))


if __name__ == "__main__":
    main()
