"""IVF_HNSW_FLAT next to IVF_FLAT on SIFT-shaped data (synth.sift_like, f32, K = 256, HNSW 7 / 20 / 150): the
1 M x 128 shape, then a 200 k x 768 shape to show how the graph stage and the search grow with d.

    python tools/hnsw_flat_timing.py [--shapes 1000000x128,200000x768] [--nq 1000] [--reps 3] [--out FILE]

Per shape it records the build time of each index (host wall clock around the blocking build; for IVF_HNSW_FLAT also
the graph stage alone, the difference of the two), and for nprobes 1 / 10 at k = 10 the search time (CUDA events
around the whole batched call, median of --reps after a warm-up) as QPS and recall@10 against the exact top-10
(lb.flat_search): IVF_FLAT, and IVF_HNSW_FLAT at ef 15 / 50 / 150.  The graph distances run one lane per row (each lane
walks its row once); the per-shape graph stage and search times are the numbers a half-warp-per-row mapping would have
to beat.  The card's name and power limit are read in the same run.  Results go to FILE as JSON (default
hnsw_flat_timing.json)."""
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


def one_shape(n, d, K, nq, reps):
    data = synth.sift_like(n, d)
    queries = synth.sift_like_queries(nq, d)
    k = 10
    truth, _, _ = lb.flat_search(data, queries, k)
    hp = lb.HnswBuildParams(max_level=7, m=20, ef_construction=150)
    out = dict(shape=dict(n=n, d=d, K=K, nq=nq, k=k, dtype="f32", data="synth.sift_like"))
    t0 = time.perf_counter()
    flat = lb.IvfFlatIndex.build(data, "l2", num_partitions=K)
    lb.synchronize()
    flat_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    hn = lb.IvfHnswFlatIndex.build(data, "l2", num_partitions=K, hnsw_params=hp)
    lb.synchronize()
    hn_s = time.perf_counter() - t0
    sizes = np.diff(hn.export()["part_offsets"].astype(np.int64))
    out["build_s"] = dict(ivf_flat=flat_s, ivf_hnsw_flat=hn_s, graph_stage=hn_s - flat_s,
                          hnsw_params=dict(max_level=7, m=20, ef_construction=150),
                          partition_rows=dict(min=int(sizes.min()), median=float(np.median(sizes)),
                                              max=int(sizes.max())))
    print(json.dumps(out), flush=True)
    rows = []
    for nprobes in (1, 10):
        ms = timed(lambda: flat.search(queries, k=k, nprobes=nprobes), reps)
        ids, _ = flat.search(queries, k=k, nprobes=nprobes)
        rows.append(dict(index="ivf_flat", nprobes=nprobes, ef=None, ms=ms, qps=nq / ms * 1e3,
                         recall_at_10=recall(ids, truth)))
        for ef in (15, 50, 150):
            ms = timed(lambda: hn.search(queries, k=k, nprobes=nprobes, ef=ef), reps)
            ids, _ = hn.search(queries, k=k, nprobes=nprobes, ef=ef)
            rows.append(dict(index="ivf_hnsw_flat", nprobes=nprobes, ef=ef, ms=ms, qps=nq / ms * 1e3,
                             recall_at_10=recall(ids, truth)))
        print(json.dumps(rows[-4:]), flush=True)
    out["search"] = rows
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1000000x128,200000x768")
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="hnsw_flat_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("hnsw_flat_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = dict(card=card, distance_mapping="one lane per row, rows walked once in 16-element chunks",
               cpu_restatement_build="not measured: the restatement is pure Python with an n_p x n_p distance "
                                     "matrix per partition, not sized for these shapes",
               runs=[])
    for s in a.shapes.split(","):
        n, d = (int(v) for v in s.split("x"))
        out["runs"].append(one_shape(n, d, a.K, a.nq, a.reps))
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
