"""IVF_HNSW_PQ next to IVF_PQ on SIFT-shaped data (synth.sift_like: 1 M x 128 f32, K = 256, PQ 16 x 8-bit, HNSW 7 / 20
/ 150).

    python tools/hnsw_pq_timing.py [--n 1000000] [--nq 1000] [--reps 3] [--out FILE]

Records the build time of each index (host wall clock around the blocking build; for IVF_HNSW_PQ also the graph stage
alone, the difference of the two), and for nprobes 1 / 10 at k = 10 the search time (CUDA events around the whole
batched call, median of --reps after a warm-up) as QPS and recall@10 against the exact top-10 (lb.flat_search):
IVF_PQ, IVF_PQ with refine factor 10, and IVF_HNSW_PQ at ef 15 / 50 / 150.

Where the graph search's time goes: every (query, partition) slot first builds the residual query's M x 256 table,
then walks the graph.  Both run in one kernel, so the table's share is bounded from above by a search at k = 1, ef = 1
(the traversal is then the greedy descent and one expansion per level 0 step); the rest of a search at ef is the
traversal.  The card's name and power limit are recorded.  Results go to FILE as JSON (default
hnsw_pq_timing.json)."""
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
    ap.add_argument("--out", default="hnsw_pq_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("hnsw_pq_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    data = synth.sift_like(a.n, a.d)
    queries = synth.sift_like_queries(a.nq, a.d)
    k = 10
    truth, _, _ = lb.flat_search(data, queries, k)
    params = lb.IvfBuildParams(num_partitions=a.K, num_sub_vectors=16, num_bits=8)
    hp = lb.HnswBuildParams(max_level=7, m=20, ef_construction=150)
    out = dict(card=card, shape=dict(n=a.n, d=a.d, K=a.K, M=16, nbits=8, nq=a.nq, k=k, data="synth.sift_like"),
               cpu_restatement_build="not measured: the restatement is pure Python with two n_p x n_p distance "
                                     "matrices per partition, not sized for 1 M rows")
    t0 = time.perf_counter()
    pq = lb.IvfPqIndex.build(data, "l2", params)
    lb.synchronize()
    pq_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    hn = lb.IvfHnswPqIndex.build(data, "l2", params, hp)
    lb.synchronize()
    hn_s = time.perf_counter() - t0
    sizes = np.diff(hn.export()["part_offsets"].astype(np.int64))
    out["build_s"] = dict(ivf_pq=pq_s, ivf_hnsw_pq=hn_s, graph_stage=hn_s - pq_s,
                          hnsw_params=dict(max_level=7, m=20, ef_construction=150),
                          partition_rows=dict(min=int(sizes.min()), median=float(np.median(sizes)),
                                              max=int(sizes.max())))
    rows, split = [], []
    for nprobes in (1, 10):
        ms = timed(lambda: pq.search(queries, k=k, nprobes=nprobes), a.reps)
        ids, _ = pq.search(queries, k=k, nprobes=nprobes)
        rows.append(dict(index="ivf_pq", nprobes=nprobes, ef=None, refine_factor=None, ms=ms, qps=a.nq / ms * 1e3,
                         recall_at_10=recall(ids, truth)))
        ms = timed(lambda: pq.search_refine(data, queries, k=k, nprobes=nprobes, refine_factor=10), a.reps)
        ids, _ = pq.search_refine(data, queries, k=k, nprobes=nprobes, refine_factor=10)
        rows.append(dict(index="ivf_pq", nprobes=nprobes, ef=None, refine_factor=10, ms=ms, qps=a.nq / ms * 1e3,
                         recall_at_10=recall(ids, truth)))
        table_ms = timed(lambda: hn.search(queries, k=1, nprobes=nprobes, ef=1), a.reps)
        for ef in (15, 50, 150):
            ms = timed(lambda: hn.search(queries, k=k, nprobes=nprobes, ef=ef), a.reps)
            ids, _ = hn.search(queries, k=k, nprobes=nprobes, ef=ef)
            rows.append(dict(index="ivf_hnsw_pq", nprobes=nprobes, ef=ef, refine_factor=None, ms=ms,
                             qps=a.nq / ms * 1e3, recall_at_10=recall(ids, truth)))
            split.append(dict(nprobes=nprobes, ef=ef, search_ms=ms, table_bound_ms=table_ms,
                              table_share_at_most=min(1.0, table_ms / ms)))
        print(json.dumps(rows[-5:]), flush=True)
    out["search"] = rows
    out["table_vs_traversal"] = dict(
        method="table_bound_ms: a k = 1, ef = 1 search with the same nprobes (every slot builds its table, the "
               "traversal is the greedy descent); an upper bound of the table build's time",
        rows=split)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["build_s"]))


if __name__ == "__main__":
    main()
