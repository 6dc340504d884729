"""The graph stage of IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT at insert_batch B = 1, 16, 64 and 256 on SIFT-shaped
data (synth.sift_like: 1 M x 128 f32, K = 256, max_level 7, m 20, ef_construction 150).

    python tools/hnsw_batch_timing.py [--n 1000000] [--nq 1000] [--batches 1,16,64,256] [--out FILE]

For each kind the base index (IVF_SQ, IVF_PQ 16 x 8-bit, IVF_FLAT) is built once and timed; each graph build is timed
with a host wall clock around the blocking build, and its graph stage is the difference.  B = 1 is timed twice: the
serial kernel (one warp per partition) and the round driver with one-node rounds (LB2_HNSW_ROUNDS=1, the same
graph).  Every build's recall@10 at nprobes 10, ef 50 against the exact top-10 (lb.flat_search) is recorded, with
whether its graph equals the serial one.  The card's name and power limit are read in the same call.  Results go to
FILE as JSON (default hnsw_batch_timing.json)."""
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


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / truth.shape[1] for a, b in zip(ids, truth)]))


def wall(build):
    t0 = time.perf_counter()
    ix = build()
    lb.synchronize()
    return ix, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--batches", default="1,16,64,256")
    ap.add_argument("--kinds", default="sq,flat,pq")
    ap.add_argument("--out", default="hnsw_batch_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("hnsw_batch_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    data = synth.sift_like(a.n, a.d)
    queries = synth.sift_like_queries(a.nq, a.d)
    k, nprobes, ef = 10, 10, 50
    truth, _, _ = lb.flat_search(data, queries, k)
    out = dict(card=card, shape=dict(n=a.n, d=a.d, K=a.K, nq=a.nq, k=k, nprobes=nprobes, ef=ef,
                                     data="synth.sift_like"),
               hnsw_params=dict(max_level=7, m=20, ef_construction=150), kinds={})
    pq_params = lb.IvfBuildParams(num_partitions=a.K, num_sub_vectors=16)
    base = {"sq": lambda: lb.IvfSqIndex.build(data, "l2", num_partitions=a.K),
            "flat": lambda: lb.IvfFlatIndex.build(data, "l2", num_partitions=a.K),
            "pq": lambda: lb.IvfPqIndex.build(data, "l2", pq_params)}
    graph = {"sq": lambda hp: lb.IvfHnswSqIndex.build(data, "l2", num_partitions=a.K, hnsw_params=hp),
             "flat": lambda hp: lb.IvfHnswFlatIndex.build(data, "l2", num_partitions=a.K, hnsw_params=hp),
             "pq": lambda hp: lb.IvfHnswPqIndex.build(data, "l2", pq_params, hp)}
    batches = [int(b) for b in a.batches.split(",")]
    for kind in a.kinds.split(","):
        ix, base_s = wall(base[kind])
        del ix
        rows, serial = [], None
        runs = [(1, "serial")] + [(b, "rounds") for b in batches if b == 1] + [(b, "rounds") for b in batches if b > 1]
        for b, engine in runs:
            if engine == "rounds" and b == 1:
                os.environ["LB2_HNSW_ROUNDS"] = "1"
            ix, s = wall(lambda: graph[kind](lb.HnswBuildParams(insert_batch=b)))
            os.environ.pop("LB2_HNSW_ROUNDS", None)
            g = ix.export()["graph"]
            if serial is None:
                serial = g
            same = all(np.array_equal(np.asarray(g[key]).view(np.uint8), np.asarray(serial[key]).view(np.uint8))
                       for key in ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up",
                                   "dists_up"))
            ids, _ = ix.search(queries, k=k, nprobes=nprobes, ef=ef)
            rows.append(dict(insert_batch=b, engine=engine, build_s=s, graph_stage_s=s - base_s,
                             recall_at_10=recall(ids, truth), graph_equals_serial=bool(same)))
            print(kind, json.dumps(rows[-1]), flush=True)
            del ix, g
        out["kinds"][kind] = dict(base_build_s=base_s, runs=rows)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
