"""Time the partition index (lb2_partition_index_build / _assign) against the exact scan (lb2_compute_partitions).

For each shape (K centroids x d) and data kind it trains nothing: the centroids are synthetic (see `centroids`) and
the rows are centroids plus noise (0.5 per element), generated on the host from a seed and copied to the device once, so the timed calls
read device-resident rows.  It reports, per shape:
  - the graph build's wall time (serial, and at --insert-batch), blocking calls;
  - the assignment's wall time through the graph and through the exact scan, median of --repeats after a warm-up;
  - the agreement rate of the two assignments, and the ratio of the graph's loss (the sum of the row-to-centroid
    distances, f64) to the exact loss;
  - the card's name, power limit and maximum SM clock, read in the same run.
One JSON line goes to stdout and to --out.

  python tools/partition_index_timing.py --rows 1000000 --out profiles/partition_index_h100.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import lance_b200 as lb  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def wall(f):
    lb.synchronize()
    t0 = time.perf_counter()
    out = f()
    lb.synchronize()
    return time.perf_counter() - t0, out


def centroids(K, d, data, rng):
    """normal: K standard-normal rows, no structure (every centroid nearly equidistant in high d); mixture: 64 standard-
    normal component means, each centroid its component's mean plus 0.35 x normal noise, so centroids have near
    neighbours as trained k-means models do"""
    if data == "normal":
        return rng.standard_normal((K, d), dtype=np.float32)
    means = rng.standard_normal((64, d), dtype=np.float32)
    return means[rng.integers(0, 64, K)] + np.float32(0.35) * rng.standard_normal((K, d), dtype=np.float32)


def shape(K, d, n, batch, repeats, seed, data):
    rng = np.random.default_rng(seed)
    cent = centroids(K, d, data, rng)
    rows = np.empty((n, d), np.float32)
    for r0 in range(0, n, 65536):
        r1 = min(n, r0 + 65536)
        rows[r0:r1] = cent[rng.integers(0, K, r1 - r0)] + np.float32(0.5) * rng.standard_normal((r1 - r0, d),
                                                                                                  dtype=np.float32)
    drows = lb.DeviceArray.from_numpy(rows)
    del rows
    out = dict(K=K, d=d, rows=n, metric="l2", data=data)
    builds = {}
    for b in (1, batch):
        t, pi = wall(lambda: lb.PartitionIndex.build(cent, "l2", mode="hnsw", seed=seed, insert_batch=b))
        builds[b] = pi
        out[f"build_s_insert_batch_{b}"] = round(t, 4)
    pi = builds[batch]
    pi.assign(drows)                                 # warm-up
    lb.compute_partitions(cent, drows, "l2")
    tg, te = [], []
    for _ in range(repeats):                         # alternate the two paths
        t, (gp, gd, gv) = wall(lambda: pi.assign(drows))
        tg.append(t)
        t, (ep, ed, ev) = wall(lambda: lb.compute_partitions(cent, drows, "l2"))
        te.append(t)
    out["assign_graph_s_median"] = round(float(np.median(tg)), 4)
    out["assign_exact_s_median"] = round(float(np.median(te)), 4)
    out["assign_graph_s_all"] = [round(v, 4) for v in tg]
    out["assign_exact_s_all"] = [round(v, 4) for v in te]
    out["graph_rows_per_s"] = round(n / float(np.median(tg)))
    out["exact_rows_per_s"] = round(n / float(np.median(te)))
    both = gv & ev
    out["valid_graph"], out["valid_exact"] = int(gv.sum()), int(ev.sum())
    out["agreement"] = float((gp[both] == ep[both]).mean())
    out["loss_ratio"] = float(gd[both].astype(np.float64).sum() / ed[both].astype(np.float64).sum())
    out["graph_from_insert_batch"] = batch
    same = builds[1].assign(drows)
    out["serial_graph_agreement"] = float((same[0][both] == gp[both]).mean())
    for p in builds.values():
        p.close()
    drows.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--shapes", default="4096x768,65536x128")
    ap.add_argument("--data", default="normal,mixture")
    ap.add_argument("--insert-batch", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("partition_index_timing: no CUDA device (there is no CPU fallback)")
    res = dict(tool="partition_index_timing", card=card(), shapes=[])
    for data in a.data.split(","):
        for s in a.shapes.split(","):
            K, d = (int(v) for v in s.split("x"))
            res["shapes"].append(shape(K, d, a.rows, a.insert_batch, a.repeats, a.seed, data))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
