"""IVF_RQ next to IVF_SQ and IVF_PQ(256, 16) on C1-shaped data (synth.sift_like: 1 M x 128 f32, K = 256).

    python tools/rq_timing.py [--n 1000000] [--nq 10000] [--reps 3] [--out FILE]

For each index: the build time (the library's CUDA-event stage times: for IVF_RQ the rotation is `quantizer_train`,
the residual rotation and encode `transform`), and for nprobes 1 / 10 / 50 at k = 10, with and without refine 10, the
search time (CUDA events around the whole batched call, median of --reps after a warm-up) as QPS, and recall@10
against an exact ground truth (IVF_FLAT with nprobes = K).  For the RQ scan it also reports the achieved bytes/s --
the algorithmic bytes, 24 per row (16 code bytes + the two f32 factors) summed over the probed (query, partition)
slots, over the `rq_scan` kernel time from the launch profiler (a separate profiled run) -- and the time of the
query-side rotation kernel.  The card's name and power limit are recorded.  Results go to FILE as JSON (default
rq_timing.json)."""
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
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="rq_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("rq_timing: no CUDA device (nothing is measured without one)")
    d, K, k, nprobe_list = 128, 256, 10, (1, 10, 50)
    x = synth.sift_like(a.n, d)
    q = synth.sift_like_queries(a.nq, d)
    xd, qd = lb.DeviceArray.from_numpy(x), lb.DeviceArray.from_numpy(q)
    oi, od = lb.DeviceArray((a.nq, k), np.uint64), lb.DeviceArray((a.nq, k), np.float32)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "nq": a.nq, "k": k, "indexes": {}}

    builds = {
        "IVF_RQ": lambda: lb.IvfRqIndex.build(xd, "l2", num_partitions=K, seed=0),
        "IVF_SQ": lambda: lb.IvfSqIndex.build(xd, "l2", num_partitions=K, seed=0),
        "IVF_PQ_256x16": lambda: lb.IvfPqIndex.build(xd, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16,
                                                                                  seed=0)),
    }
    idx = {}
    for name, b in builds.items():
        b()  # warm-up build (module loading, pool growth)
        ix = b()
        st = ix.stats
        idx[name] = ix
        res["indexes"][name] = {"build_ms": {"total": st.ms_total, "ivf_train": st.ms_ivf_train,
                                             "quantizer_train": st.ms_pq_train, "transform": st.ms_transform,
                                             "group": st.ms_group}, "search": {}}
    fl = lb.IvfFlatIndex.build(xd, "l2", num_partitions=K, seed=0)
    gt, _ = fl.search(q, k=k, nprobes=K)
    del fl

    def recall(ids):
        return float(np.mean([len(set(r.tolist()) & set(g.tolist())) / k for r, g in zip(ids, gt)]))

    for name, ix in idx.items():
        for npb in nprobe_list:
            for rf in (0, 10):
                if rf:
                    call = lambda: ix.search_refine(xd, qd, k=k, nprobes=npb, refine_factor=rf, out=(oi, od))  # noqa: E731
                else:
                    call = lambda: ix.search(qd, k=k, nprobes=npb, out=(oi, od))  # noqa: E731
                ms = timed(call, a.reps)
                res["indexes"][name]["search"][f"nprobes{npb}_refine{rf}"] = {
                    "ms": ms, "qps": a.nq / (ms / 1e3), "recall@10": recall(oi.numpy())}

    rq = idx["IVF_RQ"]
    e = rq.export()
    sizes = np.diff(e["part_offsets"].astype(np.int64))
    pids, _ = lb.kmeans_find_partitions(e["centroids"], q, max(nprobe_list), "l2")
    scan = {}
    for npb in nprobe_list:
        rq.search(qd, k=k, nprobes=npb, out=(oi, od))
        lb.profile.enable(True)
        lb.profile.reset()
        rq.search(qd, k=k, nprobes=npb, out=(oi, od))
        lb.synchronize()
        launches, kms = lb.profile.get("search:rq_scan")
        kernels = {name: ms for name, (_, ms) in lb.profile.dump().items()}
        lb.profile.enable(False)
        nbytes = int(sizes[pids[:, :npb]].sum()) * 24
        scan[str(npb)] = {"algorithmic_bytes": nbytes, "rq_scan_ms": kms, "launches": launches,
                          "bytes_per_s": nbytes / (kms / 1e3) if kms else None, "kernel_ms": kernels}
    res["rq_scan"] = scan
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
