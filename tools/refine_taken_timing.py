"""A refined batch three ways at the C1 shape (synth.sift_like: 1 M x 128 f32, IVF_PQ(256, 16)): nq 10 000, k 10,
refine factor 10, nprobes 10.

    python tools/refine_taken_timing.py [--n 1000000] [--nq 10000] [--reps 5] [--out FILE]

  device_column   search_batch with the raw column in device memory;
  pinned_column   search_batch with the raw column in pinned host memory (the whole column is copied per call);
  taken           search_candidates(distinct=True), a host take of the distinct rows from the pinned column into a
                  pinned buffer, then refine_taken on those rows.

Device phases are timed with CUDA events around each blocking call (host outputs included), the host take with a
host clock; each is the median of --reps after a warm-up.  Host-to-device bytes are the inputs each path copies.
The three results are checked equal bit for bit.  The card's name and power limit are read in the same run.
Results go to FILE as JSON (default refine_taken_timing.json)."""
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="refine_taken_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("refine_taken_timing: no CUDA device (nothing is measured without one)")
    d, K, k, rf, nprobes = 128, 256, 10, 10, 10
    x = synth.sift_like(a.n, d)
    q = synth.sift_like_queries(a.nq, d)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    xd = lb.DeviceArray.from_numpy(x)
    xp = lb.PinnedArray(x.shape, np.float32)
    xp.array[:] = x
    ix = lb.IvfPqIndex.build(xd, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, seed=0))
    nq, kc = a.nq, k * rf
    small_in = q.nbytes + nq * 44  # queries and the lb2_query_params table
    res = {"card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "nq": nq, "k": k, "refine_factor": rf,
           "nprobes": nprobes, "cases": {}}

    def record(name, **v):
        res["cases"][name] = v
        print(name, v, flush=True)

    ms, want = timed(lambda: ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=xd), a.reps)
    record("device_column", ms=ms, h2d_bytes=small_in)
    ms, got = timed(lambda: ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=xp), a.reps)
    assert all(np.array_equal(g.view(np.uint8), w.view(np.uint8)) for g, w in zip(got, want))
    record("pinned_column", ms=ms, h2d_bytes=small_in + x.nbytes)

    ms_c, cand = timed(lambda: ix.search_candidates(q, k, nprobes=nprobes, refine_factor=rf, distinct=True), a.reps)
    ci, cd, cc, cn, uniq, pos = cand
    m = len(uniq)
    taken = lb.PinnedArray((m, d), np.float32)
    rows = uniq.astype(np.int64)
    ts = []
    for _ in range(a.reps + 1):
        t0 = time.perf_counter()
        np.take(xp.array, rows, axis=0, out=taken.array)
        ts.append((time.perf_counter() - t0) * 1e3)
    ms_t = float(np.median(ts[1:]))
    ts = []
    for _ in range(a.reps + 1):  # the same take from a pageable copy of the column, for comparison
        t0 = time.perf_counter()
        np.take(x, rows, axis=0, out=taken.array)
        ts.append((time.perf_counter() - t0) * 1e3)
    ms_tp = float(np.median(ts[1:]))
    np.take(xp.array, rows, axis=0, out=taken.array)
    ms_r, got = timed(lambda: ix.refine_taken(q, (ci, cd, cc), taken, pos, k, rf), a.reps)
    assert all(np.array_equal(g.view(np.uint8), w.view(np.uint8)) for g, w in zip(got, want[:3]))
    assert np.array_equal(cn, want[3])
    cand_bytes = ci.nbytes + cd.nbytes + cc.nbytes + pos.nbytes  # the lists go back to the device for the re-rank
    record("taken", ms=ms_c + ms_t + ms_r, ms_candidates=ms_c, ms_host_take=ms_t, ms_host_take_from_pageable=ms_tp, ms_refine_taken=ms_r,
           h2d_bytes=2 * small_in + cand_bytes + taken.nbytes, taken_bytes=taken.nbytes, m=m, slots=nq * kc,
           m_over_slots=m / (nq * kc))
    taken.free()
    xp.free()
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
