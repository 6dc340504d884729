"""Searches with minimum / maximum nprobes next to fixed-nprobes searches at the C1 shape (synth.sift_like:
1 M x 128 f32, IVF_PQ(256, 16)).

    python tools/probe_timing.py [--n 1000000] [--nq 10000] [--reps 3] [--out FILE]

Cases, all at k = 10: search_ex with nprobes 10; the default query (minimum 1, maximum None); the default query under
allow lists of about 1 % and 0.01 % of the rows (bitmap, max_len and the ids, late_width 16); and minimum = maximum =
10 through lb2_index_search_probed.  Each case reports QPS (CUDA events around the whole blocking call, host outputs
included, median of --reps after a warm-up) and the mean number of partitions searched.  The card's name and power
limit are recorded.  Results go to FILE as JSON (default probe_timing.json)."""
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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="probe_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("probe_timing: no CUDA device (nothing is measured without one)")
    d, K, k = 128, 256, 10
    x = synth.sift_like(a.n, d)
    q = synth.sift_like_queries(a.nq, d)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ix = lb.IvfPqIndex.build(lb.DeviceArray.from_numpy(x), "l2",
                             lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, seed=0))
    rid = ix.export()["row_ids"]
    rng = np.random.default_rng(0)
    res = {"card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "nq": a.nq, "k": k, "cases": {}}

    def record(name, ms, nprobes):
        res["cases"][name] = {"ms": ms, "qps": a.nq / (ms / 1e3), "mean_partitions_searched": nprobes}
        print(name, res["cases"][name], flush=True)

    ms, _ = timed(lambda: ix.search_ex(q, k=k, nprobes=10), a.reps)
    record("search_ex_nprobes10", ms, 10.0)
    ms, out = timed(lambda: ix.search_probed(q, k), a.reps)
    record("default_min1_maxNone", ms, float(out[3].mean()))
    for label, frac in (("filter_1pct", 0.01), ("filter_0.01pct", 0.0001)):
        allow = np.sort(rng.choice(rid, max(1, int(a.n * frac)), replace=False))
        bm = ix.row_mask(allow, None)
        ms, out = timed(lambda: ix.search_probed(q, k, allow_bitmap=bm, mask_ids=allow, mask_max_len=len(allow),
                                                 late_width=16), a.reps)
        record(label, ms, float(out[3].mean()))
    ms, out = timed(lambda: ix.search_probed(q, k, minimum_nprobes=10, maximum_nprobes=10), a.reps)
    record("probed_min10_max10", ms, float(out[3].mean()))
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
