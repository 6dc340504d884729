"""Per-launch time of the PQ filter (tc_pq_kernel, family `tc_pq_filter`) and of pq_fallback_kernel on C1-shaped data.

    python tools/pq_filter_timing.py [--n 1000000] [--reps 5] [--out FILE]

Data: synth.sift_like rows (128 f32), 256 IVF centroids trained on a 65 536-row sample, residuals against them.
  (a) a 24-iteration PQ training (16 sub-spaces x 256 codewords) on the 65 536 sample residuals,
  (b) `quantize` of all --n rows (the residual fused in),
each run --reps times after a warm-up under the launch profiler (CUDA events per launch).  Printed per family:
launches, the median over the repetitions of the per-launch time, the scores per second (rows x 16 x 256 per filter
launch) and their share of the ALU-pipe bound.  The bound: the epilogue spends ALU_PER_SCORE min/max or byte-permute
instructions per score, and an SM retires 64 lanes of those per clock (CUDA programming guide, arithmetic throughput
of compute capability 9.0), so peak scores/s = SMs x 64 x clock / ALU_PER_SCORE, with the SM count of the device and
the SM clock read from nvidia-smi in the same run.  The undecided share is the `LB2_TC_STATS` line of one extra call.
The card's name, power limit and clocks are part of the result.  There is no CPU arm: without a GPU the script fails."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lance_b200 as lb  # noqa: E402
from lance_b200 import synth  # noqa: E402

D, K, M, KC, SAMPLE, ITERS = 128, 256, 16, 256, 65536, 24
# tc_common.cuh, top3_half<HALF, 2>: per score half a pair max and half a pack, then three min/max per entrant pair at
# levels 1..5 of the 128-pair tournament: 0.5 + 0.5 + 3 (1/4 + 1/8 + 1/16 + 1/32 + 1/64)
ALU_PER_SCORE = 1.0 + 3.0 * (1 / 4 + 1 / 8 + 1 / 16 + 1 / 32 + 1 / 64)
ALU_LANES_PER_CLK_SM = 64


def smi(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return [f.strip() for f in out.split(",")] if out else []


def stderr_of(fn):
    """what the library printed to file descriptor 2 during fn()"""
    sys.stderr.flush()
    with tempfile.TemporaryFile() as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            fn()
            lb.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        return tmp.read().decode()


def profiled(fn, reps):
    """per family ending in tc_pq_filter / tc_pq_fallback: launches per call, per-launch us of each repetition"""
    fn()  # warm-up: module load, workspace growth
    fams = {}
    clocks = []
    for _ in range(reps):
        lb.profile.enable(True)
        lb.profile.reset()
        fn()
        lb.synchronize()
        clocks.append(float(smi("clocks.sm")[0]))
        lb.profile.enable(False)
        for name, (cnt, ms) in lb.profile.dump().items():
            for fam in ("tc_pq_filter", "tc_pq_fallback"):
                if name.endswith(fam) and cnt:
                    f = fams.setdefault(fam, {"launches": cnt, "us_per_launch": []})
                    f["us_per_launch"].append(ms * 1e3 / cnt)
    return fams, float(np.median(clocks))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("pq_filter_timing: no CUDA device (nothing is measured without one)")
    lb.set_device(0)
    name, plimit, max_sm = smi("name,power.limit,clocks.max.sm")
    import ctypes as C
    sms = C.c_int(0)
    rt = C.CDLL("libcudart.so.12")
    assert rt.cudaDeviceGetAttribute(C.byref(sms), 16, 0) == 0  # cudaDevAttrMultiProcessorCount
    x = synth.sift_like(a.n, D)
    sample = x[np.sort(np.random.default_rng(0).choice(a.n, min(a.n, SAMPLE), replace=False))]
    cent = lb.train_kmeans(sample, D, K, max_iters=10).centroids
    part, _, _ = lb.compute_partitions(cent, sample)
    res = lb.compute_residual(cent, sample, part)
    init = np.stack([res[np.random.default_rng(1).choice(len(res), KC, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    part_all, _, _ = lb.compute_partitions(cent, x)
    box = {}

    def train():
        box["pq"] = lb.PQBuildParams(M, 8, max_iters=ITERS, codebook=init).build(res)

    def encode():
        box["codes"] = box["pq"].quantize(x, cent, part_all)

    out = {"card": name, "power_limit_w": float(plimit), "sm_max_mhz": float(max_sm), "sms": sms.value,
           "alu_per_score": ALU_PER_SCORE, "reps": a.reps, "runs": {}}
    for label, fn, rows in (("pq_train_65536", train, len(res)), ("quantize", encode, a.n)):
        fams, mhz = profiled(fn, a.reps)
        os.environ["LB2_TC_STATS"] = "1"
        try:
            shares = [float(v) for v in re.findall(r"exact-fallback pairs ([\d.]+)%", stderr_of(fn))]
        finally:
            os.environ.pop("LB2_TC_STATS", None)
        run = {"rows": rows, "sm_mhz": mhz, "undecided_pct": float(np.mean(shares)) if shares else None}
        peak = sms.value * ALU_LANES_PER_CLK_SM * mhz * 1e6 / ALU_PER_SCORE
        for fam, f in fams.items():
            us = float(np.median(f["us_per_launch"]))
            run[fam] = {"launches": f["launches"], "us_per_launch": us,
                        "us_min": float(min(f["us_per_launch"])), "us_max": float(max(f["us_per_launch"]))}
            if fam == "tc_pq_filter":
                rate = rows * M * KC / (us * 1e-6)
                run[fam].update(scores_per_s=rate, alu_bound_scores_per_s=peak, share_of_alu_bound=rate / peak)
        out["runs"][label] = run
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
