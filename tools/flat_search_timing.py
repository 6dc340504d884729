"""Flat KNN timing (lb2_flat_search): a SIFT-shaped 1 M x 128 column from lance_b200.synth as f32, f16 and u8, resident
on the device and in pinned host memory, at k = 10 / 100 and nq = 1 / 64 / 1 000 / 10 000.

    python tools/flat_search_timing.py [--n 1000000] [--reps 3] [--out FILE]

Per point: ms per call (CUDA events around `reps` calls after a warm-up call), the scan kernel's time from the launch
profiler (a separate pass), and that kernel's share of the larger of two lower bounds:
  * HBM: ceil(nq / 16) * n * d * sizeof(T) bytes (each 16-query tile reads the column once) at 3.35 TB/s;
  * FP32 issue: 3 (L2) or 2 (dot) instructions per (query, row) pair and element at 33.5 T instructions/s (the
    67 TFLOP/s data-sheet figure with an FMA counted as two; the rule has no FMA).
For scale at nq = 1 000 and 10 000, bench.py's torch f32 brute force (`ground_truth`, TF32 off, k = 10, 1 000 queries
per call) on the device column.
The card's name and power limit are read in the same run.  One JSON line goes to stdout and to FILE."""
import argparse
import json
import math
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)

HBM_BYTES_PER_S = 3.35e12
FP32_INSTR_PER_S = 33.5e12
QUERY_TILE = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--metric", default="l2", choices=["l2", "dot"])
    ap.add_argument("--out", default="flat_search_timing.json")
    args = ap.parse_args()
    import numpy as np

    import lance_b200 as lb
    from lance_b200 import synth

    if lb.device_count() < 1:
        raise SystemExit("flat_search_timing: no CUDA device (lance_b200 has no CPU fallback)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    n, d = args.n, 128
    x = synth.sift_like(n, d, n_components=256, seed=11)
    qall = synth.sift_like_queries(10_000, d, n_components=256, seed=11)
    cols = {"f32": (x, qall), "f16": (x.astype(np.float16), qall.astype(np.float16)),
            "u8": (np.clip(np.rint(x), 0, 255).astype(np.uint8), np.clip(np.rint(qall), 0, 255).astype(np.uint8))}
    ops = 3 if args.metric == "l2" else 2
    points = []
    for dt, (col, qs) in cols.items():
        dev = lb.DeviceArray.from_numpy(col)
        pin = lb.PinnedArray(col.shape, col.dtype)
        pin.array[...] = col
        for where, c in (("device", dev), ("pinned", pin)):
            for k in (10, 100):
                for nq in (1, 64, 1000, 10_000):
                    q = lb.DeviceArray.from_numpy(qs[:nq])
                    call = lambda: lb.flat_search(c, q, k, args.metric)  # noqa: E731
                    call()
                    lb.timer_start()
                    for _ in range(args.reps):
                        call()
                    ms = lb.timer_stop() / args.reps
                    lb.profile.reset()
                    lb.profile.enable(True)
                    call()
                    lb.profile.enable(False)
                    prof = lb.profile.dump()
                    scan_ms = prof.get("flat_search:scan", (0, 0.0))[1]
                    merge_ms = prof.get("flat_search:merge", (0, 0.0))[1]
                    hbm_ms = math.ceil(nq / QUERY_TILE) * n * d * col.itemsize / HBM_BYTES_PER_S * 1e3
                    fp_ms = nq * n * d * ops / FP32_INSTR_PER_S * 1e3
                    bound = max(hbm_ms, fp_ms)
                    points.append({"dtype": dt, "input": where, "k": k, "nq": nq, "ms_per_call": ms,
                                   "scan_kernel_ms": scan_ms, "merge_kernel_ms": merge_ms,
                                   "bound_ms": bound, "bound": "hbm" if hbm_ms >= fp_ms else "fp32_issue",
                                   "scan_share_of_bound": bound / scan_ms if scan_ms > 0 else None})
                    print(json.dumps(points[-1]), file=sys.stderr, flush=True)
                    q.free()
        dev.free()
        pin.free()
    # for scale: bench.py's torch brute force on the device column (f32, TF32 off)
    torch_ms = {}
    try:
        import torch

        sys.path.insert(0, HERE)
        from bench import ground_truth
        data = torch.from_numpy(x).cuda()
        for nq in (1000, 10_000):
            qt = torch.from_numpy(qall[:nq]).cuda()
            ground_truth(torch, data, qt[:1000], 10)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                for q0 in range(0, nq, 1000):  # 1 000 queries per call: its [nq][rows] distance block fits the card
                    ground_truth(torch, data, qt[q0:q0 + 1000], 10, return_dists=True)
            e1.record()
            torch.cuda.synchronize()
            torch_ms[str(nq)] = e0.elapsed_time(e1) / args.reps
    except Exception as e:  # noqa: BLE001 -- the comparison is for scale only
        torch_ms["error"] = repr(e)
    line = {"tool": "flat_search_timing", "gpu": gpu, "n": n, "d": d, "metric": args.metric, "reps": args.reps,
            "query_tile": QUERY_TILE, "points": points, "torch_ground_truth_k10_ms": torch_ms}
    print(json.dumps(line), flush=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
