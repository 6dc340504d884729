"""lb2_index_optimize on an IVF_HNSW_SQ index at SIFT shape (synth.sift_like: 1 M x 128 f32, K = 256, default build and
graph parameters), next to a full build of the merged rows.

    python tools/optimize_timing.py [--n 1000000] [--n-add 10000] [--reps 3] [--out FILE]

Four cases, each timed with CUDA events around the blocking call (median of --reps after one warm-up):
  (a) optimize appending n_add new rows, spread over all partitions by the index's own transform;
  (b) the same rows forced into 8 partitions (part id mod 8), so only 8 graphs are rebuilt;
  (c) a remap that only rewrites row ids (every id + 2^40): no graph is rebuilt;
  (d) lb2_ivfhnswsq_build of the merged n + n_add rows.
The rows of (a) and (b) are transformed once before the timing.  Prints one JSON line (the card's name and power
limit included) and writes it to FILE when given."""
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
    call().close()
    ts = []
    for _ in range(reps):
        lb.synchronize()
        lb.timer_start()
        out = call()
        ts.append(lb.timer_stop())
        out.close()
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--n-add", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("optimize_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    data = synth.sift_like(a.n + a.n_add, a.d)
    base, new = data[:a.n], data[a.n:]
    ix = lb.IvfHnswSqIndex.build(base, "l2", num_partitions=a.K)
    t = ix.transform(new)
    ok = t["valid"]
    part, payload = t["part_ids"][ok], t["payload"][ok]
    rid = np.arange(a.n, a.n + a.n_add, dtype=np.uint64)[ok]
    ids = np.sort(ix.export()["row_ids"])
    shift = ids + np.uint64(1 << 40)
    ms = dict(
        a_append_spread=timed(lambda: ix.optimize(add_part_ids=part, add_payload=payload, add_row_ids=rid, seed=1),
                              a.reps),
        b_append_8_partitions=timed(lambda: ix.optimize(add_part_ids=part % 8, add_payload=payload, add_row_ids=rid,
                                                        seed=1), a.reps),
        c_remap_ids_only=timed(lambda: ix.optimize(remap=(ids, shift), seed=1), a.reps),
        d_full_build=timed(lambda: lb.IvfHnswSqIndex.build(data, "l2", num_partitions=a.K), a.reps),
    )
    out = dict(tool="optimize_timing", card=card,
               shape=dict(n=a.n, d=a.d, K=a.K, n_add=int(ok.sum()), data="synth.sift_like", kind="IVF_HNSW_SQ",
                          hnsw="max_level 7, m 20, ef_construction 150"),
               reps=a.reps, ms=ms)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
