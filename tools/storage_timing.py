"""The storage-layout conversions of lb2_index_export_storage / lb2_index_load_storage at 1 M rows.

    python tools/storage_timing.py [--n 1000000] [--reps 3] [--out FILE]

Builds a 1 M x 128 IVF_HNSW_SQ index (m 20, insert_batch 256) and a 1 M x 128 IVF_RQ index (synth.sift_like, K = 256)
and times, for each, export_storage and from_storage:
  - call_ms: the whole call (host clock around a blocking call, host <-> device copies of the numpy columns included);
  - kernel_ms: the device time of the conversion kernels alone (the launch profiler's CUDA events per kernel family,
    in a separate profiled run): RaBitQ packing / unpacking, the device scans and the graph level-batch kernels.  The
    other kernels of the call (the load's grouping of the rows by partition, the partition-id and length kernels) are
    listed under other_kernels with their time; plain copies (payload, _rowid, factors) and lb2_index_load_hnsw_*'s
    neighbour checks on the host are in call_ms only;
  - converted_bytes: the least memory traffic of the conversion kernels -- each converted storage column read or
    written once (IVF_RQ: __rabit_code; IVF_HNSW_SQ: entry_point, level_offsets, __vector_id, list_offsets,
    __neighbors, _distance) plus its device-layout side read or written once (IVF_RQ: the same bytes of row-major
    codes; IVF_HNSW_SQ: 8 bytes per list entry, 4 per list count, 1 per row's level) -- and its rate over kernel_ms;
  - storage_bytes: the bytes of all storage columns (no rate: most of them are plain copies).
The card's name and power limit are read in the same run.  Results go to FILE as JSON (default storage_timing.json)."""
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

# kernel families of the conversions (LB2_LAUNCH names)
FAMILIES = ("rq_pack", "rq_unpack", "transpose_codes", "storage_scan", "hnsw_to_storage", "hnsw_from_storage")
GRAPH_COLUMNS = ("entry_point", "level_offsets", "__vector_id", "list_offsets", "__neighbors", "_distance")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def kernel_ms(call):
    lb.profile.reset()
    lb.profile.enable(True)
    call()
    lb.profile.enable(False)
    total = 0.0
    per, other = {}, {}
    for name, (_, ms) in lb.profile.dump().items():
        if name.split(":")[-1] in FAMILIES:
            per[name] = ms
            total += ms
        else:
            other[name] = ms
    return total, per, other


def converted_bytes(st):
    """the least traffic of the conversion kernels (see the module docstring)"""
    if "__rabit_code" in st:
        return 2 * st["__rabit_code"].nbytes
    storage = sum(st[k].nbytes for k in GRAPH_COLUMNS)
    rows, edges = st["__vector_id"].size, st["__neighbors"].size
    return storage + 8 * edges + 4 * rows + st["_rowid"].size


def wall_ms(call, reps):
    call()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        call()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def measure(name, ix, reopen, reps):
    st = ix.export_storage()
    nbytes = int(sum(np.asarray(v).nbytes for v in st.values() if isinstance(v, np.ndarray)))
    cb = int(converted_bytes(st))
    out = {"storage_bytes": nbytes, "converted_bytes": cb}
    for what, call in (("export", ix.export_storage), ("load", lambda: reopen(st))):
        ms = wall_ms(call, reps)
        kms, per, other = kernel_ms(call)
        out[what] = {"call_ms": ms, "kernel_ms": kms, "kernels": per, "other_kernels": other,
                     "converted_GB_per_s": cb / (kms * 1e6) if kms else None}
    print(name, json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="storage_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("storage_timing: no CUDA device")
    res = {"card": card(), "n": a.n, "d": 128, "num_partitions": 256}
    data = synth.sift_like(a.n, 128, seed=11)
    ix = lb.IvfHnswSqIndex.build(data, "l2", num_partitions=256, max_iters=10,
                                 hnsw_params=lb.HnswBuildParams(m=20, insert_batch=256))
    e = ix.export()
    res["ivf_hnsw_sq"] = measure("IVF_HNSW_SQ", ix, lambda st: lb.IvfHnswSqIndex.from_storage(
        e["centroids"], e["bounds"], st), a.reps)
    del ix
    rq = lb.IvfRqIndex.build(data, "l2", num_partitions=256, max_iters=10)
    e = rq.export()
    res["ivf_rq"] = measure("IVF_RQ", rq, lambda st: lb.IvfRqIndex.from_storage(e["centroids"], e["rotation"], st),
                            a.reps)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"]}))


if __name__ == "__main__":
    main()
