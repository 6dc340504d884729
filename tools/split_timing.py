"""The partition split of an optimize on the device next to the same decisions on the host CPU.

    python tools/split_timing.py [--n 1000000] [--append 40000] [--reps 5] [--out FILE]

SIFT-shaped rows (synth.sift_like, 1 M x 128 f32) in an IVF_PQ(256, 16) index; --append rows near the centroid of its
largest partition are transformed with the index's model, so that partition passes 4 x 8192 rows and
partition_to_split picks it.  The host fetches the raw rows of that partition and of its 64 reassign candidates (stored
and appended), and the tool times reassign_candidates + split (host clock around the blocking calls, median of --reps
after a warm-up), then, in a separate profiled run, the `split_decide` kernel alone.  The decisions are restated on
the host with numpy -- the reference's 16-lane f32 L2 order, vectorised over rows -- timed, and compared with the
device's destinations.  The card's name and power limit are read in the same run.  Results go to FILE as JSON
(default split_timing.json)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import lance_b200 as lb  # noqa: E402
import split_join_reference as sj  # noqa: E402
from lance_b200 import synth  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def l2_rows(c, x):
    """l2_distance_batch(c, x) in the reference's order: 16 f32 lanes, no FMA, folded 0..15 (d a multiple of 16)"""
    n, d = x.shape
    acc = np.zeros((n, 16), np.float32)
    for k in range(0, d, 16):
        t = x[:, k:k + 16] - c[k:k + 16]
        acc += t * t
    s = np.zeros(n, np.float32)
    for lane in range(16):
        s += acc[:, lane]
    return s


def host_decisions(cent, part, c1, c2, v, cands, cv, cp):
    """assign_vectors / reassign_vectors over whole partitions (split_join_reference's rules, vectorised)"""
    k = len(cent)
    d0, d1, d2 = (l2_rows(c, v) for c in (cent[part], c1, c2))
    near = np.where(d1 <= d2, part, k).astype(np.uint32)
    dest = near.copy()
    re = np.flatnonzero((d0 <= d1) & (d0 <= d2))
    if re.size:
        cd = np.stack([l2_rows(cent[c], v[re]) for c in cands], 1)   # batch(row, c) == batch(c, row) under L2
        j = np.argmin(cd, 1)                                          # the first minimum (no NaN here)
        m = cd[np.arange(re.size), j]
        go = (m <= d1[re]) & (m <= d2[re])
        dest[re] = np.where(go, np.asarray(cands, np.uint32)[j], near[re])
    out = [dest]
    for q in cands:
        sel = cp == q
        x = cv[sel]
        e0, e1, e2 = (l2_rows(c, x) for c in (cent[q], c1, c2))
        out.append(np.where((e0 <= e1) & (e0 <= e2), sj.STAYS, np.where(e1 <= e2, part, k)).astype(np.uint32))
    return np.concatenate(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--append", type=int, default=40_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="split_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("split_timing: no CUDA device (there is no CPU fallback)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    d, K, M = 128, 256, 16
    x = synth.sift_like(a.n, d)
    ix = lb.IvfPqIndex.build(lb.DeviceArray.from_numpy(x), "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M,
                                                                                   seed=0))
    e = ix.export()
    offs = e["part_offsets"].astype(np.int64)
    big = int(np.argmax(np.diff(offs)))
    rng = np.random.default_rng(1)
    xa = (e["centroids"][big] + rng.normal(0, 2.0, (a.append, d))).astype(np.float32)
    ida = np.arange(a.n, a.n + a.append, dtype=np.uint64)
    t = ix.transform(xa)
    assert t["valid"].all()
    part = ix.partition_to_split(t["part_ids"])
    assert part is not None, "no partition passes 4 x 8192 rows"
    col = np.concatenate([x, xa])

    def rows_of(p):
        ids = np.sort(np.concatenate([e["row_ids"][offs[p]:offs[p + 1]], ida[t["part_ids"] == p]]))
        return col[ids.astype(np.int64)], ids
    cands = ix.reassign_candidates(part)
    v, r = rows_of(part)
    parts = [rows_of(int(q)) for q in cands]
    cv = np.concatenate([p[0] for p in parts])
    cr = np.concatenate([p[1] for p in parts])
    cp = np.concatenate([np.full(len(p[1]), q, np.uint32) for p, q in zip(parts, cands)])
    vd, cvd = lb.DeviceArray.from_numpy(v), lb.DeviceArray.from_numpy(cv)
    opt = dict(add_part_ids=t["part_ids"], add_payload=t["payload"], add_row_ids=ida, seed=0)

    def device():
        c = ix.reassign_candidates(part)
        return c, ix.split(part, vd, r, cvd, cr, cp, **opt)
    device()
    ts, got = [], None
    for _ in range(a.reps):
        t0 = time.perf_counter()
        c, got = device()
        ts.append((time.perf_counter() - t0) * 1e3)
    assert np.array_equal(c, cands)
    dest = got[1]["dest"]
    newc = got[1]["new_centroids"]
    lb.profile.reset()
    lb.profile.enable(True)
    device()
    prof = lb.profile.dump()
    lb.profile.enable(False)
    th = []
    for _ in range(max(1, a.reps // 2)):
        t0 = time.perf_counter()
        want = host_decisions(e["centroids"], part, newc[part], newc[K], v, cands, cv, cp)
        th.append((time.perf_counter() - t0) * 1e3)
    same = bool(np.array_equal(dest, want))
    n_rows = len(r) + len(cr)
    dec_ms = prof.get("split_decide", (0, 0.0))[1]
    rows_bytes = n_rows * d * 4
    res = {
        "card": gpu[0] if gpu else "unknown", "n": a.n, "d": d, "K": K, "M": M, "appended": a.append,
        "split_partition": part, "split_rows": len(r), "candidates": len(cands), "candidate_rows": len(cr),
        "moved_rows": int((dest != sj.STAYS).sum()),
        "device_ms_median": float(np.median(ts)), "device_ms_all": ts,
        "host_decisions_ms_median": float(np.median(th)), "host_threads": "numpy, one process",
        "destinations_equal": same,
        "kernels_ms": {k: v[1] for k, v in sorted(prof.items())},
        "split_decide": {"ms": dec_ms, "row_bytes": rows_bytes,
                         "row_bytes_per_s": rows_bytes / (dec_ms * 1e-3) if dec_ms else None,
                         "share_of_hbm_peak": rows_bytes / HBM_BPS / (dec_ms * 1e-3) if dec_ms else None},
    }
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("card", "device_ms_median", "host_decisions_ms_median",
                                          "destinations_equal", "split_rows", "candidate_rows", "moved_rows")}))
    if not same:
        raise SystemExit("split_timing: device and host destinations differ")


if __name__ == "__main__":
    main()
