"""Exact-distance search timing, two builds of the package side by side: the IVF_FLAT scan (1 M x 128 f32; C4-shaped
200 000 x 1536 bf16), lb2_flat_topk over 1 M distances, and bench.py's C1 `query` / `query_refine`.

    python tools/exact_search_timing.py --base DIR [--reps 5] [--bench-steps 5] [--out FILE]

DIR is another built tree of this repository (e.g. the parent commit).  Each tree is imported in its own worker
process; the cases alternate between the two workers, so both see the same machine state, and every case's outputs
(ids, distances, counts) are byte-compared.  Times are CUDA-event milliseconds per call and the summed kernel time of
the case's kernel family from the launch profiler; the card's name and power limit are recorded with them.  The
results go to FILE as JSON (default: exact_search_timing.json in the current directory)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (kind, k, family of the timed kernel)
CASES = {
    "flat_f32_k10": ("flat_f32", 10, "flat_scan"),
    "flat_f32_k100": ("flat_f32", 100, "flat_scan"),
    "flat_bf16_k10": ("flat_bf16", 10, "flat_scan"),
    "topk_k10": ("topk", 10, "flat_topk"),
    "topk_k100": ("topk", 100, "flat_topk"),
    "topk_k1024": ("topk", 1024, "flat_topk"),
}


def worker(tree):
    sys.path.insert(0, tree)
    import numpy as np
    import lance_b200 as lb

    def flat_index(n, d, K, bf16, seed):
        rng = np.random.default_rng(seed)
        cent = (rng.standard_normal((K, d)) * 4).astype(np.float32)
        part = np.sort(rng.integers(0, K, n)).astype(np.uint32)
        x = cent[part] + rng.standard_normal((n, d), dtype=np.float32)
        if bf16:
            x = (x.view(np.uint32) >> 16).astype(np.uint16)
            cent = (cent.view(np.uint32) >> 16).astype(np.uint16)
        ix = lb.IvfFlatIndex.from_parts(cent, part, x, np.arange(n, dtype=np.uint64), "l2", bf16=bf16)
        return ix, rng

    data = {}
    ix, rng = flat_index(1_000_000, 128, 256, False, 1)
    data["flat_f32"] = (ix, rng.standard_normal((10_000, 128), dtype=np.float32) * 4, 10)
    ix, rng = flat_index(200_000, 1536, 256, True, 2)
    q = rng.standard_normal((1_000, 1536), dtype=np.float32) * 4
    data["flat_bf16"] = (ix, (q.view(np.uint32) >> 16).astype(np.uint16), 4)
    rng = np.random.default_rng(3)
    dists = rng.standard_normal(1_000_000, dtype=np.float32) ** 2
    rid = rng.permutation(1_000_000).astype(np.uint64)

    def run(name):
        kind, k, fam = CASES[name]
        if kind == "topk":
            call = lambda: lb.flat_topk(dists, rid, k)  # noqa: E731
        else:
            ix, q, nprobes = data[kind]
            call = lambda: ix.search(q, k=k, nprobes=nprobes)  # noqa: E731
        for _ in range(2):
            out = call()
        reps = 10
        lb.profile.reset()
        lb.profile.enable(True)
        lb.timer_start()
        for _ in range(reps):
            out = call()
        ms = lb.timer_stop() / reps
        lb.profile.enable(False)
        kms = sum(v[1] for f, v in lb.profile.dump().items() if fam in f) / reps
        blob = b"".join(np.ascontiguousarray(a).tobytes() for a in out)
        return {"ms": ms, "kernel_ms": kms, "out": blob.hex()}

    for line in sys.stdin:
        print(json.dumps(run(line.strip())), flush=True)


def bench(tree, steps, dump):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", "1", "--no-cpu-baseline",
           "--dump-outputs", dump]
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, check=True).stdout
    line = json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])
    files = {f: open(os.path.join(dump, f), "rb").read() for f in sorted(os.listdir(dump))}
    return {"query_qps": line["query"]["qps"], "query_refine_qps": line["query_refine"]["qps"]}, files


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="the other built tree")
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--out", default="exact_search_timing.json", help="where the JSON results go")
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)
    trees = {"base": os.path.abspath(args.base), "this": HERE}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    procs = {t: subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", p], stdin=subprocess.PIPE,
                                 stdout=subprocess.PIPE, text=True) for t, p in trees.items()}
    res = {"gpu": gpu, "cases": {}}
    for name in CASES:
        runs = {t: [] for t in trees}
        same = True
        for _ in range(args.reps):
            for t in trees:  # alternate base / this
                procs[t].stdin.write(name + "\n")
                procs[t].stdin.flush()
                runs[t].append(json.loads(procs[t].stdout.readline()))
            same &= runs["base"][-1]["out"] == runs["this"][-1]["out"]
        res["cases"][name] = {"identical": same, **{t: {"ms": [r["ms"] for r in v], "kernel_ms": [r["kernel_ms"] for r in v]}
                                                    for t, v in runs.items()}}
        print(name, json.dumps({t: (min(res["cases"][name][t]["ms"]), max(res["cases"][name][t]["ms"]))
                                for t in trees}), "identical" if same else "DIFFERENT", flush=True)
    for p in procs.values():
        p.stdin.close()
        p.wait()
    res["bench"] = {t: [] for t in trees}
    dumps = {}
    for _ in range(2):
        for t, p in trees.items():
            with tempfile.TemporaryDirectory() as dump:
                r, files = bench(p, args.bench_steps, dump)
            res["bench"][t].append(r)
            dumps.setdefault(t, files)
    res["bench_dumps_identical"] = dumps["base"] == dumps["this"]
    print(json.dumps(res["bench"]), "dumps identical:", res["bench_dumps_identical"], flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
