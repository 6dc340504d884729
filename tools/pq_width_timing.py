"""IVF_PQ builds at four PQ sub-vector widths: 1 M x 768 f32 rows (synth.gaussian_mixture), K = 256, 8-bit codes,
num_sub_vectors M = 96 (ds 8: the tensor-core filter, for comparison), 48 (ds 16), 16 (ds 48) and 8 (ds 96).

    python tools/pq_width_timing.py [--n 1000000] [--d 768] [--subvectors 96,48,16,8] [--out FILE]

For each M one build is timed (the build's own CUDA-event stage times: ms_pq_train, ms_transform, ms_total) and a
second, separate build runs with the launch profiler on; from it come the `pq_assign_wide` launches and their time in
PQ training and in the transform.  The transform encodes every row once, which costs 3 separately rounded FP32
instructions (sub, mul, add) per (row, codeword, dimension): 3 * n * 2^nbits * d.  At the data sheet's 67 TFLOP/s
(an FMA counted as two: 33.5 T FP32 instructions/s, a 700 W card) that is the FP32 issue bound; the share reported is
that bound over the measured transform-phase `pq_assign_wide` time.  The bound is computed, not measured.  The card's
name, power limit and maximum SM clock are read in the same call.  Results go to FILE as JSON (default
pq_width_timing.json)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lance_b200 as lb  # noqa: E402
from lance_b200 import synth  # noqa: E402

FP32_INSTR_PER_S = 67e12 / 2   # H100 SXM data sheet, dense FP32, FMA = 2 flops


def kernel_ms(prof, name):
    """(launches, ms) of kernel family `name` per phase tag"""
    out = {}
    for key, (cnt, ms) in prof.items():
        parts = key.split(":")
        if parts[-1] == name:
            tag = parts[0] if len(parts) > 1 else ""
            c, t = out.get(tag, (0, 0.0))
            out[tag] = (c + cnt, t + ms)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--subvectors", default="96,48,16,8")
    ap.add_argument("--out", default="pq_width_timing.json")
    a = ap.parse_args()
    if lb.device_count() < 1:
        raise SystemExit("pq_width_timing: no CUDA device (there is no CPU fallback to time)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    data = lb.DeviceArray.from_numpy(synth.gaussian_mixture(a.n, a.d, n_components=1024, seed=1))
    nbits = 8
    bound_ms = 3.0 * a.n * (1 << nbits) * a.d / FP32_INSTR_PER_S * 1e3
    out = dict(card=card, shape=dict(n=a.n, d=a.d, K=a.K, nbits=nbits, data="synth.gaussian_mixture, device-resident"),
               encode_fp32_bound_ms=bound_ms, runs=[])
    params = lambda M: lb.IvfBuildParams(num_partitions=a.K, num_sub_vectors=M)  # noqa: E731
    lb.IvfPqIndex.build(data, "l2", params(int(a.subvectors.split(",")[0]))).close()  # warm-up: module loads
    for M in (int(m) for m in a.subvectors.split(",")):
        ix = lb.IvfPqIndex.build(data, "l2", params(M))
        st = ix.stats
        ix.close()
        lb.profile.enable(True)
        lb.profile.reset()
        try:
            lb.IvfPqIndex.build(data, "l2", params(M)).close()
        finally:
            lb.profile.enable(False)
        prof = lb.profile.dump()
        wide = kernel_ms(prof, "pq_assign_wide")
        tc = kernel_ms(prof, "tc_pq_filter")
        row = dict(num_sub_vectors=M, ds=a.d // M, ms_pq_train=st.ms_pq_train, ms_transform=st.ms_transform,
                   ms_total=st.ms_total, pq_iters_max=st.pq_iters_max,
                   pq_assign_wide={tag: dict(launches=c, ms=t) for tag, (c, t) in wide.items()},
                   tc_pq_filter={tag: dict(launches=c, ms=t) for tag, (c, t) in tc.items()})
        if "transform" in wide:
            row["encode_share_of_fp32_bound"] = bound_ms / wide["transform"][1]
        out["runs"].append(row)
        print(json.dumps(row), flush=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
