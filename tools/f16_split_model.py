"""Numeric model (numpy + the oracle, no GPU) of the NEXT first-pass variant proposed in DESIGN.md section 8 (v):
integer-valued columns (SIFT, u8: exactly representable in f16) against f32 centroids split into two f16 terms,
c = ch + cl + r with |r| <= 2^-22 |c|, as ONE f16 GEMM over the operands A' = [x | x], B' = [ch | cl]: every
product is exact, what is lost is r, the f32 accumulation and the index byte.  Prints, for SIFT-shaped data, the share
of rows each certificate decides (unique + two-candidate) and checks that the certified rows are right.
usage: python tools/f16_split_model.py [rows] [K]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from lance_b200 import synth
from oracle import binding as ob
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from test_filter_certificate_model import TAU_TF32, certificate, tf32_trunc

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4000
K = int(sys.argv[2]) if len(sys.argv) > 2 else 256
d = 128
data = synth.sift_like(60000, d, seed=5)
cent = ob.kmeans_train(data[:40000], K, max_iters=8, nthreads=8)[0]
x = data[40000:40000 + n]
ref, _, _ = ob.compute_membership(cent, x, nthreads=8)
n2 = (cent * cent).sum(1, dtype=np.float32)
xn2 = (x * x).sum(1, dtype=np.float32)


def report(name, flag, idx):
    uniq, two = flag == 0, flag == 1
    ok = np.array_equal(idx[uniq, 0], ref[uniq]) and np.all((idx[two, 0] == ref[two]) | (idx[two, 1] == ref[two]))
    print(f"{name:34s} unique {uniq.mean():7.2%}  two-candidate {two.mean():6.2%}  undecided {(flag == 2).mean():6.2%}  certified rows correct: {ok}")


for acc in ("exact", "toward_zero"):
    flag, idx = certificate(tf32_trunc(x), tf32_trunc(cent), np.float32(-0.5) * n2, TAU_TF32 * (xn2 + n2.max()), acc)
    report(f"TF32 first pass ({acc})", flag, idx)
    assert np.array_equal(x.astype(np.float16).astype(np.float32), x)           # integer-valued: exact in f16
    ch = cent.astype(np.float16).astype(np.float32)
    cl = (cent - ch).astype(np.float16).astype(np.float32)
    a2, b2 = np.concatenate([x, x], 1), np.concatenate([ch, cl], 1)
    # budget: dropped remainder 2^-22 |x||c| <= 2^-23 (|x|^2+|c|^2); accumulation over 2d/16 MMA steps, two ulps each on
    # the running magnitude <= (2d/16) 2^-22 ...; index byte 2^-16 |score| <= 2^-16 (|x|^2 + |c|^2)/... -> covered twice by
    tau = np.float32(2.0 ** -13 + 2 * d * 2.0 ** -25) * (xn2 + n2.max())
    flag, idx = certificate(a2, b2, np.float32(-0.5) * n2, tau, acc)
    report(f"f16 split first pass ({acc})", flag, idx)
