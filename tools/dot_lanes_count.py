"""Counts, on the CPU, how often the lane count of an f16 dot product changes a k-means assignment on C3-shaped
data (f16 rows N(centre, 1) of a Gaussian mixture, d = 128): the reference assigns f16 rows under DOT with
dot_distance_batch on f16 (kmeans.rs:349-353), i.e. dot_scalar::<f16, f32, 32> (dot.rs:30-58,133), while the device's
assignment sums every element type in 16 f32 lanes.  Prints the share of (row, centroid) distances that differ and
the share of rows whose argmin (first minimum) changes.  The two sums are restated in numpy and checked against the
oracle's lo_dot_f16 (32 lanes) and lo_dot_f32 on the converted values (16 lanes) on a sample.
usage: python tools/dot_lanes_count.py [rows] [K]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle import binding as ob


def lane_dot(x, c, lanes):
    """[rows] x [K] dot products of f32 operands with `lanes` accumulators (d a multiple of lanes, no tail)"""
    d = x.shape[1]
    acc = np.zeros((x.shape[0], c.shape[0], lanes), np.float32)
    for s in range(0, d, lanes):
        acc += x[:, None, s:s + lanes] * c[None, :, s:s + lanes]     # f32 products, one rounded add per lane
    t = np.zeros(acc.shape[:2], np.float32)
    for l in range(lanes):
        t += acc[:, :, l]
    return t


def main(n=8192, K=1024, d=128, seed=3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((256, d)).astype(np.float32) * 3.0
    x = (centres[rng.integers(0, 256, n)] + rng.standard_normal((n, d))).astype(np.float16)
    c = x[rng.choice(n, K, replace=False)]                          # f16 model, initialised from rows
    x32, c32 = x.astype(np.float32), c.astype(np.float32)
    for i in range(8):                                              # the restatements are the oracle's sums
        assert lane_dot(x32[i:i + 1], c32[i:i + 1], 32)[0, 0] == np.float32(ob.dot_f16(x[i], c[i]))
        assert lane_dot(x32[i:i + 1], c32[i:i + 1], 16)[0, 0] == np.float32(ob.dot(x32[i], c32[i]))
    one = np.float32(1.0)
    dist_diff = arg_diff = 0
    for b in range(0, n, 128):
        d16 = one - lane_dot(x32[b:b + 128], c32, 16)
        d32 = one - lane_dot(x32[b:b + 128], c32, 32)
        dist_diff += int(np.sum(d16 != d32))
        arg_diff += int(np.sum(np.argmin(d16, 1) != np.argmin(d32, 1)))
    print(f"n={n} K={K} d={d}: distances that differ {dist_diff} of {n * K} ({100.0 * dist_diff / (n * K):.2f} %), "
          f"argmins that differ {arg_diff} of {n} ({100.0 * arg_diff / n:.3f} %)")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
