"""Restatement of how ANNIvfSubIndexExec decides how many partitions a query searches
(rust/lance/src/io/exec/knn.rs:714-882 initial / late search, 1108-1130 adjust_probes / early_pruning), with the
late-search width pinned as the project pins it (DESIGN.md section 2): late partition t is searched while found0 plus
the rows of the late partitions u <= t - late_width stays below the target."""
import numpy as np


def partition_point(values, pred):
    """Rust 1.90 slice::partition_point = binary_search_by(|x| if pred(x) Less else Greater): a fixed number of
    halving steps, then one last probe.  On a predicate that is not monotone (NaN) it returns what that search does."""
    size = len(values)
    if size == 0:
        return 0
    base = 0
    while size > 1:
        half = size // 2
        mid = base + half
        if pred(values[mid]):
            base = mid
        size -= half
    return base + (1 if pred(values[base]) else 0)


def early_pruning(dists, k):
    if len(dists) == 0:
        return 0
    f = np.float32(0.6) if k <= 1 else (np.float32(7.0) if k <= 10 else np.float32(81.0))
    thr = np.float32(np.float32(dists[0]) * f)
    return partition_point(dists, lambda d: np.float32(d) <= thr)


def adjust_probes(minimum, maximum, pruned):
    """(minimum_nprobes, maximum_nprobes) after adjust_probes; maximum None = unbounded"""
    minimum = max(minimum, pruned)
    if maximum is not None and minimum > maximum:
        minimum = maximum
    return minimum, maximum


def probe_count(dists, c, k, minimum=1, maximum=None, late_width=1, max_len=None, iterable=False):
    """dists: the L = min(maximum or K, K) ranked centroid distances; c[t]: rows partition P[t] returns
    (min(kc, rows the mask and range admit)).  Returns (partitions searched, shortcut taken, found0)."""
    L = len(dists)
    mn, _ = adjust_probes(minimum, maximum, early_pruning(dists, k))
    mn = min(mn, L)
    found0 = min(k, int(sum(int(x) for x in c[:mn])))
    if L <= mn or found0 >= k:
        return mn, False, found0
    if max_len is not None and iterable and found0 < max_len <= k:
        return mn, True, found0
    target = min(k, max_len) if max_len is not None else k
    n, acc = mn, found0
    for t in range(L - mn):
        if t >= late_width:
            acc += int(c[mn + t - late_width])
        if acc >= target:
            break
        n += 1
    return n, False, found0
