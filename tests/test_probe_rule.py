"""The restated probe rule of a search with minimum / maximum nprobes (tests/probe_rule.py), on the reference's own
test_adjust_probes_rules (knn.rs:1373-1404) and on hand-worked cases."""
import numpy as np

from probe_rule import adjust_probes, early_pruning, partition_point, probe_count

F = np.float32


def test_adjust_probes_rules():
    # transcribed from test_adjust_probes_rules (base_query: minimum 1, maximum None)
    assert adjust_probes(1, None, 10) == (10, None)
    assert adjust_probes(20, None, 10) == (20, None)
    assert adjust_probes(1, 25, 10) == (10, 25)
    assert adjust_probes(1, 5, 10) == (5, 5)
    assert adjust_probes(30, 50, 10) == (30, 50)


def test_early_pruning_factors_and_ties_at_threshold():
    d = np.array([1.0, 3.0, 6.999, 7.0, 7.0, 7.001, 80.0, 81.0, 81.0, 82.0], F)
    assert early_pruning(d, 2) == 5 and early_pruning(d, 10) == 5   # exactly at d0 * 7 counts
    assert early_pruning(d, 11) == 9                                # exactly at d0 * 81 counts
    assert early_pruning(d, 1) == 0                                 # 0.6: not even d0 itself
    assert early_pruning(np.array([], F), 5) == 0
    # the threshold is the f32 product d0 * 7: a distance equal to it is in, the next float is out
    d0 = F(0.3)
    thr = F(d0 * F(7.0))
    assert early_pruning(np.array([d0, thr, thr], F), 5) == 3
    assert early_pruning(np.array([d0, thr, np.nextafter(thr, F(9))], F), 5) == 2


def test_early_pruning_negative_d0_under_dot():
    d = np.array([-4.0, -3.0, -1.0, 0.5], F)
    # threshold -28 (k = 2) is below every distance, d0 included
    assert early_pruning(d, 2) == 0
    d = np.array([-0.0, 0.0, 0.0], F)
    assert early_pruning(d, 2) == 3        # -0.0 * 7 = -0.0 and 0.0 <= -0.0


def test_early_pruning_nan_is_the_binary_search_literally():
    nan = F(np.nan)
    d = np.array([1.0, nan, 2.0, 3.0, 9.0], F)      # threshold 7 (k = 2)
    # size 5: mid 2 (2.0 <= 7) -> base 2; size 3: mid 3 (3.0) -> base 3; size 2: mid 4 (9.0 > 7); last probe at 3
    assert early_pruning(d, 2) == 4
    d = np.array([1.0, 2.0, nan, nan, 3.0], F)
    # mid 2 is NaN (false) -> base 0; size 3: mid 1 (2.0) -> base 1; size 2: mid 2 NaN; last probe 2.0 -> 2
    assert early_pruning(d, 2) == 2
    d = np.array([nan, 1.0, 2.0], F)                  # d0 NaN: the threshold is NaN, nothing passes
    assert early_pruning(d, 5) == 0
    assert partition_point([1, 2, 3, 4], lambda v: v <= 2) == 2


def test_probe_count_initial_and_stop():
    d = np.array([1.0, 100.0, 200.0, 300.0, 400.0], F)
    c = [3, 3, 3, 3, 3]
    # k = 2: pruned = 1 (7 < 100); found0 = 2 >= k -> stop
    assert probe_count(d, c, 2, minimum=1) == (1, False, 2)
    # k = 10: pruned 1; found0 = 3 < 10; late search width 1: t=0 acc 3 -> search, t=1 acc 6, t=2 acc 9, t=3 acc 12 stop
    assert probe_count(d, c, 10, minimum=1) == (4, False, 3)
    # width 3: partition t is searched while found0 + c of late partitions u <= t - 3 stays below 10
    assert probe_count(d, c, 10, minimum=1, late_width=3) == (5, False, 3)
    # width larger than L: every late partition starts before any finishes
    assert probe_count(d, c, 10, minimum=1, late_width=64) == (5, False, 3)
    # maximum caps L: the list given is already P[0, L)
    assert probe_count(d[:2], c[:2], 10, minimum=1, maximum=2) == (2, False, 3)
    # minimum == maximum: no late search
    assert probe_count(d[:3], c[:3], 50, minimum=3, maximum=3) == (3, False, 9)


def test_probe_count_k_boundaries():
    d = np.array([1.0, 6.0, 7.0, 8.0, 80.0, 81.0, 82.0], F)
    c = [100] * 7
    assert probe_count(d, c, 1)[0] == 1            # pruned 0 -> min 1
    assert probe_count(d, c, 2)[0] == 3            # <= 7
    assert probe_count(d, c, 10)[0] == 3
    assert probe_count(d, c, 11)[0] == 6           # <= 81


def test_probe_count_filters_and_shortcut():
    d = np.array([1.0, 100.0, 200.0, 300.0], F)
    # an empty allow list: max_len 0 -> target 0, nothing late
    assert probe_count(d, [0, 0, 0, 0], 10, max_len=0, iterable=True) == (1, False, 0)
    # found0 < max_len <= k with iterable ids: shortcut
    assert probe_count(d, [2, 1, 0, 0], 10, max_len=3, iterable=True) == (1, True, 2)
    # not iterable: late search up to target = max_len
    assert probe_count(d, [2, 1, 0, 0], 10, max_len=3, iterable=False) == (2, False, 2)
    # max_len > k: no shortcut, target k
    assert probe_count(d, [2, 1, 0, 8], 5, max_len=30, iterable=True) == (4, False, 2)
    # target < k and found0 >= max_len: no late partition
    assert probe_count(d, [3, 1, 0, 0], 10, max_len=3, iterable=True) == (1, False, 3)
    assert probe_count(d, [3, 1, 0, 0], 10, max_len=3, iterable=False) == (1, False, 3)
    # block list only: no max_len -> the late search runs to k
    assert probe_count(d, [2, 1, 0, 0], 10) == (4, False, 2)
