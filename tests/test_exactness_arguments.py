"""Arguments the device code relies on, checked on the CPU (no GPU, no product code; section 3 is at the end).

1. Order-independent sums (DESIGN.md section 3; lloyd.cu `update_body_warp` / `stats_body` fast paths): the reference
   adds a cluster's members sequentially (f32 centroid sums kmeans.rs:388-418, f64 loss :266-280).  If every term is an
   integer multiple of 2^g and sum|term| < 2^(g+p) (p = 24 for f32, 53 for f64) no addition of ANY association rounds,
   so a parallel tree reduction returns the sequential result bit for bit.  Outside the condition it does not.

2. Convergence through progress words (DESIGN.md section 3; lloyd.cu `PollWords`, `epilogue_kernel`): a problem
   posts iteration << 1 | active only while it is active, so its last word names the iteration that converged it;
   the host resets the word to 1 and, after enqueuing iteration `it`, stops once every problem converged at an
   iteration <= it - 1.  A thread-per-rank simulation checks (a) that a single rank always stops, at most one no-op
   iteration late, however late it reads; (b) WHY the word is frozen at convergence rather than the current active
   bit read: a rank that reads the current bit late sees a later iteration's bit, enqueues fewer iterations than its
   peer, and the peer's next collective never completes; (c) that with the frozen word ranks reading late enqueue the
   same iterations and never hang."""
import threading
import time

import numpy as np


def _tree_sum(v, dtype):
    v = v.astype(dtype)
    while len(v) > 1:
        if len(v) & 1:
            v = np.concatenate([v, np.zeros(1, dtype)])
        v = (v[0::2] + v[1::2]).astype(dtype)
    return v[0]


def _seq_sum(v, dtype):
    acc = dtype(0)
    for t in v.astype(dtype):
        acc = dtype(acc + t)
    return acc


def _granule(v):
    """largest g with every non-zero term a multiple of 2^g (lloyd.cu pow2_granule)"""
    g = None
    for t in v:
        if t == 0:
            continue
        m, e = np.frexp(np.float64(abs(t)))        # t = m * 2^e, 0.5 <= m < 1
        k = 0
        while m != np.floor(m):
            m *= 2
            k += 1
        g = (e - k) if g is None else min(g, e - k)
    return g


def test_integer_valued_f32_terms_sum_identically_in_any_order():
    rng = np.random.default_rng(1)
    for _ in range(50):
        n = int(rng.integers(2, 3000))
        v = rng.integers(0, 256, n).astype(np.float32)          # SIFT / u8 columns: g = 0, sum < 2^24
        assert v.sum(dtype=np.float64) < 2 ** 24
        s = _seq_sum(v, np.float32)
        assert _tree_sum(v, np.float32) == s
        assert _tree_sum(rng.permutation(v), np.float32) == s
        assert s == np.float32(v.sum(dtype=np.float64))


def test_general_granule_condition_for_the_f64_loss():
    rng = np.random.default_rng(2)
    for _ in range(30):
        n = int(rng.integers(2, 2000))
        g = int(rng.integers(-30, 10))
        v = rng.integers(0, 1 << 20, n).astype(np.float64) * 2.0 ** g      # f32 distances widened to f64
        assert _granule(v) >= g and np.abs(v).sum() < 2.0 ** (g + 53)
        s = _seq_sum(v, np.float64)
        assert _tree_sum(v, np.float64) == s and _tree_sum(rng.permutation(v), np.float64) == s


def test_outside_the_condition_the_order_matters():
    """why the kernels TEST the condition per cluster and otherwise run the sequential chain"""
    rng = np.random.default_rng(3)
    differs = 0
    for _ in range(20):
        v = (rng.standard_normal(2000) * 100).astype(np.float32)            # arbitrary f32 residuals
        differs += int(_tree_sum(v, np.float32) != _seq_sum(v, np.float32))
    assert differs > 0
    big = np.full(70000, 255.0, np.float32)                                 # integers, but sum >= 2^24
    assert big.sum(dtype=np.float64) >= 2 ** 24
    assert _seq_sum(big, np.float32) != np.float32(big.sum(dtype=np.float64)) or _tree_sum(big, np.float32) != _seq_sum(big, np.float32)


def _settled(word, want, mode):
    """PollWords::done waits on a problem until this holds"""
    if mode == "frozen":
        return not (word & 1) or (word >> 1) >= want
    return (word >> 1) >= want


def _converged_by(word, want, mode):
    """the host's decision for one problem once its word has settled"""
    if mode == "frozen":
        return not (word & 1) and (word >> 1) <= want
    return not (word & 1)


class _Rank:
    """one rank of the simulation: a `device` thread executes enqueued iterations in order (each takes `iter_s`);
    iteration j contains the collective of iteration j, i.e. it needs every rank's device to reach it (a barrier).
    Its epilogue posts the progress word of `mode`:
      * "frozen" (what lloyd_train does): j << 1 | active, posted only while the problem is active, so the last word
        names the iteration that converged it; the host resets the word to 1 (iteration 0, active) before iteration 1;
      * "current_bit": (epilogues run) << 1 | active, posted by every epilogue; the host resets it to 0.
    The host loop is lloyd_train's; `late_by` makes the host read only once the device is that many iterations
    further than it had to wait for (pre-emption, a slow graph launch, a CPU quota ...) -- scripted in ticks, not in
    seconds, so that the tests do not depend on the machine's speed."""

    def __init__(self, world, barrier_for, converge_at, max_iters, mode, late_by=0, iter_s=0.0):
        self.world, self.barrier_for, self.converge_at, self.max_iters = world, barrier_for, converge_at, max_iters
        self.mode, self.late_by, self.iter_s = mode, late_by, iter_s
        self.queue, self.cv = [], threading.Condition()
        self.word = 1 if mode == "frozen" else 0
        self.executed = self.enqueued = self.executed_active = 0
        self.hist = {0: self.word}                     # iteration -> the word once that iteration has run
        self.stop = self.hung = False

    def device(self):
        active = True
        while True:
            with self.cv:
                while not self.queue and not self.stop:
                    self.cv.wait(0.001)
                if not self.queue:
                    return
                j = self.queue.pop(0)
            try:
                self.barrier_for(j).wait(timeout=4.0)  # the exchange inside the captured iteration
            except threading.BrokenBarrierError:
                self.hung = True                       # a peer never enqueued iteration j: NCCL would wait forever
                return
            time.sleep(self.iter_s)
            posts = active or self.mode == "current_bit"
            if active:
                self.executed_active += 1
                active = j < self.converge_at          # kmeans.rs:704 on identical models: same j on every rank
            word = (j << 1) | int(active) if posts else self.word
            self.hist[j] = word
            self.executed = j
            self.word = word

    def host(self):
        def launch(j):
            with self.cv:
                self.queue.append(j)
                self.enqueued += 1
                self.cv.notify()
        launch(1)
        done, it = self.max_iters == 1, 2
        while it <= self.max_iters and not done:
            launch(it)
            want = it - 1
            t0 = time.monotonic()
            while not _settled(self.word, want, self.mode) and not self.hung:  # (the real host spins)
                time.sleep(0.0001)
                assert time.monotonic() - t0 < 20, "progress word never arrived"
            seen = min(want + self.late_by, self.enqueued)     # the iteration whose word this (late) read observes
            t1 = time.monotonic()
            while self.executed < seen and not self.hung and time.monotonic() - t1 < 6.0:
                time.sleep(0.0001)
            done = _converged_by(self.hist[min(seen, self.executed)], want, self.mode)
            it += 1
        t0 = time.monotonic()
        while self.executed < self.enqueued and not self.hung and time.monotonic() - t0 < 8:
            time.sleep(0.0001)                                 # the final synchronise of lloyd_train
        self.stop = True


def _simulate(world, converge_at, max_iters, mode="frozen", late=None, iter_s=0.0):
    barriers, lock = {}, threading.Lock()

    def barrier_for(j):
        with lock:
            if j not in barriers:
                barriers[j] = threading.Barrier(world)
            return barriers[j]

    ranks = [_Rank(world, barrier_for, converge_at, max_iters, mode, (late or [0] * world)[r], iter_s) for r in range(world)]
    threads = [threading.Thread(target=r.device) for r in ranks] + [threading.Thread(target=r.host) for r in ranks]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=60)
        assert not t.is_alive(), "simulation did not end"
    return ranks


def test_the_reset_word_reads_as_active_and_a_zero_would_read_as_converged():
    for want in range(1, 6):
        assert not _settled(1, want, "frozen") and not _converged_by(1, want, "frozen")
        assert _settled(0, want, "frozen") and _converged_by(0, want, "frozen")


def test_single_rank_always_stops_at_most_one_noop_late_whatever_the_read_timing():
    for mode in ("frozen", "current_bit"):
        for converge_at, max_iters, late in ((7, 50, 0), (7, 50, 1), (7, 50, 3), (1, 50, 0), (50, 50, 0), (60, 50, 1),
                                             (3, 4, 0), (2, 4, 1), (1, 1, 0)):
            r, = _simulate(1, converge_at, max_iters, mode=mode, late=[late], iter_s=0.0005)
            last_real = min(converge_at, max_iters)
            assert not r.hung and r.executed_active == last_real            # extra iterations were no-ops
            assert last_real <= r.enqueued <= min(max_iters, last_real + 1)
            if mode == "frozen":                                            # and the count does not depend on timing
                assert r.enqueued == min(max_iters, last_real + 1)


def test_two_ranks_reading_the_current_bit_can_diverge_which_is_why_the_word_freezes_at_convergence():
    # rank 0 reads one iteration late: waiting for iteration 4 it already sees iteration 5's bit and stops after
    # enqueuing 5; rank 1 sees that bit one check later, after enqueuing 6 -- whose collective rank 0 never joins
    ranks = _simulate(2, 5, 50, mode="current_bit", late=[1, 0], iter_s=0.0005)
    assert ranks[0].enqueued == 5 and ranks[1].enqueued == 6 and ranks[1].hung


def test_reporting_the_tick_of_convergence_is_independent_of_read_timing():
    for converge_at, max_iters, late in ((5, 50, [1, 0]), (5, 50, [0, 1, 0]), (5, 50, [1, 1]), (5, 50, [3, 0]),
                                         (2, 50, [0, 2]), (3, 4, [1, 0]), (9, 6, [2, 0, 1])):
        ranks = _simulate(len(late), converge_at, max_iters, late=late, iter_s=0.0005)
        last_real = min(converge_at, max_iters)
        assert not any(r.hung for r in ranks)
        assert {r.enqueued for r in ranks} == {min(max_iters, last_real + 1)}
        assert all(r.executed_active == last_real for r in ranks)


# ---- 3. the k + 1 rule of every top-k path (DESIGN.md section 5 "Ties at the k-th distance"; topk.cuh) ----------
# The GPU selects k + 1 candidates per list.  Argument: when the (k+1)-th smallest distance differs from the k-th, the
# reference's BinaryHeap result (flat/index.rs:82-177, restated in the oracle) is the unique set of the k smallest --
# whatever order the rows were pushed in -- so any selection algorithm returns it; only when they are equal does the
# result depend on the heap's sift order, and only then the slot is replayed with the heap's own operations.
def test_topk_set_is_order_free_unless_the_boundary_is_tied():
    from oracle import binding as ob
    rng = np.random.default_rng(4)
    tied_boundaries = 0
    for trial in range(200):
        n, k = int(rng.integers(5, 400)), int(rng.integers(1, 20))
        d = rng.integers(0, 40, n).astype(np.float32)                      # small integers: ties everywhere
        if trial % 3 == 0:
            d = d + rng.random(n).astype(np.float32)                        # and some tie-free inputs
        rid = np.arange(n, dtype=np.uint64)
        ids, dd = ob.flat_topk(d, rid, k)
        srt = np.sort(d, kind="stable")
        kk = min(k, n)
        assert np.array_equal(np.sort(dd), srt[:kk])                        # the distance multiset is always exact
        if kk < n and srt[kk] == srt[kk - 1]:
            tied_boundaries += 1                                            # heap order decides: the replay's domain
            continue
        expect = set(np.flatnonzero(d <= srt[kk - 1]).tolist()) if kk else set()
        assert set(ids.tolist()) == expect and len(expect) == kk
        perm = rng.permutation(n)                                           # push order does not matter here
        ids2, _ = ob.flat_topk(d[perm], rid[perm], k)
        assert set(ids2.tolist()) == expect
    assert tied_boundaries > 20                                             # the tied case is common on such data
