// kmeans.cu -- the k-means entry (KMeans::new_with_params, kmeans.rs:1008-1030): train_kmeans chooses between one
// flat Lloyd run (lloyd.cu) and the hierarchical tree for K > 256, which is host orchestration around many small
// Lloyd runs.
#include <algorithm>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <thread>
#include <unordered_map>

#include "assign.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "kmeans.cuh"
#include "member_sort.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// hierarchical k-means for k > 256 (kmeans.rs:746-1003): top level with k0 = min(16, k, n), then the
// largest cluster is repeatedly split by a small k-means (k' <= 16) on its rows until k clusters
// exist.  The heap is Rust's BinaryHeap restated (push = sift_up, pop = swap + sift_down_to_bottom +
// sift_up; library/alloc/src/collections/binary_heap) ordered by (not finalized, size); the j-th
// training call uses seed + j (the reference is unseeded).  Row index lists stay on the device.
// ------------------------------------------------------------------------------------------------
namespace {
struct HCluster {
  uint32_t id;
  uint32_t off, loc;  // this rank's segment of the device index array (loc rows)
  uint64_t len;       // rows of the cluster over ALL ranks: what the reference's heap orders by
  bool finalized;
};
inline bool hc_le(const HCluster& a, const HCluster& b) {  // a <= b in the reference's Ord
  if (a.finalized != b.finalized) return a.finalized;  // finalized < not finalized
  return a.len <= b.len;
}
struct RustHeap {
  std::vector<HCluster> data;
  void sift_up(size_t start, size_t pos) {
    HCluster elt = data[pos];
    while (pos > start) {
      size_t parent = (pos - 1) / 2;
      if (hc_le(elt, data[parent])) break;
      data[pos] = data[parent];
      pos = parent;
    }
    data[pos] = elt;
  }
  void push(const HCluster& c) {
    data.push_back(c);
    sift_up(0, data.size() - 1);
  }
  HCluster pop() {
    HCluster item = data.back();
    data.pop_back();
    if (!data.empty()) {
      std::swap(item, data[0]);
      size_t end = data.size(), pos = 0;
      HCluster elt = data[0];
      size_t child = 1;
      while (child + 1 < end) {
        if (hc_le(data[child], data[child + 1])) child += 1;
        data[pos] = data[child];
        pos = child;
        child = 2 * pos + 1;
      }
      if (child + 1 == end) {
        data[pos] = data[child];
        pos = child;
      }
      data[pos] = elt;
      sift_up(0, pos);
    }
    return item;
  }
};
__global__ void gather_rows_u32_kernel(const float* __restrict__ x, const uint32_t* __restrict__ rows,
                                       uint64_t s, int d, float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= s * d) return;
  out[g] = x[(uint64_t)rows[g / d] * d + g % d];
}
__global__ void compose_index_kernel(const uint32_t* __restrict__ parent, const uint32_t* __restrict__ members,
                                     uint32_t cnt, uint32_t* __restrict__ out) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < cnt) out[g] = parent[members[g]];
}
}  // namespace

namespace {
// ---- one split = gather the cluster's rows, Lloyd, membership, stable sort, children's row lists -----------------
struct SplitOut {
  int ck = 0;
  std::vector<uint32_t> counts, offs;
  DevBuf<float> subc;       // [ck][d]
  DevBuf<uint32_t> order;   // the parent's row list re-ordered by (child, position), `kept` entries
  uint32_t kept = 0;
  std::map<std::string, ProfEntry> prof;  // kernels of a worker thread, merged into the caller's profile
  uint64_t launches = 0;
  std::exception_ptr err;
};
// the split of cluster `id` trains with seed + 1 + id
void split_cluster(const float* x, int d, const uint32_t* idx_seg, uint32_t loc, int ck, const LloydParams& p, uint32_t id,
                   SplitOut& o) {
  o.ck = ck;
  o.subc.alloc((size_t)ck * d);
  const uint64_t n1 = std::max<uint32_t>(loc, 1);
  DevBuf<float> sub(n1 * d);
  DevBuf<uint32_t> ids(n1);
  DevBuf<uint8_t> valid(n1);
  if (loc)
    LB2_LAUNCH("gather_rows", gather_rows_u32_kernel, cdiv((uint64_t)loc * d, 256), 256, 0, x, idx_seg, (uint64_t)loc, d,
               sub.p);
  LloydParams ps = p;
  ps.seed = p.seed + 1 + id;
  lloyd_train(sub.p, loc, d, 1, d, ck, ps, nullptr, o.subc.p, nullptr, nullptr);
  assign_f32(sub.p, loc, d, o.subc.p, ck, p.metric, nullptr, ids.p, nullptr, valid.p);
  MemberSort ms;
  ms.run(ids.p, valid.p, loc, ck, 1, nullptr);
  o.counts.resize(ck);
  o.offs.resize(ck + 1);
  d2h(o.counts.data(), ms.counts.p, ck);
  d2h(o.offs.data(), ms.offsets.p, ck + 1);
  sync_stream();
  // children's row lists = parent's list re-ordered by (child, position): stable; rows dropped as None by the
  // membership step leave the lists
  o.kept = o.offs[ck];
  if (o.kept) {
    o.order.alloc(o.kept);
    LB2_LAUNCH("compose_index", compose_index_kernel, cdiv(o.kept, 256), 256, 0, idx_seg, ms.members.p, o.kept, o.order.p);
  }
  sync_stream();
}

// ---- worker threads: independent splits train concurrently (each thread has its own stream) ---------------------
// A split is a chain of small dependent kernels (a few thousand rows, k <= 16): one stream leaves the GPU almost
// idle.  The sequential algorithm is kept EXACTLY -- splits are committed in the heap's pop order -- but the
// clusters that will reach the top of the heap soon are trained ahead of time on worker threads; their results
// wait in a cache keyed by cluster id (a split depends only on the cluster's rows, ck and seed + 1 + id).
class SplitWorkers {
 public:
  static SplitWorkers& get() {
    static SplitWorkers* w = new SplitWorkers();  // lives (with its detached threads) until the process exits
    return *w;
  }
  int threads() const { return nthreads_; }
  // The pool is shared by every thread that trains at once, so each caller counts only its own tasks: a wave waits
  // for its tasks, not for a queue that another training keeps filling.
  struct Wave {
    int pending = 0;
  };
  void submit(Wave& w, std::function<void()> f) {
    {
      std::lock_guard<std::mutex> lk(m_);
      ++w.pending;
      q_.push_back([this, &w, f = std::move(f)] {
        f();
        std::lock_guard<std::mutex> lk(m_);
        if (--w.pending == 0) done_.notify_all();
      });
    }
    cv_.notify_one();
  }
  void wait(Wave& w) {
    std::unique_lock<std::mutex> lk(m_);
    done_.wait(lk, [&] { return w.pending == 0; });
  }

 private:
  SplitWorkers() {
    const char* e = getenv("LB2_SPLIT_THREADS");
    nthreads_ = e && *e ? std::max(0, atoi(e) - 1) : 2;  // measured: 482 / 379 / 378 / 484 ms at 1 / 2 / 4 / 8 threads (launch-throughput bound)
    for (int i = 0; i < nthreads_; ++i) std::thread([this] { loop(); }).detach();
  }
  void loop() {
    for (;;) {
      std::function<void()> f;
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return !q_.empty(); });
        f = std::move(q_.front());
        q_.pop_front();
      }
      f();
    }
  }
  int nthreads_ = 0;
  std::mutex m_;
  std::condition_variable cv_, done_;
  std::deque<std::function<void()>> q_;
};
}  // namespace

// Sharded (SURVEY 8e): every rank holds a row shard of the sample and runs the SAME split loop -- the heap is
// ordered by the clusters' global sizes (one small all-reduce of <= 16 counters per split), each Lloyd run
// exchanges its partial sums once per iteration (lloyd_train), the row index lists stay local to the rank.
void hierarchical_train(const float* x, uint64_t n, int d, int K, const LloydParams& p, int hk, float* centroids_out) {
  Comm* cm = current_comm();
  const bool dist = cm && cm->nranks > 1;
  LB2_REQUIRE(n < 0xffffffffull, "KMeans: too many vectors");
  // local per-cluster counts -> global counts (identity on one GPU)
  auto global_counts = [&](const std::vector<uint32_t>& local, int k, std::vector<uint64_t>& out) {
    std::vector<uint32_t> sum(local.begin(), local.begin() + k);
    sum_over_ranks(sum);
    out.assign(sum.begin(), sum.end());
  };
  std::vector<uint32_t> n_sum(1, (uint32_t)n);
  sum_over_ranks(n_sum);
  const uint64_t n_global = n_sum[0];
  LB2_REQUIRE(n_global >= (uint64_t)K, "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n_global);
  const int k0 = (int)std::min<uint64_t>(std::min(hk, K), n_global);
  const uint64_t n1 = std::max<uint64_t>(n, 1);
  DevBuf<float> top((size_t)k0 * d), store((size_t)2 * K * d + (size_t)k0 * d);
  DevBuf<uint32_t> ids(n1), idx(n1);
  DevBuf<uint8_t> valid(n1);
  lloyd_train(x, n, d, 1, d, k0, p, nullptr, top.p, nullptr, nullptr);
  assign_f32(x, n, d, top.p, k0, p.metric, nullptr, ids.p, nullptr, valid.p);
  std::vector<uint32_t> counts(std::max(k0, hk)), offs(std::max(k0, hk) + 1);
  std::vector<uint64_t> gcounts;
  {
    MemberSort ms;
    ms.run(ids.p, valid.p, n, k0, 1, nullptr);
    d2h(counts.data(), ms.counts.p, k0);
    d2h(offs.data(), ms.offsets.p, k0 + 1);
    if (n) d2d(idx.p, ms.members.p, n);
    sync_stream();
  }
  ids.release();
  valid.release();
  global_counts(counts, k0, gcounts);
  RustHeap heap;
  uint32_t next_id = 0;
  const size_t store_slots = (size_t)2 * K + k0;
  for (int i = 0; i < k0; ++i) {
    if (gcounts[i] == 0) continue;
    d2d(store.p + (size_t)next_id * d, top.p + (size_t)i * d, d);
    heap.push(HCluster{next_id++, offs[i], counts[i], gcounts[i], false});
  }
  auto children_of = [&](uint64_t len, int remaining) {
    if (len <= (uint64_t)hk) return std::min(std::min(2, remaining), (int)len);
    return std::max(2, std::min(std::min((int)std::min<uint64_t>(len / hk, 1u << 30), remaining), hk));
  };
  // concurrency only without a communicator (NCCL calls of one communicator must not interleave across threads;
  // sharded builds whose sample fits one GPU gather it and come here without one, build.cu:train_ivf)
  SplitWorkers* workers = dist ? nullptr : &SplitWorkers::get();
  const int width = workers ? workers->threads() + 1 : 1;
  std::unordered_map<uint32_t, std::unique_ptr<SplitOut>> cache;
  int device = 0;
  cudaGetDevice(&device);
  Ctx& me = ctx();
  while ((int)heap.data.size() < K) {
    LB2_REQUIRE(!heap.data.empty(), "No cluster can be further split");
    HCluster big = heap.pop();
    if (big.finalized || big.len <= 1) {  // kmeans.rs:868-881: stop splitting
      heap.push(big);
      break;
    }
    const int remaining = K - (int)heap.data.size();
    const int ck = children_of(big.len, remaining);
    std::unique_ptr<SplitOut> out;
    auto hit = cache.find(big.id);
    if (hit != cache.end()) {
      if (hit->second->ck == ck) out = std::move(hit->second);  // else: the end game changed ck -> train again
      cache.erase(hit);
    }
    if (!out) {
      // this cluster + the clusters that will be popped soon (largest first; the exact pop order among equals
      // does not matter here -- a result is only used when its cluster is popped, and checked against ck then)
      std::vector<HCluster> wave{big};
      std::vector<int> wck{ck};
      if (width > 1 && remaining - ck > 2 * hk) {
        auto lt = [&](size_t a, size_t b) { return !hc_le(heap.data[b], heap.data[a]); };  // max-first
        std::priority_queue<size_t, std::vector<size_t>, decltype(lt)> front(lt);
        if (!heap.data.empty()) front.push(0);
        uint64_t rows = big.loc;
        int budget = remaining - ck;
        while (!front.empty() && (int)wave.size() < width) {
          const size_t i = front.top();
          front.pop();
          const HCluster& c = heap.data[i];
          if (c.finalized || c.len <= 1) break;  // the sequential loop stops there
          if (2 * i + 1 < heap.data.size()) front.push(2 * i + 1);
          if (2 * i + 2 < heap.data.size()) front.push(2 * i + 2);
          if (cache.count(c.id)) continue;
          const int cck = children_of(c.len, K);  // `remaining` not binding ...
          budget -= cck;
          if (budget <= 2 * hk) break;            // ... which is only certain away from the end game
          rows += c.loc;
          if (rows * (uint64_t)d * 4 > (4ull << 30)) break;
          wave.push_back(c);
          wck.push_back(cck);
        }
      }
      std::vector<std::unique_ptr<SplitOut>> outs(wave.size());
      for (auto& o : outs) o.reset(new SplitOut());
      sync_stream();  // the row lists written by earlier commits are visible to the workers' streams
      const bool prof_on = me.profiling;
      const std::string tag = me.tag;
      SplitWorkers::Wave tasks;
      for (size_t w = 1; w < wave.size(); ++w) {
        SplitOut* o = outs[w].get();
        const HCluster c = wave[w];
        const int cck = wck[w];
        workers->submit(tasks, [=, &idx]() {
          try {
            lb2_set_device(device);
            Ctx& wc = ctx();
            wc.profiling = prof_on;
            wc.tag = tag;
            wc.prof.clear();
            wc.launches = 0;
            split_cluster(x, d, idx.p + c.off, c.loc, cck, p, c.id, *o);
            wc.flush_profile();
            o->prof.swap(wc.prof);
            o->launches = wc.launches;
            wc.profiling = false;
          } catch (...) {
            o->err = std::current_exception();
          }
        });
      }
      try {
        split_cluster(x, d, idx.p + big.off, big.loc, ck, p, big.id, *outs[0]);
      } catch (...) {
        outs[0]->err = std::current_exception();
      }
      if (wave.size() > 1) workers->wait(tasks);
      for (size_t w = 0; w < wave.size(); ++w) {
        if (outs[w]->err) std::rethrow_exception(outs[w]->err);
        me.launches += outs[w]->launches;
        for (auto& kv : outs[w]->prof) {
          me.prof[kv.first].launches += kv.second.launches;
          me.prof[kv.first].total_ms += kv.second.total_ms;
        }
        if (w) cache[wave[w].id] = std::move(outs[w]);
      }
      out = std::move(outs[0]);
    }
    global_counts(out->counts, ck, gcounts);
    int nonzero = 0;
    for (int i = 0; i < ck; ++i) nonzero += gcounts[i] > 0;
    if (nonzero <= 1) {  // ineffective split: finalise the original cluster (kmeans.rs:957-962)
      big.finalized = true;
      heap.push(big);
      continue;
    }
    if (out->kept) d2d(idx.p + big.off, out->order.p, out->kept);
    for (int i = 0; i < ck; ++i) {
      if (gcounts[i] == 0) continue;
      LB2_REQUIRE(next_id < store_slots, "hierarchical k-means: centroid store exhausted");
      d2d(store.p + (size_t)next_id * d, out->subc.p + (size_t)i * d, d);
      heap.push(HCluster{next_id++, big.off + out->offs[i], out->counts[i], gcounts[i], false});
    }
    sync_stream();  // `out` (and its device buffers) goes away here
  }
  if ((int)heap.data.size() != K)
    fail(LB2_INVALID_ARG, "hierarchical k-means produced %zu of %d clusters (no cluster can be further split)",
         heap.data.size(), K);
  std::vector<HCluster> all = heap.data;
  std::sort(all.begin(), all.end(), [](const HCluster& a, const HCluster& b) { return a.id < b.id; });
  for (int i = 0; i < K; ++i) d2d(centroids_out + (size_t)i * d, store.p + (size_t)all[i].id * d, d);
  sync_stream();
}

void train_kmeans(const float* x, uint64_t n, int d, int K, int metric, const lb2_kmeans_params& kp, const float* init,
                  float* centroids, std::vector<double>* loss, std::vector<uint32_t>* iters) {
  const LloydParams p{metric, kp.balance_factor / (float)(n * comm_nranks()), (int)kp.max_iters, kp.tolerance, kp.seed};
  if (!kmeans_uses_tree(K, kp, init)) {
    lloyd_train(x, n, d, 1, d, K, p, init, centroids, loss, iters);
    return;
  }
  hierarchical_train(x, n, d, K, p, (int)kp.hierarchical_k, centroids);
  loss->assign(1, 0.0);
  iters->assign(1, 0);
}

}  // namespace lb2
