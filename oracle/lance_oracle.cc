// lance_oracle.cc -- CPU restatement of the reference's IVF-PQ hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under lance_b200/ may include, link or call this file;
// only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it.
//
// Every function cites the reference file:line (relative to /root/reference/rust) whose operation
// ORDER it follows.  It is compiled with FP contraction off (see Makefile), because Rust/LLVM never
// fuses `a*b+c` for the reference's scalar loops.
//
// Parity pinning: the known-answer literals from the reference's own unit tests are stored in
// tests/golden/reference_known_answers.json and checked against this file by tests/test_oracle_golden.py.
// What is NOT pinned (reference is unseeded / implementation-defined there, see SURVEY.md 8c):
//   * the k-means RNG stream (init rows, split_clusters donors)  -> we define our own (splitmix64),
//   * the order among EQUAL centroid distances in find_partitions (arrow-ord partial sort)
//       -> we define ascending (distance, id).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <condition_variable>
#include <functional>
#include <limits>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace {

// ---------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------
// Persistent worker pool (the reference runs these loops on rayon's global pool: threads are created once
// and parked between jobs, rust/lance-index/src/vector/kmeans.rs:335-356 `par_chunks`).  Like rayon:
//   * workers SPIN for the next job for a while before they sleep (the ~1000 short parallel regions of a
//     k-means run are microseconds apart), a job is published with two atomic stores, no wake-up storm;
//   * a job is finished when its CHUNKS are finished, not when every worker has shown up: a worker the OS
//     has descheduled (shared hosts) simply contributes nothing; it can never touch a finished job's closure,
//     because the closure is only entered after claiming a chunk and all chunks are claimed before the
//     caller returns (the job record itself is reference counted).
// Per-row results do not depend on the schedule.
class Pool {
  struct Job {
    std::function<void(size_t, size_t)> f;
    size_t n = 0, chunk = 1, total_chunks = 0, helpers = 0;
    std::atomic<size_t> next{0}, done_chunks{0};
    void work() {
      for (;;) {
        const size_t b = next.fetch_add(chunk, std::memory_order_relaxed);
        if (b >= n) break;
        f(b, std::min(n, b + chunk));
        done_chunks.fetch_add(1, std::memory_order_release);
      }
    }
  };

 public:
  static Pool& get() {
    static Pool p;
    return p;
  }
  template <class F>
  void run(size_t n, int nthreads, F&& f) {
    std::lock_guard<std::mutex> run_lock(run_mu_);  // one job at a time
    const size_t nt = std::min<size_t>(std::min<size_t>(size_t(nthreads), n), 4096);
    ensure(nt - 1);
    auto job = std::make_shared<Job>();
    job->f = std::ref(f);
    job->n = n;
    job->chunk = std::max<size_t>(1, n / (nt * 8));
    job->total_chunks = (n + job->chunk - 1) / job->chunk;
    job->helpers = nt - 1;
    std::atomic_store(&cur_, job);
    gen_.fetch_add(1, std::memory_order_release);
    if (sleepers_.load(std::memory_order_acquire) > 0) {
      std::lock_guard<std::mutex> lk(mu_);
      cv_.notify_all();
    }
    job->work();
    while (job->done_chunks.load(std::memory_order_acquire) != job->total_chunks) cpu_relax();
    std::atomic_store(&cur_, std::shared_ptr<Job>());
  }

 private:
  Pool() = default;
  ~Pool() {
    stop_.store(true);
    {
      std::lock_guard<std::mutex> lk(mu_);
      gen_.fetch_add(1);
      cv_.notify_all();
    }
    for (auto& t : th_) t.join();
  }
  static void cpu_relax() {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#else
    std::this_thread::yield();
#endif
  }
  void ensure(size_t helpers) {
    while (th_.size() < helpers) {
      const size_t id = th_.size();
      const uint64_t start_gen = gen_.load();
      th_.emplace_back([this, id, start_gen] { worker(id, start_gen); });
    }
  }
  void worker(size_t id, uint64_t seen) {
    for (;;) {
      int spins = 0;
      while (gen_.load(std::memory_order_acquire) == seen) {
        if (++spins < 20000) {  // ~0.2 ms of polling: the next parallel region is usually that close
          cpu_relax();
        } else {
          sleepers_.fetch_add(1, std::memory_order_acq_rel);
          {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] { return gen_.load(std::memory_order_acquire) != seen; });
          }
          sleepers_.fetch_sub(1, std::memory_order_acq_rel);
          spins = 0;
        }
      }
      seen = gen_.load(std::memory_order_acquire);
      if (stop_.load()) return;
      std::shared_ptr<Job> job = std::atomic_load(&cur_);
      if (job && id < job->helpers) job->work();
    }
  }
  std::mutex mu_, run_mu_;
  std::condition_variable cv_;
  std::vector<std::thread> th_;
  std::shared_ptr<Job> cur_;
  std::atomic<uint64_t> gen_{0};
  std::atomic<int> sleepers_{0};
  std::atomic<bool> stop_{false};
};

template <class F>
void parallel_for(size_t n, int nthreads, F f) {
  if (nthreads <= 1 || n < 2) {
    f(size_t(0), n);
    return;
  }
  Pool::get().run(n, nthreads, f);
}

// splitmix64: OUR rng for init / split_clusters (reference uses an unseeded SmallRng,
// lance-index/src/vector/kmeans.rs:181,646 -> parity unpinned by design).
struct SplitMix64 {
  uint64_t s;
  explicit SplitMix64(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  // uniform in [0,1) with 24 bits, like rand's Standard f32 sampling
  float next_f32() { return float(next() >> 40) * (1.0f / 16777216.0f); }
};

inline float half_to_float(uint16_t h) {
  uint32_t sign = (uint32_t(h) & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1f;
  uint32_t man = h & 0x3ff;
  uint32_t f;
  if (exp == 0) {
    if (man == 0) {
      f = sign;
    } else {
      int e = -1;
      do {
        man <<= 1;
        ++e;
      } while (!(man & 0x400));
      f = sign | uint32_t(127 - 15 - e) << 23 | (man & 0x3ff) << 13;
    }
  } else if (exp == 31) {
    f = sign | 0x7f800000u | man << 13;
  } else {
    f = sign | (exp + 112) << 23 | man << 13;
  }
  float out;
  std::memcpy(&out, &f, 4);
  return out;
}
inline float bf16_to_float(uint16_t h) {
  uint32_t f = uint32_t(h) << 16;
  float out;
  std::memcpy(&out, &f, 4);
  return out;
}

// ---------------------------------------------------------------------------------------------
// A1. squared L2, f32, 16 lanes   (lance-linalg/src/distance/l2.rs:57-91, LANES=16 at :161-168)
// ---------------------------------------------------------------------------------------------
template <class T, class Conv>
inline float l2_lanes16(const T* x, const T* y, size_t d, Conv conv) {
  const size_t n16 = d / 16 * 16;
  // remainder first: `.sum::<f32>()` folds left-to-right (l2.rs:69-79)
  float s = 0.0f;
  for (size_t i = n16; i < d; ++i) {
    float diff = conv(x[i]) - conv(y[i]);
    s += diff * diff;
  }
  float sums[16];
  for (int l = 0; l < 16; ++l) sums[l] = 0.0f;
  for (size_t c = 0; c < n16; c += 16)  // l2.rs:82-88
    for (int l = 0; l < 16; ++l) {
      float diff = conv(x[c + l]) - conv(y[c + l]);
      sums[l] += diff * diff;
    }
  float t = 0.0f;  // `sums.iter().copied().sum()` (l2.rs:90)
  for (int l = 0; l < 16; ++l) t += sums[l];
  return s + t;
}
inline float l2_f32(const float* x, const float* y, size_t d) {
  return l2_lanes16(x, y, d, [](float v) { return v; });
}

// A2. dot, f32, 16 lanes (lance-linalg/src/distance/dot.rs:30-58, LANES=16 at :138-143)
inline float dot_f32(const float* x, const float* y, size_t d) {
  const size_t n16 = d / 16 * 16;
  float s = 0.0f;
  for (size_t i = n16; i < d; ++i) s += x[i] * y[i];
  float sums[16];
  for (int l = 0; l < 16; ++l) sums[l] = 0.0f;
  for (size_t c = 0; c < n16; c += 16)
    for (int l = 0; l < 16; ++l) sums[l] += x[c + l] * y[c + l];
  float t = 0.0f;
  for (int l = 0; l < 16; ++l) t += sums[l];
  return s + t;
}
// norm_l2 f32 (lance-linalg/src/distance/norm_l2.rs:106-130, LANES=16 for f32)
inline float norm_l2_f32(const float* x, size_t d) {
  const size_t n16 = d / 16 * 16;
  float s = 0.0f;
  for (size_t i = n16; i < d; ++i) s += x[i] * x[i];
  float sums[16];
  for (int l = 0; l < 16; ++l) sums[l] = 0.0f;
  for (size_t c = 0; c < n16; c += 16)
    for (int l = 0; l < 16; ++l) sums[l] += x[c + l] * x[c + l];
  float t = 0.0f;
  for (int l = 0; l < 16; ++l) t += sums[l];
  return std::sqrt(s + t);
}

inline float metric_dist(int metric, const float* x, const float* y, size_t d) {
  // 0 = L2, 2 = Dot (dot_distance = 1 - dot, dot.rs:68-70)
  return metric == 2 ? 1.0f - dot_f32(x, y, d) : l2_f32(x, y, d);
}

// A4. argmin with bias (lance-linalg/src/kernels.rs:79-111)
//   strict `<` against +inf start -> first minimum wins, NaN / +inf never win.
inline bool argmin_row(const float* centroids, size_t k, size_t d, const float* v, int metric,
                       const float* bias, uint32_t* idx_out, float* val_out) {
  float min_value = std::numeric_limits<float>::infinity();
  float min_orig = std::numeric_limits<float>::infinity();
  bool found = false;
  uint32_t min_idx = 0;
  for (size_t c = 0; c < k; ++c) {
    float val = metric_dist(metric, v, centroids + c * d, d);
    float cmp = bias ? val + bias[c] : val;
    if (cmp < min_value) {
      min_value = cmp;
      min_orig = val;
      min_idx = uint32_t(c);
      found = true;
    }
  }
  *idx_out = min_idx;
  *val_out = min_orig;
  return found;
}

// Rust std::collections::BinaryHeap<OrderedNode> restated (push = sift_up, pop = swap-with-last +
// sift_down_to_bottom + sift_up), ordered by f32::total_cmp on dist
// (lance-index/src/vector/graph.rs:66-121).  Rust std is third-party to /root/reference; its
// algorithm is restated from the published std source (library/alloc/src/collections/binary_heap).
struct Node {
  uint64_t id;
  float dist;
};
inline int32_t total_key(float f) {
  int32_t b;
  std::memcpy(&b, &f, 4);
  return b ^ int32_t(uint32_t(b >> 31) >> 1);
}
inline bool le(const Node& a, const Node& b) { return total_key(a.dist) <= total_key(b.dist); }
inline bool gt(float a, float b) { return total_key(a) > total_key(b); }
struct RustMaxHeap {
  std::vector<Node> data;
  void sift_up(size_t start, size_t pos) {
    Node elt = data[pos];
    while (pos > start) {
      size_t parent = (pos - 1) / 2;
      if (le(elt, data[parent])) break;
      data[pos] = data[parent];
      pos = parent;
    }
    data[pos] = elt;
  }
  void push(Node n) {
    size_t old = data.size();
    data.push_back(n);
    sift_up(0, old);
  }
  void sift_down_to_bottom(size_t pos) {
    size_t end = data.size();
    size_t start = pos;
    Node elt = data[pos];
    size_t child = 2 * pos + 1;
    while (child + 1 < end) {  // child <= end.saturating_sub(2)
      if (le(data[child], data[child + 1])) child += 1;
      data[pos] = data[child];
      pos = child;
      child = 2 * pos + 1;
    }
    if (child + 1 == end) {
      data[pos] = data[child];
      pos = child;
    }
    data[pos] = elt;
    sift_up(start, pos);
  }
  Node pop() {
    Node item = data.back();
    data.pop_back();
    if (!data.empty()) {
      std::swap(item, data[0]);
      sift_down_to_bottom(0);
    }
    return item;
  }
};

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------
// distances
// ---------------------------------------------------------------------------------------------
float lo_l2_f32(const float* x, const float* y, uint64_t d) { return l2_f32(x, y, d); }
float lo_dot_f32(const float* x, const float* y, uint64_t d) { return dot_f32(x, y, d); }
float lo_norm_l2_f32(const float* x, uint64_t d) { return norm_l2_f32(x, d); }
// u8: sum |x-y|^2 in u32, cast to f32 (l2.rs:44-49)
float lo_l2_u8(const uint8_t* x, const uint8_t* y, uint64_t d) {
  uint32_t s = 0;
  for (uint64_t i = 0; i < d; ++i) {
    uint32_t a = x[i] > y[i] ? x[i] - y[i] : y[i] - x[i];
    s += a * a;
  }
  return float(s);
}
// f16 / bf16 scalar path: convert each element to f32, LANES=16 (l2.rs:100-106,156)
float lo_l2_f16(const uint16_t* x, const uint16_t* y, uint64_t d) {
  return l2_lanes16(x, y, d, [](uint16_t v) { return half_to_float(v); });
}
float lo_l2_bf16(const uint16_t* x, const uint16_t* y, uint64_t d) {
  return l2_lanes16(x, y, d, [](uint16_t v) { return bf16_to_float(v); });
}
// f16 / bf16 dot: dot_scalar::<T, f32, 32> (dot.rs:30-58): every element converted to f32, the d % 32 tail summed
// first, then 32 lane accumulators folded 0..31.  bf16 always takes it (dot.rs:78-83); f16 takes it where the
// fp16kernels C kernel is not compiled in (dot.rs:105-136, fallback at :133).
static float dot_lanes32(const uint16_t* x, const uint16_t* y, uint64_t d, float (*conv)(uint16_t)) {
  const uint64_t n32 = d / 32 * 32;
  float s = 0.0f;
  for (uint64_t i = n32; i < d; ++i) s += conv(x[i]) * conv(y[i]);
  float sums[32];
  for (int l = 0; l < 32; ++l) sums[l] = 0.0f;
  for (uint64_t c = 0; c < n32; c += 32)
    for (int l = 0; l < 32; ++l) sums[l] += conv(x[c + l]) * conv(y[c + l]);
  float t = 0.0f;
  for (int l = 0; l < 32; ++l) t += sums[l];
  return s + t;
}
float lo_dot_f16(const uint16_t* x, const uint16_t* y, uint64_t d) {
  return dot_lanes32(x, y, d, half_to_float);
}
float lo_dot_bf16(const uint16_t* x, const uint16_t* y, uint64_t d) {
  return dot_lanes32(x, y, d, bf16_to_float);
}
// u8 dot: exact u32 sum of the products, converted to f32 once (dot.rs:152-161)
float lo_dot_u8(const uint8_t* x, const uint8_t* y, uint64_t d) {
  uint32_t s = 0;
  for (uint64_t i = 0; i < d; ++i) s += uint32_t(x[i]) * uint32_t(y[i]);
  return float(s);
}
// cosine distance, scalar fallback form (cosine.rs:233-238 cosine_scalar with x_norm = norm_l2(x)).
// The reference f32 path uses f32x16 FMA + platform reduce_sum (cosine.rs:143-174) whose summation
// order is ISA-specific: tolerance parity only (the reference itself tests at assert_relative_eq).
float lo_cosine_f32(const float* x, const float* y, uint64_t d) {
  float xn = norm_l2_f32(x, d);
  float y_sq = dot_f32(y, y, d);
  float xy = dot_f32(x, y, d);
  return 1.0f - xy / (xn * std::sqrt(y_sq));
}
void lo_l2_batch_f32(const float* from, const float* to, uint64_t n, uint64_t d, float* out) {
  for (uint64_t i = 0; i < n; ++i) out[i] = l2_f32(from, to + i * d, d);  // l2.rs:194-203
}

// A3. normalize (lance-linalg/src/kernels.rs:141-146): norm = sqrt(sum x^2) sequential in T,
// then x / norm.  Returns the norm.
float lo_normalize_f32(const float* x, uint64_t d, float* out) {
  float s = 0.0f;
  for (uint64_t i = 0; i < d; ++i) s += x[i] * x[i];  // powi(2) == x*x
  float norm = std::sqrt(s);
  for (uint64_t i = 0; i < d; ++i) out[i] = x[i] / norm;
  return norm;
}
void lo_normalize_rows_f32(const float* x, uint64_t n, uint64_t d, float* out, int nthreads) {
  parallel_for(n, nthreads, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; ++i) lo_normalize_f32(x + i * d, d, out + i * d);
  });
}
// KeepFiniteVectors (lance-index/src/vector/transform.rs:112-159): row is kept iff all finite.
void lo_is_finite_rows_f32(const float* x, uint64_t n, uint64_t d, uint8_t* keep) {
  for (uint64_t i = 0; i < n; ++i) {
    bool ok = true;
    for (uint64_t j = 0; j < d; ++j) ok = ok && std::isfinite(x[i * d + j]);
    keep[i] = ok;
  }
}

// ---------------------------------------------------------------------------------------------
// a5/a8  compute_membership_and_dist (kmeans.rs:317-369) / compute_partitions_with_dists (:1275)
//   bias[c] = balance_factor * cluster_sizes[c] as f32 when cluster_sizes != NULL (kmeans.rs:341-345)
// ---------------------------------------------------------------------------------------------
void lo_compute_membership(const float* centroids, uint64_t k, uint64_t d, const float* data,
                           uint64_t n, int metric, float balance_factor,
                           const uint64_t* cluster_sizes, uint32_t* ids, float* dists,
                           uint8_t* valid, int nthreads) {
  std::vector<float> bias;
  if (cluster_sizes) {
    bias.resize(k);
    for (uint64_t c = 0; c < k; ++c) bias[c] = balance_factor * float(cluster_sizes[c]);
  }
  const float* bp = cluster_sizes ? bias.data() : nullptr;
  parallel_for(n, nthreads, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; ++i) {
      uint32_t id;
      float val;
      bool ok = argmin_row(centroids, k, d, data + i * d, metric, bp, &id, &val);
      ids[i] = ok ? id : 0;
      if (dists) dists[i] = ok ? val : std::numeric_limits<float>::quiet_NaN();
      if (valid) valid[i] = ok;
    }
  });
}

// ---------------------------------------------------------------------------------------------
// a6/a7  Lloyd loop (kmeans.rs:610-719), update (:371-446), split_clusters (:174-207),
//        compute_cluster_sizes (:210-232), compute_balance_loss (:234-237)
//   init_centroids == NULL -> choose k distinct rows with OUR rng (partial Fisher-Yates).
//   balance_factor is the value AFTER `params.balance_factor /= n` (kmeans.rs:1344).
// Returns the number of iterations executed.
// ---------------------------------------------------------------------------------------------
int lo_kmeans_train(const float* data_in, uint64_t n_in, uint64_t d, uint64_t k, int max_iters,
                    double tolerance, float balance_factor_param, int metric, uint64_t seed,
                    const float* init_centroids, float* centroids_out, double* loss_out,
                    int nthreads) {
  // kmeans.rs:623-627: keep only the first 512*k rows
  uint64_t n = n_in >= k * 512 ? k * 512 : n_in;
  const float* data = data_in;
  std::vector<float> cent(k * d);
  SplitMix64 rng(seed);
  if (init_centroids) {
    std::memcpy(cent.data(), init_centroids, sizeof(float) * k * d);
  } else {
    std::vector<uint32_t> idx(n);
    for (uint64_t i = 0; i < n; ++i) idx[i] = uint32_t(i);
    for (uint64_t i = 0; i < k; ++i) {
      uint64_t j = i + rng.next() % (n - i);
      std::swap(idx[i], idx[j]);
      std::memcpy(&cent[i * d], data + uint64_t(idx[i]) * d, sizeof(float) * d);
    }
  }
  std::vector<uint64_t> cluster_sizes(k, 0);
  std::vector<uint32_t> ids(n);
  std::vector<float> dists(n);
  std::vector<uint8_t> valid(n);
  float adjusted_balance_factor = std::numeric_limits<float>::max();
  double loss = std::numeric_limits<double>::max();
  double last_loss = loss;
  int it = 0;
  for (it = 1; it <= max_iters; ++it) {
    // f32::min returns the non-NaN operand (kmeans.rs:679)
    float balance_factor = std::fmin(adjusted_balance_factor, balance_factor_param);
    lo_compute_membership(cent.data(), k, d, data, n, metric, balance_factor, cluster_sizes.data(),
                          ids.data(), dists.data(), valid.data(), nthreads);
    // compute_membership_and_loss (kmeans.rs:266-280): radius = max, loss = f64 sum in row order
    std::vector<float> radius(k, 0.0f);
    std::vector<double> losses(k, 0.0);
    for (uint64_t i = 0; i < n; ++i)
      if (valid[i]) {
        radius[ids[i]] = std::max(radius[ids[i]], dists[i]);
        losses[ids[i]] += double(dists[i]);
      }
    // compute_cluster_sizes (kmeans.rs:210-232)
    std::fill(cluster_sizes.begin(), cluster_sizes.end(), 0);
    uint64_t max_id = 0, max_size = 0;
    for (uint64_t i = 0; i < n; ++i)
      if (valid[i]) {
        uint64_t c = ids[i];
        cluster_sizes[c] += 1;
        if (cluster_sizes[c] > max_size) {
          max_size = cluster_sizes[c];
          max_id = c;
        }
      }
    adjusted_balance_factor =
        (radius[max_id] - float(losses[max_id]) / float(cluster_sizes[max_id])) / float(n);
    // compute_balance_loss (kmeans.rs:234-237)
    uint64_t size_sq = 0;
    for (uint64_t c = 0; c < k; ++c) size_sq += cluster_sizes[c] * cluster_sizes[c];
    float balance_loss = balance_factor * (float(size_sq) - float(n * n) / float(k));
    double sum_losses = 0.0;
    for (uint64_t c = 0; c < k; ++c) sum_losses += losses[c];
    last_loss = sum_losses + double(balance_loss);
    // to_kmeans (kmeans.rs:371-446): per-cluster sum in row order IN T, then *= 1/cnt
    //   The reference splits the CENTROIDS into chunks, one rayon task each, and every task walks all rows
    //   and adds the ones that belong to its chunk (kmeans.rs:383-408): per centroid the rows are still
    //   added in row order, so the bits do not depend on the number of tasks.
    std::fill(cent.begin(), cent.end(), 0.0f);
    {
      uint64_t ncpu = nthreads > 2 ? uint64_t(nthreads - 2) : 1;  // get_num_compute_intensive_cpus()
      if (k < ncpu || k < 16) ncpu = 1;
      const uint64_t chunk_size = k / ncpu;
      const uint64_t nchunks = (k + chunk_size - 1) / chunk_size;
      parallel_for(nchunks, nthreads, [&](size_t cb, size_t ce) {
        for (size_t ch = cb; ch < ce; ++ch) {
          const uint64_t start = ch * chunk_size, end = std::min<uint64_t>((ch + 1) * chunk_size, k);
          for (uint64_t i = 0; i < n; ++i) {
            const uint64_t cid = ids[i];
            if (valid[i] && start <= cid && cid < end) {
              float* c = &cent[cid * d];
              const float* v = data + i * d;
              for (uint64_t j = 0; j < d; ++j) c[j] += v[j];
            }
          }
        }
      });
    }
    for (uint64_t c = 0; c < k; ++c)
      if (cluster_sizes[c] > 0) {
        float norm = 1.0f / float(cluster_sizes[c]);
        for (uint64_t j = 0; j < d; ++j) cent[c * d + j] *= norm;
      }
    // split_clusters (kmeans.rs:174-207), our rng
    {
      const float eps = 1.0f / 1024.0f;
      for (uint64_t i = 0; i < k; ++i)
        if (cluster_sizes[i] == 0) {
          uint64_t j = 0;
          for (uint64_t tries = 0;; ++tries) {
            float p = (float(cluster_sizes[j]) - 1.0f) / float(n - k);
            if (rng.next_f32() < p) break;
            j = (j + 1) % k;
            if (tries >= 64 * k) {  // guard (ours): the reference would spin forever when no
              j = 0;                // cluster has more than one row; take the largest instead
              for (uint64_t c = 1; c < k; ++c)
                if (cluster_sizes[c] > cluster_sizes[j]) j = c;
              break;
            }
          }
          cluster_sizes[i] = cluster_sizes[j] / 2;
          cluster_sizes[j] -= cluster_sizes[i];
          for (uint64_t t = 0; t < d; ++t) {
            if (t % 2 == 0) {
              cent[i * d + t] = cent[j * d + t] * (1.0f + eps);
              cent[j * d + t] *= 1.0f - eps;
            } else {
              cent[i * d + t] = cent[j * d + t] * (1.0f - eps);
              cent[j * d + t] *= 1.0f + eps;
            }
          }
        }
    }
    if (std::fabs(loss - last_loss) < tolerance * last_loss) break;  // kmeans.rs:704
    loss = last_loss;
  }
  if (it > max_iters) it = max_iters;
  std::memcpy(centroids_out, cent.data(), sizeof(float) * k * d);
  if (loss_out) *loss_out = last_loss;
  return it;
}

// ---------------------------------------------------------------------------------------------
// A6  hierarchical k-means for k > 256 (kmeans.rs:746-1003).  Heap = Rust BinaryHeap restated,
// ordered by (not finalized, size); the top-level run uses `seed`, the split of cluster id uses seed + 1 + id
// (the reference's RNG is unseeded; a seed tied to the cluster, not to the call order, lets the product train
// independent splits concurrently without changing any result).
// Returns the number of clusters produced (== k unless no cluster can be split further).
// ---------------------------------------------------------------------------------------------
int lo_hierarchical_kmeans(const float* data, uint64_t n, uint64_t d, uint64_t target_k, int max_iters,
                           double tolerance, float balance_factor, int metric, uint64_t hk, uint64_t seed,
                           float* centroids_out, int nthreads) {
  struct Cl {
    uint32_t id;
    std::vector<uint32_t> idx;
    std::vector<float> c;
    bool fin;
  };
  auto le = [](const Cl& a, const Cl& b) {
    if (a.fin != b.fin) return a.fin;
    return a.idx.size() <= b.idx.size();
  };
  std::vector<Cl> heap;
  auto sift_up = [&](size_t start, size_t pos) {
    Cl elt = std::move(heap[pos]);
    while (pos > start) {
      size_t parent = (pos - 1) / 2;
      if (le(elt, heap[parent])) break;
      heap[pos] = std::move(heap[parent]);
      pos = parent;
    }
    heap[pos] = std::move(elt);
  };
  auto push = [&](Cl c) {
    heap.push_back(std::move(c));
    sift_up(0, heap.size() - 1);
  };
  auto pop = [&]() {
    Cl item = std::move(heap.back());
    heap.pop_back();
    if (!heap.empty()) {
      std::swap(item, heap[0]);
      size_t end = heap.size(), pos = 0;
      Cl elt = std::move(heap[0]);
      size_t child = 1;
      while (child + 1 < end) {
        if (le(heap[child], heap[child + 1])) child += 1;
        heap[pos] = std::move(heap[child]);
        pos = child;
        child = 2 * pos + 1;
      }
      if (child + 1 == end) {
        heap[pos] = std::move(heap[child]);
        pos = child;
      }
      heap[pos] = std::move(elt);
      sift_up(0, pos);
    }
    return item;
  };
  const uint64_t k0 = std::min(std::min(hk, target_k), n);
  std::vector<float> top(k0 * d);
  double loss;
  lo_kmeans_train(data, n, d, k0, max_iters, tolerance, balance_factor, metric, seed, nullptr,
                  top.data(), &loss, nthreads);
  std::vector<uint32_t> ids(n);
  std::vector<uint8_t> valid(n);
  lo_compute_membership(top.data(), k0, d, data, n, metric, 0.0f, nullptr, ids.data(), nullptr, valid.data(), nthreads);
  uint32_t next_id = 0;
  for (uint64_t i = 0; i < k0; ++i) {
    Cl c;
    for (uint64_t r = 0; r < n; ++r)
      if (valid[r] && ids[r] == i) c.idx.push_back(uint32_t(r));
    if (c.idx.empty()) continue;
    c.id = next_id++;
    c.c.assign(top.begin() + i * d, top.begin() + (i + 1) * d);
    c.fin = false;
    push(std::move(c));
  }
  std::vector<float> sub, subc(hk * d);
  while (heap.size() < target_k) {
    if (heap.empty()) break;
    Cl big = pop();
    if (big.fin || big.idx.size() <= 1) {
      push(std::move(big));
      break;
    }
    const uint64_t size = big.idx.size(), remaining = target_k - heap.size();
    uint64_t ck;
    if (size <= hk)
      ck = std::min<uint64_t>(std::min<uint64_t>(2, remaining), size);
    else
      ck = std::max<uint64_t>(2, std::min(std::min(size / hk, remaining), hk));
    sub.resize(size * d);
    for (uint64_t r = 0; r < size; ++r) std::memcpy(&sub[r * d], data + uint64_t(big.idx[r]) * d, sizeof(float) * d);
    lo_kmeans_train(sub.data(), size, d, ck, max_iters, tolerance, balance_factor, metric, seed + 1 + big.id, nullptr,
                    subc.data(), &loss, nthreads);
    ids.resize(size);
    valid.resize(size);
    lo_compute_membership(subc.data(), ck, d, sub.data(), size, metric, 0.0f, nullptr, ids.data(), nullptr,
                          valid.data(), nthreads);
    std::vector<std::vector<uint32_t>> ch(ck);
    for (uint64_t r = 0; r < size; ++r)
      if (valid[r]) ch[ids[r]].push_back(big.idx[r]);
    int nonzero = 0;
    for (auto& v : ch) nonzero += !v.empty();
    if (nonzero <= 1) {
      big.fin = true;
      push(std::move(big));
      continue;
    }
    for (uint64_t i = 0; i < ck; ++i) {
      if (ch[i].empty()) continue;
      Cl c;
      c.id = next_id++;
      c.idx = std::move(ch[i]);
      c.c.assign(subc.begin() + i * d, subc.begin() + (i + 1) * d);
      c.fin = false;
      push(std::move(c));
    }
  }
  std::sort(heap.begin(), heap.end(), [](const Cl& a, const Cl& b) { return a.id < b.id; });
  for (size_t i = 0; i < heap.size() && i < target_k; ++i)
    std::memcpy(centroids_out + i * d, heap[i].c.data(), sizeof(float) * d);
  return int(heap.size());
}

// ---------------------------------------------------------------------------------------------
// a12  kmeans_find_partitions (kmeans.rs:1134-1158): all K distances, ascending partial sort.
//   tie order among equal distances: arrow-ord is unpinned -> ascending (dist, id); NaN last.
// ---------------------------------------------------------------------------------------------
void lo_find_partitions(const float* centroids, uint64_t k, uint64_t d, const float* query,
                        uint64_t nprobes, int metric, uint32_t* ids, float* dists) {
  std::vector<float> dv(k);
  for (uint64_t c = 0; c < k; ++c) dv[c] = metric_dist(metric, query, centroids + c * d, d);
  std::vector<uint32_t> order(k);
  for (uint64_t c = 0; c < k; ++c) order[c] = uint32_t(c);
  auto cmp = [&](uint32_t a, uint32_t b) {
    bool an = std::isnan(dv[a]), bn = std::isnan(dv[b]);
    if (an != bn) return bn;
    if (!an && dv[a] != dv[b]) return dv[a] < dv[b];
    return a < b;
  };
  uint64_t p = std::min(nprobes, k);
  std::partial_sort(order.begin(), order.begin() + p, order.end(), cmp);
  for (uint64_t i = 0; i < p; ++i) {
    ids[i] = order[i];
    dists[i] = dv[order[i]];
  }
}

// a9  residual (residual.rs:86-95): r = x - centroid[part] elementwise in T
void lo_compute_residual(const float* centroids, uint64_t d, const float* vectors, uint64_t n,
                         const uint32_t* part_ids, float* out, int nthreads) {
  parallel_for(n, nthreads, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; ++i) {
      const float* c = centroids + uint64_t(part_ids[i]) * d;
      for (uint64_t j = 0; j < d; ++j) out[i * d + j] = vectors[i * d + j] - c[j];
    }
  });
}

// ---------------------------------------------------------------------------------------------
// a11  PQ training (pq/builder.rs:89-157): M independent k-means (k = 2^nbits) on the sub-vector
//   columns (pq/utils.rs:14-49), each through the free fn train_kmeans (kmeans.rs:1309-1347:
//   first sample_rate*k rows, balance 0).  Sub-space m uses seed + m.  init_codebook may be NULL.
//   iters_out[M] (nullable) receives the iteration counts.
// ---------------------------------------------------------------------------------------------
void lo_pq_train(const float* data, uint64_t n, uint64_t d, uint64_t M, int nbits, int max_iters,
                 uint64_t sample_rate, int metric, uint64_t seed, const float* init_codebook,
                 float* codebook_out, int* iters_out, int nthreads) {
  const uint64_t k = uint64_t(1) << nbits;
  const uint64_t ds = d / M;
  uint64_t rows = n > sample_rate * k ? sample_rate * k : n;
  std::vector<float> sub(rows * ds);
  for (uint64_t m = 0; m < M; ++m) {
    for (uint64_t i = 0; i < rows; ++i)
      std::memcpy(&sub[i * ds], data + i * d + m * ds, sizeof(float) * ds);
    double loss;
    int it = lo_kmeans_train(sub.data(), rows, ds, k, max_iters, 1e-4, 0.0f, metric, seed + m,
                             init_codebook ? init_codebook + m * k * ds : nullptr,
                             codebook_out + m * k * ds, &loss, nthreads);
    if (iters_out) iters_out[m] = it;
  }
}

// a10  PQ encode (pq.rs:116-191): per row, per sub-vector argmin over the codebook rows
//   (compute_partition kmeans.rs:1350-1369, no bias), None -> 0; 4-bit packs (v[1]<<4)|v[0].
void lo_pq_encode(const float* codebook, uint64_t M, int nbits, uint64_t d, int metric,
                  const float* vectors, uint64_t n, uint8_t* codes_out, int nthreads) {
  const uint64_t k = uint64_t(1) << nbits;
  const uint64_t ds = d / M;
  const uint64_t bytes_per_row = nbits == 4 ? M / 2 : M;
  parallel_for(n, nthreads, [&](size_t b, size_t e) {
    std::vector<uint8_t> tmp(M);
    for (size_t i = b; i < e; ++i) {
      for (uint64_t m = 0; m < M; ++m) {
        uint32_t id;
        float val;
        bool ok = argmin_row(codebook + m * k * ds, k, ds, vectors + i * d + m * ds, metric,
                             nullptr, &id, &val);
        tmp[m] = ok ? uint8_t(id) : 0;
      }
      if (nbits == 4)
        for (uint64_t j = 0; j < M / 2; ++j)
          codes_out[i * bytes_per_row + j] = uint8_t((tmp[2 * j + 1] << 4) | tmp[2 * j]);
      else
        std::memcpy(codes_out + i * bytes_per_row, tmp.data(), M);
    }
  });
}

// a14  ADC lookup table (pq/distance.rs:24-92): LUT[m*2^nbits + c] = dist(q_m, cb[m][c])
void lo_build_lut(const float* codebook, int nbits, uint64_t M, uint64_t d, int metric,
                  const float* query, float* lut) {
  const uint64_t k = uint64_t(1) << nbits;
  const uint64_t ds = d / M;
  for (uint64_t m = 0; m < M; ++m)
    for (uint64_t c = 0; c < k; ++c)
      lut[m * k + c] = metric_dist(metric, query + m * ds, codebook + (m * k + c) * ds, ds);
}

// a18  transpose [n][M] -> [M][n] (pq/storage.rs:430-450)
void lo_transpose_codes(const uint8_t* codes, uint64_t n, uint64_t M, uint8_t* out) {
  for (uint64_t i = 0; i < n; ++i)
    for (uint64_t m = 0; m < M; ++m) out[m * n + i] = codes[i * M + m];
}

// a15  compute_pq_distance, 8-bit, transposed codes (pq/distance.rs:109-144):
//   dist[j] = 0; for m: dist[j] += LUT[m*256 + codeT[m*n + j]]   (f32 adds in m order)
//   Dot: PQDistCalculator::distance_all subtracts (M-1) afterwards (pq/storage.rs:957-958).
void lo_pq_scan(const float* lut, uint64_t M, const uint8_t* codes_t, uint64_t n, int metric,
                float* dists) {
  for (uint64_t j = 0; j < n; ++j) dists[j] = 0.0f;
  for (uint64_t m = 0; m < M; ++m) {
    const float* t = lut + m * 256;
    const uint8_t* c = codes_t + m * n;
    for (uint64_t j = 0; j < n; ++j) dists[j] += t[c[j]];
  }
  if (metric == 2)
    for (uint64_t j = 0; j < n; ++j) dists[j] -= float(M) - 1.0f;
}

// a19  compute_pq_distance_4bit (pq/distance.rs:147-242) + quantize_distance_table (:284-295) +
//   PQDistCalculator::distance_all's Dot fix-up (pq/storage.rs:957-958).
//   lut: M x 16 f32; codes_t: TRANSPOSED packed codes [M/2][n], low nibble = sub-vector 2i, high nibble =
//   sub-vector 2i+1 (pq.rs:168-173).  The first flat_num = min(max(200, k_hint), n) rows and the last
//   n % 16 rows are exact f32 sums (two adds per byte, byte order); every other row is the SATURATING u8
//   sum (u8x16 `+=` is _mm_adds_epu8, lance-linalg/src/simd/u8.rs:303-321) of the table quantised to
//   u8 with qmin = min(table), qmax = max(first flat_num distances) (total order), dequantised as
//   q * ((qmax - qmin) / 255) + qmin.
void lo_pq_scan_4bit(const float* lut, uint64_t M, const uint8_t* codes_t, uint64_t n, uint64_t k_hint,
                     int metric, float* dists) {
  const uint64_t nb = M / 2;
  for (uint64_t j = 0; j < n; ++j) dists[j] = 0.0f;
  if (n == 0) return;
  auto flat = [&](uint64_t off, uint64_t len) {
    for (uint64_t i = 0; i < nb; ++i) {
      const float* t0 = lut + (2 * i) * 16;
      const float* t1 = lut + (2 * i + 1) * 16;
      const uint8_t* c = codes_t + i * n;
      for (uint64_t j = off; j < off + len; ++j) {
        dists[j] += t0[c[j] & 0xF];
        dists[j] += t1[c[j] >> 4];
      }
    }
  };
  k_hint = std::min<uint64_t>(k_hint, n);
  const uint64_t flat_num = std::min<uint64_t>(std::max<uint64_t>(200, k_hint), n);
  flat(0, flat_num);
  float qmax = dists[0];
  for (uint64_t j = 1; j < flat_num; ++j)  // max_by(total_cmp): the LAST maximum wins, same value either way
    if (total_key(dists[j]) >= total_key(qmax)) qmax = dists[j];
  float qmin = std::numeric_limits<float>::infinity();
  for (uint64_t i = 0; i < M * 16; ++i) qmin = std::fmin(qmin, lut[i]);  // f32::min ignores NaN
  const float factor = 255.0f / (qmax - qmin);
  std::vector<uint8_t> qt(M * 16);
  for (uint64_t i = 0; i < M * 16; ++i) {
    const float v = std::round((lut[i] - qmin) * factor);  // f32::round: half away from zero
    qt[i] = std::isnan(v) ? 0 : v <= 0.0f ? 0 : v >= 255.0f ? 255 : uint8_t(v);  // `as u8` saturates, NaN -> 0
  }
  const uint64_t rem = n % 16;
  std::vector<uint8_t> q(n, 0);
  for (uint64_t i = 0; i < nb; ++i) {
    const uint8_t* t0 = qt.data() + (2 * i) * 16;
    const uint8_t* t1 = qt.data() + (2 * i + 1) * 16;
    const uint8_t* c = codes_t + i * n;
    for (uint64_t j = 0; j < n - rem; ++j) {
      unsigned a = q[j] + t0[c[j] & 0xF];
      a = a > 255 ? 255 : a;
      a += t1[c[j] >> 4];
      q[j] = uint8_t(a > 255 ? 255 : a);
    }
  }
  if (rem > 0) {
    const uint64_t off = std::max(n - rem, flat_num);
    flat(off, n - off);
  }
  const float range = (qmax - qmin) / 255.0f;
  for (uint64_t j = flat_num; j < n - rem; ++j) dists[j] = float(q[j]) * range + qmin;
  if (metric == 2) {
    const float diff = float(M) - 1.0f;
    for (uint64_t j = 0; j < n; ++j) dists[j] = dists[j] - diff;
  }
}

// a19  sum_4bit_dist_table_scalar (lance-linalg/src/simd/dist_table.rs:62-91): u8 table sums over 4-bit
//   codes laid out in PERM0 order, 32 vectors per block, code_len bytes per vector; u16 saturating adds.
//   (The IVF_PQ 4-bit path uses compute_pq_distance_4bit above; this kernel serves the reference's RabitQ
//   storage, bq/storage.rs:333 -- restated because it carries the reference's only 4-bit literal,
//   dist_table.rs:179-217, and its C twin dist_table.c:8 compiles into oracle/_ref.)
void lo_sum_4bit_dist_table(uint64_t n, uint64_t code_len, const uint8_t* codes, const uint8_t* dist_table,
                            uint16_t* dists) {
  static const uint64_t PERM0[16] = {0, 8, 1, 9, 2, 10, 3, 11, 4, 12, 5, 13, 6, 14, 7, 15};
  auto sat = [](uint16_t a, uint16_t b) { uint32_t s = uint32_t(a) + b; return uint16_t(s > 65535 ? 65535 : s); };
  for (uint64_t vb = 0; vb * 32 < n; ++vb) {
    const uint8_t* blocks = codes + vb * 32 * code_len;
    for (uint64_t sv = 0; sv * 32 < 32 * code_len; ++sv) {
      const uint8_t* block = blocks + sv * 32;
      const uint8_t* cur = dist_table + sv * 2 * 16;
      const uint8_t* nxt = dist_table + (sv * 2 + 1) * 16;
      for (uint64_t j = 0; j < 16; ++j) {
        const uint64_t lo_id = vb * 32 + PERM0[j], hi_id = lo_id + 16;
        dists[lo_id] = sat(sat(dists[lo_id], cur[block[j] & 0x0F]), nxt[block[j + 16] & 0x0F]);
        dists[hi_id] = sat(sat(dists[hi_id], cur[block[j] >> 4]), nxt[block[j + 16] >> 4]);
      }
    }
  }
}

// a16  FlatIndex::search fast path (flat/index.rs:97-127): size-k Rust BinaryHeap, push while
//   len<k else replace the root iff root.dist > dist (total_cmp).  Output = heap's internal
//   vector order (`into_iter`), unsorted.  Optional [lower, upper) range (flat/index.rs:101-115).
uint64_t lo_flat_topk(const float* dists, const uint64_t* row_ids, uint64_t n, uint64_t k,
                      int use_range, float lower, float upper, uint64_t* out_ids,
                      float* out_dists) {
  RustMaxHeap h;
  if (k == 0) return 0;
  for (uint64_t j = 0; j < n; ++j) {
    float dist = dists[j];
    if (use_range && (total_key(dist) < total_key(lower) || total_key(dist) >= total_key(upper)))
      continue;
    if (h.data.size() < k) {
      h.push({row_ids ? row_ids[j] : j, dist});
    } else if (gt(h.data[0].dist, dist)) {
      h.pop();
      h.push({row_ids ? row_ids[j] : j, dist});
    }
  }
  for (size_t i = 0; i < h.data.size(); ++i) {
    out_ids[i] = h.data[i].id;
    out_dists[i] = h.data[i].dist;
  }
  return h.data.size();
}

// RowIdMask::selected (lance-core/src/utils/mask.rs:84-93): allow list AND NOT block list; either
// list may be absent (NULL).  Lists are sorted ascending (RoaringTreemap iteration order).
struct RowMask {
  const uint64_t* allow; uint64_t n_allow; int has_allow;
  const uint64_t* block; uint64_t n_block; int has_block;
  bool empty() const { return !has_allow && !has_block; }
  bool selected(uint64_t id) const {
    if (has_allow && !std::binary_search(allow, allow + n_allow, id)) return false;
    if (has_block && std::binary_search(block, block + n_block, id)) return false;
    return true;
  }
};

// a16  FlatIndex::search prefilter path (flat/index.rs:129-165): rows are visited in storage order,
//   unselected rows are skipped BEFORE the distance is looked at, then the same heap rule.
// flat/index.rs:101-102,132-133: lower_bound.unwrap_or(f32::MIN), upper_bound.unwrap_or(f32::MAX)
struct Range {
  int use; float lower, upper;
  bool excludes(float dist) const {
    return use && (total_key(dist) < total_key(lower) || total_key(dist) >= total_key(upper));
  }
};
static Range make_range(int has_lower, float lower, int has_upper, float upper) {
  return Range{has_lower || has_upper, has_lower ? lower : std::numeric_limits<float>::lowest(),
               has_upper ? upper : std::numeric_limits<float>::max()};
}
static uint64_t flat_topk_masked(const float* dists, const uint64_t* row_ids, uint64_t n, uint64_t k,
                                 const RowMask& mask, const Range& range, uint64_t* out_ids, float* out_dists) {
  RustMaxHeap h;
  if (k == 0) return 0;
  for (uint64_t j = 0; j < n; ++j) {
    if (!mask.selected(row_ids[j])) continue;
    float dist = dists[j];
    if (range.excludes(dist)) continue;
    if (h.data.size() < k) {
      h.push({row_ids[j], dist});
    } else if (gt(h.data[0].dist, dist)) {
      h.pop();
      h.push({row_ids[j], dist});
    }
  }
  for (size_t i = 0; i < h.data.size(); ++i) {
    out_ids[i] = h.data[i].id;
    out_dists[i] = h.data[i].dist;
  }
  return h.data.size();
}

// a17  FlatDistanceCal::distance_all (flat/storage.rs:397-403): exact distances to every row
void lo_flat_distance_all(const float* query, const float* vectors, uint64_t n, uint64_t d,
                          int metric, float* out, int nthreads) {
  parallel_for(n, nthreads, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; ++i) {
      const float* v = vectors + i * d;
      out[i] = metric == 1 ? lo_cosine_f32(query, v, d) : metric_dist(metric, query, v, d);
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Query pipeline for one IVF_PQ index held as CSR-by-partition arrays (the same arrays the
// product keeps on the device).  Follows rust/lance/src/index/vector/ivf/v2.rs:455-500:
//   find_partitions -> per probed partition: residual query (v2.rs:316-332), LUT, scan, heap top-k
//   -> global merge sorted by (_distance asc, _rowid asc), first k (scanner.rs:3450-3466).
// codes: row-major [n][M] in partition order (transposed internally per partition as the
// reference storage does).  Parallel over queries (reference: one query at a time, partitions in
// parallel; results are independent of that schedule).
// out arrays are [nq][k]; out_counts[nq].
// ---------------------------------------------------------------------------------------------
static void ivfpq_search_impl(const float* centroids, uint64_t K, uint64_t d, int metric,
                     const float* codebook, uint64_t M, int nbits, const uint64_t* part_offsets,
                     const uint8_t* codes, const uint64_t* row_ids, const float* queries,
                     uint64_t nq, uint64_t k, uint64_t nprobes, const RowMask& mask, const Range& range,
                     uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nthreads) {
  const uint64_t ncode = uint64_t(1) << nbits;
  uint64_t max_part = 0;
  for (uint64_t p = 0; p < K; ++p) max_part = std::max(max_part, part_offsets[p + 1] - part_offsets[p]);
  // transposed copies per partition, built once (ProductQuantizationStorage::new transposes);
  // 4-bit: M/2 packed bytes per row (pq.rs:168-173), transposed byte-wise
  const uint64_t cw = nbits == 4 ? M / 2 : M;
  std::vector<uint8_t> codes_t(part_offsets[K] * cw);
  for (uint64_t p = 0; p < K; ++p) {
    uint64_t n = part_offsets[p + 1] - part_offsets[p];
    lo_transpose_codes(codes + part_offsets[p] * cw, n, cw, codes_t.data() + part_offsets[p] * cw);
  }
  const int cmetric = metric == 1 ? 0 : metric;  // cosine -> L2 on normalised vectors
  parallel_for(nq, nthreads, [&](size_t b, size_t e) {
    std::vector<uint32_t> pids(nprobes);
    std::vector<float> pd(nprobes), q(d), qr(d), lut(M * ncode), dist(max_part);
    std::vector<uint64_t> hid(k);
    std::vector<float> hd(k);
    std::vector<Node> cand;
    for (size_t qi = b; qi < e; ++qi) {
      const float* qin = queries + qi * d;
      if (metric == 1)
        lo_normalize_f32(qin, d, q.data());  // knn.rs:497-499
      else
        std::memcpy(q.data(), qin, sizeof(float) * d);
      uint64_t np = std::min(nprobes, K);
      lo_find_partitions(centroids, K, d, q.data(), np, cmetric, pids.data(), pd.data());
      cand.clear();
      for (uint64_t pi = 0; pi < np; ++pi) {
        uint64_t p = pids[pi];
        uint64_t n = part_offsets[p + 1] - part_offsets[p];
        if (n == 0) continue;
        const float* qq = q.data();
        if (cmetric == 0) {  // residual query for L2/cosine (v2.rs:316-332)
          for (uint64_t j = 0; j < d; ++j) qr[j] = q[j] - centroids[p * d + j];
          qq = qr.data();
        }
        lo_build_lut(codebook, nbits, M, d, cmetric, qq, lut.data());
        if (nbits == 4)  // DistCalculator::distance_all(k_hint = k), flat/index.rs:99 -> pq/distance.rs:147;
                         // with a prefilter the rows are scored one by one with the EXACT
                         // DistCalculator::distance (flat/index.rs:152, pq/storage.rs:895-916): k_hint = n
          lo_pq_scan_4bit(lut.data(), M, codes_t.data() + part_offsets[p] * cw, n, mask.empty() ? k : n, cmetric,
                          dist.data());
        else
          lo_pq_scan(lut.data(), M, codes_t.data() + part_offsets[p] * M, n, cmetric, dist.data());
        uint64_t got = mask.empty()
                           ? lo_flat_topk(dist.data(), row_ids + part_offsets[p], n, k, range.use, range.lower,
                                          range.upper, hid.data(), hd.data())
                           : flat_topk_masked(dist.data(), row_ids + part_offsets[p], n, k, mask, range, hid.data(),
                                              hd.data());
        for (uint64_t i = 0; i < got; ++i) cand.push_back({hid[i], hd[i]});
      }
      std::sort(cand.begin(), cand.end(), [](const Node& a, const Node& c) {
        int32_t ka = total_key(a.dist), kc = total_key(c.dist);
        if (ka != kc) return ka < kc;
        return a.id < c.id;
      });
      uint64_t got = std::min<uint64_t>(k, cand.size());
      for (uint64_t i = 0; i < got; ++i) {
        out_ids[qi * k + i] = cand[i].id;
        out_dists[qi * k + i] = cand[i].dist;
      }
      for (uint64_t i = got; i < k; ++i) {
        out_ids[qi * k + i] = ~uint64_t(0);
        out_dists[qi * k + i] = std::numeric_limits<float>::infinity();
      }
      out_counts[qi] = uint32_t(got);
    }
  });
}

void lo_ivfpq_search(const float* centroids, uint64_t K, uint64_t d, int metric,
                     const float* codebook, uint64_t M, int nbits, const uint64_t* part_offsets,
                     const uint8_t* codes, const uint64_t* row_ids, const float* queries,
                     uint64_t nq, uint64_t k, uint64_t nprobes, uint64_t* out_ids,
                     float* out_dists, uint32_t* out_counts, int nthreads) {
  const RowMask none{nullptr, 0, 0, nullptr, 0, 0};
  ivfpq_search_impl(centroids, K, d, metric, codebook, M, nbits, part_offsets, codes, row_ids, queries, nq, k,
                    nprobes, none, Range{0, 0, 0}, out_ids, out_dists, out_counts, nthreads);
}
// the same with a prefilter (PreFilter::mask -> RowIdMask, lance-index/src/prefilter.rs:27-51)
void lo_ivfpq_search_masked(const float* centroids, uint64_t K, uint64_t d, int metric,
                            const float* codebook, uint64_t M, int nbits, const uint64_t* part_offsets,
                            const uint8_t* codes, const uint64_t* row_ids, const float* queries,
                            uint64_t nq, uint64_t k, uint64_t nprobes, const uint64_t* allow,
                            uint64_t n_allow, int has_allow, const uint64_t* block, uint64_t n_block,
                            int has_block, uint64_t* out_ids, float* out_dists, uint32_t* out_counts,
                            int nthreads) {
  const RowMask mask{allow, n_allow, has_allow, block, n_block, has_block};
  ivfpq_search_impl(centroids, K, d, metric, codebook, M, nbits, part_offsets, codes, row_ids, queries, nq, k,
                    nprobes, mask, Range{0, 0, 0}, out_ids, out_dists, out_counts, nthreads);
}
// ... and with the range branch of FlatIndex::search (flat/index.rs:100-115,131-148)
void lo_ivfpq_search_ex(const float* centroids, uint64_t K, uint64_t d, int metric,
                        const float* codebook, uint64_t M, int nbits, const uint64_t* part_offsets,
                        const uint8_t* codes, const uint64_t* row_ids, const float* queries,
                        uint64_t nq, uint64_t k, uint64_t nprobes, const uint64_t* allow,
                        uint64_t n_allow, int has_allow, const uint64_t* block, uint64_t n_block,
                        int has_block, int has_lower, float lower, int has_upper, float upper,
                        uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nthreads) {
  const RowMask mask{allow, n_allow, has_allow, block, n_block, has_block};
  ivfpq_search_impl(centroids, K, d, metric, codebook, M, nbits, part_offsets, codes, row_ids, queries, nq, k,
                    nprobes, mask, make_range(has_lower, lower, has_upper, upper), out_ids, out_dists, out_counts,
                    nthreads);
}

// IVF_FLAT query (lance-index/src/vector/flat/index.rs:82-177 over FlatFloatStorage,
// flat/storage.rs:345-403): partitions found with L2 on the normalised query for cosine
// (ivf.rs:149-185), every row of the probed partitions scored with the index's metric.
// `vectors` are the STORED vectors (normalised for cosine) in partition order.
static void ivfflat_search_impl(const float* centroids, uint64_t K, uint64_t d, int metric,
                       const uint64_t* part_offsets, const float* vectors, const uint64_t* row_ids,
                       const float* queries, uint64_t nq, uint64_t k, uint64_t nprobes, const RowMask& mask,
                       const Range& range, uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nthreads) {
  uint64_t max_part = 0;
  for (uint64_t p = 0; p < K; ++p) max_part = std::max(max_part, part_offsets[p + 1] - part_offsets[p]);
  const int cmetric = metric == 2 ? 2 : 0;
  parallel_for(nq, nthreads, [&](size_t b, size_t e) {
    std::vector<uint32_t> pids(nprobes);
    std::vector<float> pd(nprobes), q(d), dist(max_part);
    std::vector<uint64_t> hid(k);
    std::vector<float> hd(k);
    std::vector<Node> cand;
    for (size_t qi = b; qi < e; ++qi) {
      const float* qin = queries + qi * d;
      if (metric == 1)
        lo_normalize_f32(qin, d, q.data());
      else
        std::memcpy(q.data(), qin, sizeof(float) * d);
      uint64_t np = std::min(nprobes, K);
      lo_find_partitions(centroids, K, d, q.data(), np, cmetric, pids.data(), pd.data());
      cand.clear();
      for (uint64_t pi = 0; pi < np; ++pi) {
        uint64_t p = pids[pi];
        uint64_t n = part_offsets[p + 1] - part_offsets[p];
        if (n == 0) continue;
        lo_flat_distance_all(q.data(), vectors + part_offsets[p] * d, n, d, metric, dist.data(), 1);
        uint64_t got = mask.empty()
                           ? lo_flat_topk(dist.data(), row_ids + part_offsets[p], n, k, range.use, range.lower,
                                          range.upper, hid.data(), hd.data())
                           : flat_topk_masked(dist.data(), row_ids + part_offsets[p], n, k, mask, range, hid.data(),
                                              hd.data());
        for (uint64_t i = 0; i < got; ++i) cand.push_back({hid[i], hd[i]});
      }
      std::sort(cand.begin(), cand.end(), [](const Node& a, const Node& c) {
        int32_t ka = total_key(a.dist), kc = total_key(c.dist);
        if (ka != kc) return ka < kc;
        return a.id < c.id;
      });
      uint64_t got = std::min<uint64_t>(k, cand.size());
      for (uint64_t i = 0; i < got; ++i) {
        out_ids[qi * k + i] = cand[i].id;
        out_dists[qi * k + i] = cand[i].dist;
      }
      for (uint64_t i = got; i < k; ++i) {
        out_ids[qi * k + i] = ~uint64_t(0);
        out_dists[qi * k + i] = std::numeric_limits<float>::infinity();
      }
      out_counts[qi] = uint32_t(got);
    }
  });
}

void lo_ivfflat_search(const float* centroids, uint64_t K, uint64_t d, int metric,
                       const uint64_t* part_offsets, const float* vectors, const uint64_t* row_ids,
                       const float* queries, uint64_t nq, uint64_t k, uint64_t nprobes,
                       uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nthreads) {
  const RowMask none{nullptr, 0, 0, nullptr, 0, 0};
  ivfflat_search_impl(centroids, K, d, metric, part_offsets, vectors, row_ids, queries, nq, k, nprobes, none,
                      Range{0, 0, 0}, out_ids, out_dists, out_counts, nthreads);
}
void lo_ivfflat_search_masked(const float* centroids, uint64_t K, uint64_t d, int metric,
                              const uint64_t* part_offsets, const float* vectors, const uint64_t* row_ids,
                              const float* queries, uint64_t nq, uint64_t k, uint64_t nprobes,
                              const uint64_t* allow, uint64_t n_allow, int has_allow, const uint64_t* block,
                              uint64_t n_block, int has_block, uint64_t* out_ids, float* out_dists,
                              uint32_t* out_counts, int nthreads) {
  const RowMask mask{allow, n_allow, has_allow, block, n_block, has_block};
  ivfflat_search_impl(centroids, K, d, metric, part_offsets, vectors, row_ids, queries, nq, k, nprobes, mask,
                      Range{0, 0, 0}, out_ids, out_dists, out_counts, nthreads);
}
void lo_ivfflat_search_ex(const float* centroids, uint64_t K, uint64_t d, int metric,
                          const uint64_t* part_offsets, const float* vectors, const uint64_t* row_ids,
                          const float* queries, uint64_t nq, uint64_t k, uint64_t nprobes,
                          const uint64_t* allow, uint64_t n_allow, int has_allow, const uint64_t* block,
                          uint64_t n_block, int has_block, int has_lower, float lower, int has_upper, float upper,
                          uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nthreads) {
  const RowMask mask{allow, n_allow, has_allow, block, n_block, has_block};
  ivfflat_search_impl(centroids, K, d, metric, part_offsets, vectors, row_ids, queries, nq, k, nprobes, mask,
                      make_range(has_lower, lower, has_upper, upper), out_ids, out_dists, out_counts, nthreads);
}

// exact brute-force ground truth (rust/lance/src/index/vector/ivf/v2.rs:959-983 `ground_truth`)
void lo_brute_force_topk(const float* data, uint64_t n, uint64_t d, int metric,
                         const float* queries, uint64_t nq, uint64_t k, uint64_t* out_ids,
                         float* out_dists, int nthreads) {
  parallel_for(nq, nthreads, [&](size_t b, size_t e) {
    std::vector<Node> all(n);
    for (size_t qi = b; qi < e; ++qi) {
      for (uint64_t i = 0; i < n; ++i) {
        const float* v = data + i * d;
        float dd = metric == 1 ? lo_cosine_f32(queries + qi * d, v, d)
                               : metric_dist(metric, queries + qi * d, v, d);
        all[i] = {i, dd};
      }
      uint64_t kk = std::min(k, n);
      std::partial_sort(all.begin(), all.begin() + kk, all.end(), [](const Node& a, const Node& c) {
        if (a.dist != c.dist) return a.dist < c.dist;
        return a.id < c.id;
      });
      for (uint64_t i = 0; i < kk; ++i) {
        out_ids[qi * k + i] = all[i].id;
        out_dists[qi * k + i] = all[i].dist;
      }
    }
  });
}

int lo_hardware_threads() { return int(std::thread::hardware_concurrency()); }

}  // extern "C"
