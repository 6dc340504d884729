// partition_index.cu -- the reference's SimpleIndex: an HNSW graph over the IVF centroids that assigns rows to
// partitions by one graph search each, in place of the exact scan, once the model is large.
//
// Replaces  SimpleIndex::try_new / may_train_index / search   lance-index/src/vector/utils.rs:26-108
//           PartitionTransformer::new / transform's graph arm  lance-index/src/vector/ivf/transform.rs:48-68,112-124
//
// The graph is IVF_HNSW_FLAT's graph of one partition holding the K centroids (hnsw_build_rows: the engine of hnsw.cu
// with FlatDist's f32 distances), built with max_level 7, m 12 and ef_construction 15, the levels drawn with
// hnsw_level_draw(seed, 0, i).  A row is assigned by search_basic with k = 1 and ef = 15 (builder.rs:164-235):
// entry node 0, greedy_search at every level from max_level - 1 down to 0, beam_search at level 0 with no bounds
// (f32::MIN <= dist < f32::MAX, graph.rs:290-291), then the first of into_sorted_vec.
//
// centroid_assign_kernel: one warp per row, persistent over the grid.  The row lives in shared memory; the two
// half-warps compute two neighbour distances at a time with the 16-lane rule of row_distance.cuh (IVF_FLAT's scan
// rule: lb2_compute_partitions' f32 L2 / dot distance, bit for bit).  Lane 0 runs the reference's heap updates in
// its order with topk.cuh's BinaryHeap (the result heap of ef = 15 entries in shared memory, the candidate heap in
// the warp's global scratch, sized K + 1 because it can hold every visited node).  The visited set is a K-bit
// bitset per warp in global memory, set with atomicOr by the lane that holds each neighbour (a list names a node at
// most once); only the words of the nodes a row visited are cleared afterwards (all of them if it visited more
// than VCAP nodes), so a row costs its visits, not K / 32 words.
#include <algorithm>
#include <memory>
#include <mutex>

#include "comm.cuh"
#include "common.cuh"
#include "hnsw.cuh"
#include "partition_index.cuh"
#include "row_distance.cuh"
#include "staging.cuh"
#include "topk.cuh"

struct lb2_partition_index {
  uint32_t k = 0, d = 0;
  int metric = 0;  // METRIC_L2 or METRIC_DOT
  uint64_t seed = 0;
  uint32_t insert_batch = 1;
  lb2::DevBuf<float> centroids;  // [k][d] f32
  std::unique_ptr<lb2::HnswGraph> graph;
  // the assignment's per-warp scratch, kept between calls (zero between them); a call holds `mu` until its stream
  // has finished with it
  mutable std::mutex mu;
  mutable lb2::DevBuf<uint32_t> scratch;
};

namespace lb2 {

namespace {

constexpr int CA_WARPS = 4;            // warps per block
constexpr uint32_t CA_EF = 15;         // SimpleIndex::search's ef (utils.rs:93-108)
constexpr uint32_t CA_VCAP = 512;      // visited nodes a row records for the clear
constexpr uint32_t KEY_INF = 0xff800000u;  // unsigned order key of f32::INFINITY
constexpr uint32_t NONE = 0xffffffffu;
constexpr int PI_MAX_LEVEL = 7, PI_M = 12, PI_EFC = 15;  // HnswBuildParams::default().ef_construction(15).num_edges(12)

__device__ __forceinline__ uint32_t ukey(float f) { return (uint32_t)total_order_key(f) ^ 0x80000000u; }
__device__ __forceinline__ float fkey(uint32_t k) { return key_to_float((int32_t)(k ^ 0x80000000u)); }

struct WarpShared {
  uint32_t bid[32], bk[32];            // a list's unvisited nodes (at most 2m = 24) and their keys
  uint32_t rk[CA_EF + 1], rid[CA_EF + 1];  // the result heap
  uint32_t vl[CA_VCAP];                // the nodes the row visited, for the clear
  uint32_t cur, key, go;
};

// keys[j] = the order key of the distance of q (shared memory) to centroid ids[j], j < n: half-warp h takes
// j = h, h + 2, ..; ids must be visible to every lane
template <int METRIC>
__device__ __forceinline__ void keys_of(const float* q, const float* __restrict__ cent, int d, const uint32_t* ids,
                                        uint32_t n, uint32_t* keys) {
  const int lane = threadIdx.x & 31, h = lane >> 4;
  const unsigned mask = h ? 0xffff0000u : 0x0000ffffu;
  for (uint32_t j = h; j < n; j += 2) {
    const float f = flat_row_distance<METRIC>(q, cent + (uint64_t)ids[j] * d, d, lane & 15, mask, 0.0f);
    if ((lane & 15) == 0) keys[j] = ukey(f);
  }
  __syncwarp();
}

// SimpleIndex::search of rows x [n][d] (f32) over the graph g of the K centroids.  A row with a non-finite element
// never reaches the transformer (KeepFiniteVectors, ivf.rs:149-166) and a row whose search keeps no result (every
// distance it meets outside [f32::MIN, f32::MAX)) has no answer: both are part 0, dist NaN, valid 0, as the exact
// scan writes its None rows.  scratch: per warp `words` u32, the bitset zero on entry and on return.
template <int METRIC>
__global__ void __launch_bounds__(CA_WARPS * 32, 4)
centroid_assign_kernel(GraphDev g, const float* __restrict__ cent, uint32_t K, int d, const float* __restrict__ x,
                       uint64_t n, uint32_t* __restrict__ part, float* __restrict__ dist, uint8_t* __restrict__ valid,
                       uint32_t* __restrict__ scratch, uint64_t words, int32_t lo, int32_t hi) {
  extern __shared__ float sh_rows[];
  __shared__ WarpShared sh_w[CA_WARPS];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpShared& S = sh_w[w];
  float* q = sh_rows + (size_t)w * ((d + 3) & ~3);
  const uint64_t gw = (uint64_t)blockIdx.x * CA_WARPS + w, nw = (uint64_t)gridDim.x * CA_WARPS;
  const uint32_t vwords = (K + 31) / 32;
  uint32_t* vis = scratch + gw * words;
  uint32_t* ck = vis + vwords;
  uint32_t* cid = ck + K + 1;
  const unsigned hmask = lane >> 4 ? 0xffff0000u : 0x0000ffffu;
  auto in_range = [&](uint32_t key) {
    const int32_t sk = (int32_t)(key ^ 0x80000000u);
    return sk >= lo && sk < hi;
  };
  for (uint64_t r = gw; r < n; r += nw) {
    bool fin = true;
    const float* xr = x + r * d;
    for (int e = lane; e < d; e += 32) {
      const float v = xr[e];
      q[e] = v;
      fin = fin && isfinite(v);
    }
    fin = __all_sync(0xffffffffu, fin);
    __syncwarp();
    if (!fin) {
      if (lane == 0) {
        part[r] = 0;
        if (dist) dist[r] = __int_as_float(0x7fc00000);
        if (valid) valid[r] = 0;
      }
      continue;
    }
    // search_inner (builder.rs:164-201): node 0, then greedy_search (graph.rs:375-409) at every level down to 0
    uint32_t cur = 0, ckey = ukey(flat_row_distance<METRIC>(q, cent, d, lane & 15, hmask, 0.0f));
    for (int level = g.max_level - 1; level >= 0; --level) {
      for (;;) {
        const ListRef L = list_of(g, cur, level);
        const uint32_t c = *L.cnt;
        keys_of<METRIC>(q, cent, d, L.ids, c, S.bk);
        if (lane == 0) {
          uint32_t next = NONE;
          float cf = fkey(ckey);
          for (uint32_t j = 0; j < c; ++j) {
            const float f = fkey(S.bk[j]);
            if (f < cf) {
              cf = f;
              ckey = S.bk[j];
              next = L.ids[j];
            }
          }
          if (next != NONE) cur = next;
          S.cur = cur;
          S.key = ckey;
          S.go = next != NONE;
        }
        __syncwarp();
        cur = S.cur;
        ckey = S.key;
        const bool go = S.go;
        __syncwarp();
        if (!go) break;
      }
    }
    // beam_search (graph.rs:275-355) at level 0 from (cur, ckey) with ef = 15 and no bounds or bitset
    uint32_t clen = 0, rlen = 0, furthest = 0, vcount = 1;
    if (lane == 0) {
      atomicOr(vis + (cur >> 5), 1u << (cur & 31));
      S.vl[0] = cur;
      rheap_push(ck, cid, clen, ~ckey, cur);
      if (in_range(ckey)) rheap_push(S.rk, S.rid, rlen, ckey, cur);
    }
    for (;;) {
      if (lane == 0) {
        uint32_t go = 0, node = 0;
        if (clen > 0) {
          const uint32_t cur_key = ~ck[0];
          node = cid[0];
          rheap_pop(ck, cid, clen);
          furthest = rlen ? S.rk[0] : KEY_INF;
          go = !(cur_key > furthest && rlen == CA_EF);
        }
        S.go = go;
        S.cur = node;
      }
      __syncwarp();
      const bool go = S.go;
      const uint32_t node = S.cur;
      __syncwarp();
      if (!go) break;
      // the unvisited neighbours in list order, each marked visited (the list names a node at most once)
      const ListRef L = list_of(g, node, 0);
      const uint32_t c = *L.cnt;
      uint32_t id = 0;
      bool fresh = false;
      if ((uint32_t)lane < c) {
        id = L.ids[lane];
        const uint32_t bit = 1u << (id & 31);
        fresh = (atomicOr(vis + (id >> 5), bit) & bit) == 0;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, fresh);
      if (fresh) {
        const uint32_t pos = __popc(bal & ((1u << lane) - 1u));
        S.bid[pos] = id;
        if (vcount + pos < CA_VCAP) S.vl[vcount + pos] = id;
      }
      const uint32_t nn = __popc(bal);
      vcount += nn;
      __syncwarp();
      keys_of<METRIC>(q, cent, d, S.bid, nn, S.bk);
      if (lane == 0) {
        for (uint32_t j = 0; j < nn; ++j) {
          const uint32_t key = S.bk[j], nid = S.bid[j];
          if (key <= furthest || rlen < CA_EF) {
            if (in_range(key)) {
              if (rlen < CA_EF) {
                rheap_push(S.rk, S.rid, rlen, key, nid);
              } else if (key < S.rk[0]) {
                rheap_pop(S.rk, S.rid, rlen);
                rheap_push(S.rk, S.rid, rlen, key, nid);
              }
            }
            rheap_push(ck, cid, clen, ~key, nid);
          }
        }
      }
      __syncwarp();
    }
    if (lane == 0) {  // the first of into_sorted_vec
      rheap_into_sorted(S.rk, S.rid, rlen);
      const bool ok = rlen > 0;
      part[r] = ok ? S.rid[0] : 0u;
      if (dist) dist[r] = ok ? fkey(S.rk[0]) : __int_as_float(0x7fc00000);
      if (valid) valid[r] = ok ? 1 : 0;
    }
    if (vcount <= CA_VCAP) {
      for (uint32_t j = lane; j < vcount; j += 32) vis[S.vl[j] >> 5] = 0;
    } else {
      for (uint32_t j = lane; j < vwords; j += 32) vis[j] = 0;
    }
    __syncwarp();
  }
}

// may_train_index (utils.rs:67-91): EXACT never uses the graph, AUTO when the centroid values number at least 10^6,
// HNSW always; only an f32 model has one (u8 columns have f32 models), so f16 / bf16 models are always exact
bool resolve_graph(uint64_t k, uint32_t d, lb2_dtype dtype, uint32_t mode) {
  LB2_REQUIRE(dtype == LB2_F32 || dtype == LB2_F16 || dtype == LB2_BF16 || dtype == LB2_U8, "unknown dtype %d",
              (int)dtype);
  bool graph;
  switch (mode) {
    case LB2_PARTITION_INDEX_EXACT: graph = false; break;
    case LB2_PARTITION_INDEX_AUTO: graph = k * (uint64_t)d >= 1000000ull; break;
    case LB2_PARTITION_INDEX_HNSW: graph = true; break;
    default: fail(LB2_INVALID_ARG, "unknown partition index mode %u", mode);
  }
  return graph && model_dtype(dtype) == LB2_F32;
}

int pi_metric(lb2_metric metric) {
  const int m = metric_of(metric);
  if (m == METRIC_COSINE) fail(LB2_INVALID_ARG, "partition index: normalise and use L2 for cosine");
  return m;
}

}  // namespace

// the rows x [n][d] (f32 on the device) through pi's graph; scratch grows to the launch's need and stays zeroed
static void centroid_assign(const lb2_partition_index& pi, const float* x, uint64_t n, uint32_t* part, float* dist,
                            uint8_t* valid, DevBuf<uint32_t>& scratch) {
  if (n == 0) return;
  const uint32_t K = pi.k;
  const int d = (int)pi.d;
  const uint64_t words = (uint64_t)(K + 31) / 32 + 2 * ((uint64_t)K + 1);
  const size_t smem = (size_t)CA_WARPS * ((d + 3) & ~3) * sizeof(float);
  auto kern = pi.metric == METRIC_DOT ? centroid_assign_kernel<METRIC_DOT> : centroid_assign_kernel<METRIC_L2>;
  LB2_REQUIRE(smem_with_static(kern, smem) <= ctx().smem_optin, "partition index: d = %d does not fit shared memory", d);
  set_smem(kern, smem_with_static(kern, smem));
  int occ = 0;
  LB2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, CA_WARPS * 32, smem));
  // as many warps as fill the GPU, as rows need, and as a quarter of the free device memory (at most 1 GB) holds
  size_t free_b = 0, total_b = 0;
  LB2_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const uint64_t cap = std::max<uint64_t>(std::min<uint64_t>(1ull << 30, free_b / 4), words * 4 * CA_WARPS);
  const uint64_t fit = std::max<uint64_t>(1, cap / (words * 4 * CA_WARPS));
  const uint64_t grid = std::min<uint64_t>({(uint64_t)std::max(occ, 1) * ctx().num_sms, cdiv(n, CA_WARPS), fit});
  if (scratch.n < grid * CA_WARPS * words) {
    scratch.alloc(grid * CA_WARPS * words);
    scratch.zero();
  }
  const int32_t lo = host_total_key(-3.40282347e+38f), hi = host_total_key(3.40282347e+38f);  // f32::MIN, f32::MAX
  LB2_LAUNCH("centroid_assign", kern, (unsigned)grid, CA_WARPS * 32, smem, dev_view(*pi.graph), pi.centroids.p, K, d,
             x, n, part, dist, valid, scratch.p, words, lo, hi);
}

void PartitionIndexDeleter::operator()(lb2_partition_index* p) const { delete p; }

bool partition_index_uses_graph(uint64_t k, uint32_t d, lb2_dtype dtype, uint32_t mode) {
  return resolve_graph(k, d, dtype, mode);
}

PartitionIndexPtr partition_index_make(const float* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, int metric,
                                       uint32_t mode, uint64_t seed, uint32_t insert_batch) {
  LB2_REQUIRE(k >= 1 && d >= 1, "partition index: needs k >= 1 centroids of d >= 1 elements");
  LB2_REQUIRE(insert_batch <= 65536, "partition index: insert_batch %u is above 65536", insert_batch);
  LB2_REQUIRE(metric == METRIC_L2 || metric == METRIC_DOT, "partition index: the graph's metric is L2 or dot");
  if (!resolve_graph(k, d, dtype, mode)) return nullptr;  // the exact scan: no index (may_train_index's None)
  if (comm_nranks() > 1) fail(LB2_UNSUPPORTED, "partition index: a graph under more than one rank is not implemented");
  if (d % 4 != 0) fail(LB2_UNSUPPORTED, "partition index: the graph needs a dimension that is a multiple of 4, d = %u", d);
  PartitionIndexPtr pi(new lb2_partition_index());
  pi->k = k;
  pi->d = d;
  pi->metric = metric;
  pi->seed = seed;
  pi->insert_batch = std::max<uint32_t>(insert_batch, 1);
  pi->centroids.alloc((size_t)k * d);
  d2d(pi->centroids.p, centroids, (size_t)k * d);
  pi->graph.reset(new HnswGraph());
  HnswGraph& g = *pi->graph;
  g.kind = "partition index";
  g.max_level = PI_MAX_LEVEL;
  g.m = PI_M;
  g.ef_construction = PI_EFC;
  g.insert_batch = pi->insert_batch;
  {
    TagScope tg("partition_index_build");
    hnsw_build_rows(g, pi->centroids.p, k, (int)d, metric, seed);
  }
  sync_stream();
  return pi;
}

void partition_index_assign(const lb2_partition_index& pi, const float* x, uint64_t n, uint32_t* part, float* dist,
                            uint8_t* valid) {
  std::lock_guard<std::mutex> lk(pi.mu);
  centroid_assign(pi, x, n, part, dist, valid, pi.scratch);
  sync_stream();  // the scratch is free for the next call
}

}  // namespace lb2

using namespace lb2;

extern "C" {

lb2_status lb2_partition_index_uses_graph(uint64_t k, uint32_t d, lb2_dtype dtype, lb2_partition_index_mode mode,
                                          int* uses_graph_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(uses_graph_out, "null argument");
  *uses_graph_out = resolve_graph(k, d, dtype, (uint32_t)mode) ? 1 : 0;
  LB2_API_END
}

lb2_status lb2_partition_index_build(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                     lb2_partition_index_mode mode, uint64_t seed, uint32_t insert_batch,
                                     lb2_partition_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out, "null argument");
  *out = nullptr;
  LB2_REQUIRE(centroids && k >= 1 && d >= 1, "partition index: needs k >= 1 centroids of d >= 1 elements");
  const int m = pi_metric(metric);
  if (!resolve_graph(k, d, dtype, (uint32_t)mode)) return LB2_OK;  // the exact scan: no index (may_train_index's None)
  VecIn c(centroids, (size_t)k * d, LB2_F32);
  *out = partition_index_make(c.get(), k, d, dtype, m, (uint32_t)mode, seed, insert_batch).release();
  LB2_API_END
}

lb2_status lb2_partition_index_assign(const lb2_partition_index* pi, const void* centroids, uint32_t k, uint32_t d,
                                      lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n,
                                      uint32_t* part_out, float* dist_out, uint8_t* valid_out) {
  if (!pi) return lb2_compute_partitions(centroids, k, d, dtype, metric, vectors, n, part_out, dist_out, valid_out);
  LB2_API_BEGIN
  LB2_REQUIRE(k == pi->k && d == pi->d, "partition index: built over %u x %u centroids, called with %u x %u", pi->k,
              pi->d, k, d);
  LB2_REQUIRE(pi_metric(metric) == pi->metric, "partition index: called with another metric than it was built with");
  LB2_REQUIRE(model_dtype(dtype) == LB2_F32, "partition index: the graph takes f32 or u8 rows, not dtype %d", (int)dtype);
  OutArg<uint32_t> p(part_out, n);
  OutArg<float> dd(dist_out, n);
  OutArg<uint8_t> v(valid_out, n);
  if (n) {
    LB2_REQUIRE(vectors && part_out, "null argument");
    TagScope tg("partition_index_assign");
    Source src(vectors, n, (int)d, dtype);
    src.start_resident_copy();
    std::lock_guard<std::mutex> lk(pi->mu);
    for_each_chunk(src, [&](const float* xf, const void*, uint64_t r0, uint64_t rows) {
      centroid_assign(*pi, xf, rows, p.get() + r0, dd.get() ? dd.get() + r0 : nullptr, v.get() ? v.get() + r0 : nullptr,
                      pi->scratch);
    });
    sync_stream();  // the scratch is free for the next call
  }
  p.commit(); dd.commit(); v.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_partition_index_info(const lb2_partition_index* pi, uint32_t* k, uint32_t* d, uint32_t* max_level,
                                    uint32_t* m, uint32_t* ef_construction, uint64_t* num_upper_rows) {
  LB2_API_BEGIN
  LB2_REQUIRE(pi, "null argument");
  if (k) *k = pi->k;
  if (d) *d = pi->d;
  if (max_level) *max_level = (uint32_t)pi->graph->max_level;
  if (m) *m = (uint32_t)pi->graph->m;
  if (ef_construction) *ef_construction = (uint32_t)pi->graph->ef_construction;
  if (num_upper_rows) *num_upper_rows = pi->graph->n_up;
  LB2_API_END
}

lb2_status lb2_partition_index_export(const lb2_partition_index* pi, uint8_t* levels_out, uint32_t* counts0_out,
                                      uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                      uint32_t* neighbors_up_out, float* dists_up_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(pi, "null argument");
  const HnswGraph& g = *pi->graph;
  const size_t n = pi->k, nu = g.n_up, m = (size_t)g.m;
  cudaStream_t st = ctx().stream;
  auto out = [&](void* dst, const void* src, size_t bytes) {
    if (dst && bytes) LB2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, st));
  };
  out(levels_out, g.nlev.p, n);
  out(counts0_out, g.cnt0.p, 4 * n);
  out(neighbors0_out, g.nbr0.p, 4 * n * 2 * m);
  out(dists0_out, g.dst0.p, 4 * n * 2 * m);
  out(counts_up_out, g.cntu.p, 4 * nu);
  out(neighbors_up_out, g.nbru.p, 4 * nu * m);
  out(dists_up_out, g.dstu.p, 4 * nu * m);
  sync_stream();
  LB2_API_END
}

lb2_status lb2_partition_index_destroy(lb2_partition_index* pi) {
  LB2_API_BEGIN
  delete pi;
  LB2_API_END
}

}  // extern "C"
