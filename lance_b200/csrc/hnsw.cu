// hnsw.cu -- IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT: an HNSW graph per partition over the partition's SQ codes, PQ
// codes or raw vectors, built and searched on the device (lance-index/src/vector/hnsw/builder.rs, graph.rs, hnsw.rs,
// graph/builder.rs).
//
// Replaces  HNSW::index_vectors / HnswBuilder::insert      hnsw/builder.rs:386-507,742-775
//           select_neighbors_heuristic                   hnsw.rs:60-88
//           beam_search / greedy_search                  graph.rs:275-409
//           HNSW::search / search_inner / flat_search    hnsw/builder.rs:164-280,678-739
//
// The engine is generic over a distance policy (SqDist, PqDist, FlatDist below; with_policy picks an index's), as the
// reference is over VectorStore: `key` is the distance of the query (or of the inserting node) to a node, `between` the heuristic's
// dist_between.
//  * SQ: both are the SQ row rule of sq.cuh (sq/storage.rs:387-444, storage.rs:102-105): an integer sum times one
//    constant, so the build is deterministic and bit-exact.
//  * PQ (pq/storage.rs:675-919): `key` sums a lookup table over the node's codes; the table is the residual query's
//    at search time and, while a node is inserted, the table of the node's own decoded codes (dist_calculator_from_id);
//    `between` is the full-width distance of the two decoded rows (dist_between).
//  * FLAT (flat/storage.rs:345-410): all three are the IVF_FLAT scan's rule on the stored rows, cosine included.
//
// One warp owns one partition (serial build), one inserting node or one back-linked list (batched build, in rounds;
// see the round kernels) or one (query, partition) slot (search).  Its heaps, visited bitset and (PQ) table live in a
// per-warp global scratch sized by the largest partition, so no partition is refused for its size.
// Lane 0 runs the reference's serial heap and list updates in the reference's order; the 32 lanes compute the
// distances of a neighbour list or of a candidate's accepted neighbours, one row per lane, and build a PQ table
// together.  Control decisions reach the other lanes through shared memory after a __syncwarp.
#include <algorithm>
#include <cstdlib>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "exact.cuh"
#include "hnsw.cuh"
#include "index.cuh"
#include "ivf_search.cuh"
#include "pq_lut.cuh"
#include "probe.cuh"
#include "row_distance.cuh"
#include "sq.cuh"
#include "topk.cuh"

namespace lb2 {

namespace {

constexpr uint32_t KEY_INF = 0xff800000u;  // unsigned order key of f32::INFINITY
constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ uint32_t ukey_of(float f) { return (uint32_t)total_order_key(f) ^ 0x80000000u; }
__device__ __forceinline__ float float_of(uint32_t uk) { return key_to_float((int32_t)(uk ^ 0x80000000u)); }

// per-warp scratch (u32 words): PQ table tab[TW] (PQ only) and query / row qv[QW] (PQ and flat), vis[words(nmax)],
// candidate heap ck / cid [nmax + 1], result heap rk / rid [E + 1], batch bid / bk [B], list lid / lk / ord [LB],
// accepted aid / ak [B].  With a table or a query buffer the warp's share is a multiple of 4 words, so tab and qv
// stay 16-byte aligned (TW and QW are multiples of 4).
struct Scratch {
  float *tab, *qv;
  uint32_t *vis, *ck, *cid, *rk, *rid, *bid, *bk, *lid, *lk, *ord, *aid, *ak;
};
__host__ __device__ inline size_t scratch_words(uint64_t nmax, uint32_t E, uint32_t B, uint32_t LB, uint32_t TW = 0,
                                                uint32_t QW = 0) {
  const size_t w = (size_t)TW + QW + (nmax + 31) / 32 + 2 * (nmax + 1) + 2 * ((size_t)E + 1) + 4 * (size_t)B +
                   3 * (size_t)LB;
  return TW || QW ? (w + 3) & ~(size_t)3 : w;
}
__device__ inline Scratch scratch_at(uint32_t* base, uint64_t nmax, uint32_t E, uint32_t B, uint32_t LB,
                                     uint32_t TW = 0, uint32_t QW = 0) {
  Scratch s;
  s.tab = reinterpret_cast<float*>(base);
  s.qv = s.tab + TW;
  s.vis = base + TW + QW;
  s.ck = s.vis + (nmax + 31) / 32;
  s.cid = s.ck + nmax + 1;
  s.rk = s.cid + nmax + 1;
  s.rid = s.rk + E + 1;
  s.bid = s.rid + E + 1;
  s.bk = s.bid + B;
  s.aid = s.bk + B;
  s.ak = s.aid + B;
  s.lid = s.ak + B;
  s.lk = s.lid + LB;
  s.ord = s.lk + LB;
  return s;
}

template <int METRIC>
__device__ __forceinline__ uint32_t pair_key(const uint8_t* a, const uint8_t* b, int d, float r2) {
  const uint32_t* x = reinterpret_cast<const uint32_t*>(a);
  const uint32_t* y = reinterpret_cast<const uint32_t*>(b);
  uint32_t acc = 0;
  for (int w = 0; w < (d >> 2); ++w) acc = sq_word<METRIC>(__ldg(x + w), __ldg(y + w), acc);
  return ukey_of(sq_distance<METRIC>(acc, r2));
}

// The distance policies.  A policy is bound to one partition (storage positions off .. off + n - 1) and provides
//   node_ctx(i, s):       the context of inserting node i (all lanes call it; it may fill the warp's scratch)
//   query_ctx(qi, p, s):  the context of query qi of the slab in probed partition p (all lanes)
//   key(ctx, node):       the order key of the context's distance to a node (one lane)
//   between(u, v):        the order key of dist_between(u, v), the heuristic's distance (one lane)

// IVF_HNSW_SQ: every distance is the SQ row rule over d code bytes (sq/storage.rs:387-444, storage.rs:102-105)
template <int METRIC>
struct SqDist {
  const uint8_t* base;    // the index's code rows [n][d]
  const uint8_t* qcodes;  // the slab's query codes [qn][d] (search)
  int d;
  float r2;
  const uint8_t* codes;  // the partition's first code row
  uint64_t off;          // its first storage position
  uint32_t n;
  using Ctx = const uint8_t*;
  static constexpr bool TABLE = false, QUERY = false;  // no table or query rows in the scratch
  __device__ __forceinline__ void bind(uint64_t o, uint32_t cnt) {
    off = o;
    n = cnt;
    codes = base + o * d;
  }
  void at_slab(uint64_t q0) { qcodes += q0 * d; }  // a search's queries from query q0 on
  __device__ __forceinline__ Ctx node_ctx(uint32_t i, const Scratch&) const { return codes + (uint64_t)i * d; }
  __device__ __forceinline__ Ctx query_ctx(uint64_t qi, uint32_t, const Scratch&) const { return qcodes + qi * d; }
  __device__ __forceinline__ uint32_t key(Ctx q, uint32_t node) const {
    return pair_key<METRIC>(q, codes + (uint64_t)node * d, d, r2);
  }
  __device__ __forceinline__ uint32_t between(uint32_t u, uint32_t v) const {
    return pair_key<METRIC>(codes + (uint64_t)u * d, codes + (uint64_t)v * d, d, r2);
  }
};

// IVF_HNSW_PQ over ProductQuantizationStorage (pq/storage.rs:600-1037); METRIC is L2 (also for cosine: the storage
// carries L2, pq/storage.rs:465-468) or dot.
//  * key: PQDistCalculator::distance (:891-919) on a table of M x 2^NBITS f32 entries in the warp's scratch: 8-bit the
//    m-ascending sum (pq8_row_distance), 4-bit the byte-ordered sum of pair sums; dot subtracts M - 1.  The search
//    table is the IVF_PQ scan's (the residual query under L2, the raw query under dot, ivf/v2.rs:316-332); the
//    build table is the node's own decoded codes' (dist_calculator_from_id, :675-749), both from build_lut.
//  * between: dist_between (:751-841): distance_type.func() over the two decoded full-width rows, with the element
//    type's lane rule of row_distance.cuh (RULE: 16 lanes, or 32 lanes for 16-bit dot).
template <int METRIC, int NBITS, int RULE>
struct PqDist {
  const uint8_t* base;       // the index's code rows [n][cw]
  const float* codebook;     // [M][2^NBITS][ds]
  const float* queries;      // the slab's queries [qn][d] (search; normalised under cosine)
  const float* centroids;    // [K][d]
  int d, M, ds, cw;
  const uint8_t* codes;
  uint64_t off;
  uint32_t n;
  using Ctx = const float*;  // the table
  static constexpr bool TABLE = true, QUERY = true;
  __device__ __forceinline__ void bind(uint64_t o, uint32_t cnt) {
    off = o;
    n = cnt;
    codes = base + o * cw;
  }
  void at_slab(uint64_t q0) { queries += q0 * d; }
  // element e of a row's decoded vector (get_centroids / get_centroids_4bit: the codewords concatenated)
  __device__ __forceinline__ float elem(const uint8_t* row, int e) const {
    const int m = e / ds, t = e - m * ds;
    const uint32_t c = NBITS == 8 ? __ldg(row + m) : (__ldg(row + (m >> 1)) >> ((m & 1) * 4)) & 0xF;
    return __ldg(codebook + ((size_t)m * (1 << NBITS) + c) * ds + t);
  }
  __device__ __forceinline__ Ctx table_of_qv(const Scratch& s) const {
    __syncwarp();
    build_lut<METRIC, NBITS, 32>(s.tab, s.qv, codebook, M, ds, threadIdx.x & 31);
    __syncwarp();
    return s.tab;
  }
  __device__ __forceinline__ Ctx node_ctx(uint32_t i, const Scratch& s) const {
    const uint8_t* row = codes + (uint64_t)i * cw;
    for (int e = threadIdx.x & 31; e < d; e += 32) s.qv[e] = elem(row, e);
    return table_of_qv(s);
  }
  __device__ __forceinline__ Ctx query_ctx(uint64_t qi, uint32_t p, const Scratch& s) const {
    const float* q = queries + qi * d;
    for (int t = threadIdx.x & 31; t < d; t += 32)
      s.qv[t] = METRIC == METRIC_DOT ? q[t] : __fsub_rn(q[t], centroids[(size_t)p * d + t]);
    return table_of_qv(s);
  }
  __device__ __forceinline__ uint32_t key(Ctx lut, uint32_t node) const {
    const uint8_t* row = codes + (uint64_t)node * cw;
    float dist = NBITS == 8 ? pq8_row_distance(lut, row, M) : pq4_pair_distance(lut, row, cw);
    // storage.rs:917-918; a NaN passes through, as on x86 (pq_scan.cu does the same)
    if (METRIC == METRIC_DOT && dist == dist) dist = __fsub_rn(dist, (float)M - 1.0f);
    return ukey_of(dist);
  }
  __device__ __forceinline__ uint32_t between(uint32_t u, uint32_t v) const {
    const uint8_t* ru = codes + (uint64_t)u * cw;
    const uint8_t* rv = codes + (uint64_t)v * cw;
    LaneAcc<RULE, METRIC> acc[16];  // the 16 lanes of the rule, walked one after the other; lane 0 takes the tail
#pragma unroll
    for (int l = 0; l < 16; ++l)
      rule_walk<RULE>(d, l, [&](int e, auto part) {
        constexpr int PART = decltype(part)::value;
        if (PART != 2 || l == 0) acc[l].template step<PART>(elem(ru, e), elem(rv, e));
      });
    return ukey_of(fold_partials<RULE, METRIC>([&](int i) { return acc[i].a; }, [&](int i) { return acc[i].b; },
                                               [](int) { return 0u; }, acc[0].s, 0.0f));
  }
};

// IVF_HNSW_FLAT's row access: 4 elements from a multiple of 4 as f32.  An IVF_FLAT row holds d % 4 == 0 elements, so
// they are one aligned 16-byte (f32) or 8-byte (16-bit) load; a 16-bit row that starts on 16 bytes reads 8 at a time.
struct ScratchRow {  // the query or inserting row in the warp's scratch: written by the warp, so not read through __ldg
  const float* p;
  __device__ __forceinline__ void get4(int e, float* o) const {
    const float4 v = *reinterpret_cast<const float4*>(p + e);
    o[0] = v.x, o[1] = v.y, o[2] = v.z, o[3] = v.w;
  }
  __device__ __forceinline__ void get16(int e, float* o) const {
#pragma unroll
    for (int t = 0; t < 16; t += 4) get4(e + t, o + t);
  }
};
__device__ __forceinline__ void unpack2(uint32_t w, const __half*, float* o) {
  o[0] = __half2float(__ushort_as_half((unsigned short)(w & 0xffffu)));
  o[1] = __half2float(__ushort_as_half((unsigned short)(w >> 16)));
}
__device__ __forceinline__ void unpack2(uint32_t w, const __nv_bfloat16*, float* o) {
  o[0] = __uint_as_float(w << 16);
  o[1] = __uint_as_float(w & 0xffff0000u);
}
template <class T>
struct StoredRow {  // a stored f16 / bf16 row
  const T* p;
  bool a16;  // the row starts on 16 bytes
  __device__ __forceinline__ static StoredRow at(const T* r) {
    return {r, (reinterpret_cast<uintptr_t>(r) & 15) == 0};
  }
  __device__ __forceinline__ void get4(int e, float* o) const {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(p + e));
    unpack2(w.x, p, o);
    unpack2(w.y, p, o + 2);
  }
  __device__ __forceinline__ void get16(int e, float* o) const {
    if (a16) {
#pragma unroll
      for (int t = 0; t < 16; t += 8) {
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(p + e + t));
        unpack2(w.x, p, o + t);
        unpack2(w.y, p, o + t + 2);
        unpack2(w.z, p, o + t + 4);
        unpack2(w.w, p, o + t + 6);
      }
    } else {
#pragma unroll
      for (int t = 0; t < 16; t += 4) get4(e + t, o + t);
    }
  }
};
template <>
struct StoredRow<float> {
  const float* p;
  __device__ __forceinline__ static StoredRow at(const float* r) { return {r}; }
  __device__ __forceinline__ void get4(int e, float* o) const {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p + e));
    o[0] = v.x, o[1] = v.y, o[2] = v.z, o[3] = v.w;
  }
  __device__ __forceinline__ void get16(int e, float* o) const {
#pragma unroll
    for (int t = 0; t < 16; t += 4) get4(e + t, o + t);
  }
};

// The IVF_FLAT scan's rule (scan_rule<METRIC>) of one (query role q, row v) pair on one lane.  The lane walks both rows
// once, 16 elements at a time, into the rule's 16 LaneAccs in registers: element e goes to accumulator e % 16, as
// lane e % 16 of a half-warp takes it in row_distance, and the 16-lane rule's d % 16 tail goes to the sequential sum,
// so every accumulator sees its elements in the rule's order.  QNORM: q's norm is accumulated in the same walk
// (norm_l2's 16 FMA lanes, xor tree, sqrt, as ivfflat_scan_kernel computes the query's); otherwise q_norm is used.
template <int METRIC, bool QNORM, class QR, class VR>
__device__ __forceinline__ float lane_pair_distance(const QR& q, const VR& v, int d, float q_norm) {
  constexpr int RULE = scan_rule<METRIC>();
  LaneAcc<RULE, METRIC> acc[16];
  float qq[16];
#pragma unroll
  for (int l = 0; l < 16; ++l) qq[l] = 0.0f;
  const int n16 = d & ~15;
  for (int c = 0; c < n16; c += 16) {
    float a[16], b[16];
    q.get16(c, a);
    v.get16(c, b);
#pragma unroll
    for (int l = 0; l < 16; ++l) {
      acc[l].template step<0>(a[l], b[l]);
      if (QNORM) qq[l] = fmaf(a[l], a[l], qq[l]);
    }
  }
#pragma unroll
  for (int g = 0; g < 3; ++g) {  // the d % 16 rest, 4 elements at a time
    const int e = n16 + 4 * g;
    if (e < d) {
      float a[4], b[4];
      q.get4(e, a);
      v.get4(e, b);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if constexpr (RULE == RULE_COSINE) {
          acc[4 * g + t].template step<0>(a[t], b[t]);
          if (QNORM) qq[4 * g + t] = fmaf(a[t], a[t], qq[4 * g + t]);
        } else {
          acc[0].template step<2>(a[t], b[t]);
        }
      }
    }
  }
  if (RULE == RULE_COSINE && QNORM) q_norm = sqrtf(tree16([&](int i) { return qq[i]; }));
  return fold_partials<RULE, METRIC>([&](int i) { return acc[i].a; }, [&](int i) { return acc[i].b; },
                                     [](int) { return 0u; }, acc[0].s, q_norm);
}

// IVF_HNSW_FLAT over FlatFloatStorage (flat/storage.rs:31-185,345-410): the stored rows as they are (normalised under
// cosine by the IVF transformer), and every distance FlatDistanceCal's distance_type.func() with the index's own
// type, cosine included (storage.rs:108-158, flat/storage.rs:353-366).  Each is the IVF_FLAT scan's rule for the
// column type, on one lane, so a list distance is bit-identical to the distance IVF_FLAT's scan gives the pair:
//  * key: the context (the query, or the inserting node's row, as f32 in qv, with its norm) to a node
//    (dist_calculator / dist_calculator_from_id);
//  * between: dist_between(u, v) with u in the query role (hnsw.rs:82, storage.rs:102-105): cosine rounds the two
//    norms separately, so the orientation matters.
template <int METRIC, class T>
struct FlatDist {
  const T* base;          // the index's vectors [n][d]
  const float* queries;   // the slab's queries [qn][d] (search; normalised under cosine)
  int d;
  const T* rows;          // the partition's first row
  uint64_t off;
  uint32_t n;
  struct Ctx {
    const float* q;  // the row in qv
    float norm;      // its norm (cosine)
  };
  static constexpr bool TABLE = false, QUERY = true;
  __device__ __forceinline__ void bind(uint64_t o, uint32_t cnt) {
    off = o;
    n = cnt;
    rows = base + o * d;
  }
  void at_slab(uint64_t q0) { queries += q0 * d; }
  __device__ __forceinline__ StoredRow<T> row(uint32_t i) const { return StoredRow<T>::at(rows + (uint64_t)i * d); }
  // the norm of the row in qv with ivfflat_scan_kernel's 16 FMA lanes, xor tree and sqrt (norm_l2.rs:106-130)
  __device__ __forceinline__ Ctx ctx_of_qv(const Scratch& s) const {
    __syncwarp();
    float nrm = 0.0f;
    if (METRIC == METRIC_COSINE) {
      float a = 0.0f;
      for (int e = threadIdx.x & 15; e < d; e += 16) a = fmaf(s.qv[e], s.qv[e], a);
#pragma unroll
      for (int o = 8; o >= 1; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o, 16);
      nrm = sqrtf(a);
    }
    return {s.qv, nrm};
  }
  __device__ __forceinline__ Ctx node_ctx(uint32_t i, const Scratch& s) const {
    const T* r = rows + (uint64_t)i * d;
    for (int e = threadIdx.x & 31; e < d; e += 32) s.qv[e] = ldf<T>(r, e);
    return ctx_of_qv(s);
  }
  __device__ __forceinline__ Ctx query_ctx(uint64_t qi, uint32_t, const Scratch& s) const {
    const float* q = queries + qi * d;
    for (int e = threadIdx.x & 31; e < d; e += 32) s.qv[e] = q[e];
    return ctx_of_qv(s);
  }
  __device__ __forceinline__ uint32_t key(const Ctx& c, uint32_t node) const {
    return ukey_of(lane_pair_distance<METRIC, false>(ScratchRow{c.q}, row(node), d, c.norm));
  }
  __device__ __forceinline__ uint32_t between(uint32_t u, uint32_t v) const {
    return ukey_of(lane_pair_distance<METRIC, true>(row(u), row(v), d, 0.0f));
  }
};

// keys[j] = key(q, node ids[j]) for j < n, one node per lane; the ids must be visible to every lane
template <class Dist>
__device__ __forceinline__ void warp_keys(const Dist& P, typename Dist::Ctx q, const uint32_t* ids, uint32_t n,
                                          uint32_t* keys) {
  for (uint32_t j = threadIdx.x & 31; j < n; j += 32) keys[j] = P.key(q, ids[j]);
  __syncwarp();
}

__device__ __forceinline__ bool allowed(const uint64_t* allow, uint64_t pos) {
  return allow == nullptr || ((allow[pos >> 6] >> (pos & 63)) & 1ull) != 0;
}

// greedy_search (graph.rs:375-409): neighbours in list order, strictly closer (f32 `<`) moves on
template <class Dist>
__device__ void greedy(const GraphDev& g, const Dist& P, typename Dist::Ctx q, int level, uint32_t& cur, uint32_t& ckey,
                       const Scratch& s) {
  __shared__ uint32_t sh_cur, sh_key, sh_go;
  const int lane = threadIdx.x & 31;
  for (;;) {
    const ListRef L = list_of(g, P.off + cur, level);
    const uint32_t n = *L.cnt;
    warp_keys(P, q, L.ids, n, s.bk);
    if (lane == 0) {
      uint32_t next = NONE;
      float cf = float_of(ckey);
      for (uint32_t j = 0; j < n; ++j) {
        const float f = float_of(s.bk[j]);
        if (f < cf) {
          cf = f;
          ckey = s.bk[j];
          next = L.ids[j];
        }
      }
      if (next != NONE) cur = next;
      sh_cur = cur;
      sh_key = ckey;
      sh_go = next != NONE;
    }
    __syncwarp();
    cur = sh_cur;
    ckey = sh_key;
    const bool go = sh_go;
    __syncwarp();
    if (!go) return;
  }
}

// beam_search (graph.rs:275-355) at `level` from (ep, ep_key) with `ef`; the bitmap (bits at off + node, nullable)
// and the range [lo, hi) (signed total-order keys) filter the results, not the traversal.  `furthest` is read once
// per expanded node.  Returns the number of results, left ascending (into_sorted_vec) at rk / rid.
template <class Dist>
__device__ uint32_t beam_search(const GraphDev& g, const Dist& P, typename Dist::Ctx q, int level, uint32_t ep,
                                uint32_t ep_key, uint32_t ef, const uint64_t* allow, int32_t lo, int32_t hi,
                                const Scratch& s) {
  __shared__ uint32_t sh_go, sh_n;
  const int lane = threadIdx.x & 31;
  for (uint32_t w = lane; w < (P.n + 31) / 32; w += 32) s.vis[w] = 0;
  __syncwarp();
  auto in_range = [&](uint32_t key) {
    const int32_t sk = (int32_t)(key ^ 0x80000000u);
    return sk >= lo && sk < hi;
  };
  uint32_t clen = 0, rlen = 0, furthest = 0;
  if (lane == 0) {
    s.vis[ep >> 5] |= 1u << (ep & 31);
    rheap_push(s.ck, s.cid, clen, ~ep_key, ep);
    if (allowed(allow, P.off + ep) && in_range(ep_key)) rheap_push(s.rk, s.rid, rlen, ep_key, ep);
  }
  for (;;) {
    if (lane == 0) {
      uint32_t go = 0, n = 0;
      if (clen > 0) {
        const uint32_t cur_key = ~s.ck[0], cur = s.cid[0];
        rheap_pop(s.ck, s.cid, clen);
        furthest = rlen ? s.rk[0] : KEY_INF;
        if (!(cur_key > furthest && rlen == ef)) {
          go = 1;
          const ListRef L = list_of(g, P.off + cur, level);
          const uint32_t c = *L.cnt;
          for (uint32_t j = 0; j < c; ++j) {
            const uint32_t id = L.ids[j];
            const uint32_t bit = 1u << (id & 31);
            if (s.vis[id >> 5] & bit) continue;
            s.vis[id >> 5] |= bit;
            s.bid[n++] = id;
          }
        }
      }
      sh_go = go;
      sh_n = n;
    }
    __syncwarp();
    const bool go = sh_go;
    const uint32_t n = sh_n;
    if (!go) break;
    warp_keys(P, q, s.bid, n, s.bk);
    if (lane == 0) {
      for (uint32_t j = 0; j < n; ++j) {
        const uint32_t key = s.bk[j], id = s.bid[j];
        if (key <= furthest || rlen < ef) {
          if (allowed(allow, P.off + id) && in_range(key)) {
            if (rlen < ef) {
              rheap_push(s.rk, s.rid, rlen, key, id);
            } else if (key < s.rk[0]) {
              rheap_pop(s.rk, s.rid, rlen);
              rheap_push(s.rk, s.rid, rlen, key, id);
            }
          }
          rheap_push(s.ck, s.cid, clen, ~key, id);
        }
      }
    }
    __syncwarp();
  }
  if (lane == 0) {
    rheap_into_sorted(s.rk, s.rid, rlen);
    sh_n = rlen;
  }
  __syncwarp();
  const uint32_t r = sh_n;
  __syncwarp();
  return r;
}

// HnswBuilder::prune (builder.rs:491-507) of a ranked list (ids / keys, c entries in push order) into dst: up to
// m_max entries stay in push order, a longer list goes through select_neighbors_heuristic (hnsw.rs:60-88) with a
// STABLE sort by distance in f32::total_cmp order (OrderedFloat's partial_cmp, graph.rs:68-82; the reference's
// sort_unstable_by leaves tied candidates in an unspecified order).
template <class Dist>
__device__ void prune_into(const Dist& P, const uint32_t* ids, const uint32_t* keys, uint32_t c, uint32_t m_max,
                           const ListRef& dst, const Scratch& s) {
  __shared__ uint32_t sh_na;
  const int lane = threadIdx.x & 31;
  if (c <= m_max) {
    if (lane == 0) {
      for (uint32_t j = 0; j < c; ++j) {
        dst.ids[j] = ids[j];
        dst.dist[j] = float_of(keys[j]);
      }
      *dst.cnt = c;
    }
    __syncwarp();
    return;
  }
  if (lane == 0) {  // insertion sort of positions by order key, ties keep their order
    for (uint32_t j = 0; j < c; ++j) {
      const uint32_t key = keys[j];
      uint32_t t = j;
      while (t > 0 && keys[s.ord[t - 1]] > key) {
        s.ord[t] = s.ord[t - 1];
        --t;
      }
      s.ord[t] = j;
    }
    sh_na = 0;
  }
  __syncwarp();
  uint32_t na = 0;
  for (uint32_t t = 0; t < c && na < m_max; ++t) {
    const uint32_t u = s.ord[t], uid = ids[u], ukey = keys[u];
    bool ok = true;
    for (uint32_t j = lane; j < na; j += 32) ok = ok && ukey < P.between(uid, s.aid[j]);
    ok = __all_sync(0xffffffffu, ok);
    if (ok) {
      if (lane == 0) {
        s.aid[na] = uid;
        s.ak[na] = ukey;
      }
      ++na;
    }
    __syncwarp();
  }
  if (lane == 0) {
    const uint32_t old = *dst.cnt;  // a back-link prune can shorten the list: the slots it drops go back to zero
    for (uint32_t j = 0; j < na; ++j) {
      dst.ids[j] = s.aid[j];
      dst.dist[j] = float_of(s.ak[j]);
    }
    for (uint32_t j = na; j < old; ++j) {
      dst.ids[j] = 0;
      dst.dist[j] = 0.0f;
    }
    *dst.cnt = na;
  }
  __syncwarp();
}

// the search half of HnswBuilder::insert (builder.rs:396-463) of node i: the descent, a beam search per level of the
// node from its target level down, and the node's own lists, the pruned results.  Reads the lists the searches reach,
// writes only node i's.
template <class Dist>
__device__ void insert_search(const GraphDev& g, const Dist& P, uint32_t i, uint32_t efc, int32_t lo, int32_t hi,
                              const Scratch& s) {
  const typename Dist::Ctx q = P.node_ctx(i, s);  // dist_calculator_from_id(node)
  const int target = (int)g.nlev[P.off + i] - 1;
  uint32_t ep = 0, ekey = P.key(q, 0);
  for (int level = g.max_level - 1; level > target; --level) greedy(g, P, q, level, ep, ekey, s);
  for (int level = target; level >= 0; --level) {
    const uint32_t R = beam_search(g, P, q, level, ep, ekey, efc, nullptr, lo, hi, s);
    ep = s.rid[0];
    ekey = s.rk[0];
    const uint32_t m_max = level == 0 ? 2 * g.m : g.m;
    prune_into(P, s.rid, s.rk, R, m_max, list_of(g, P.off + i, level), s);
  }
}

// one back-link of insert (builder.rs:446-460): node i, at order key `ekey` in its own list, enters `other` when it is
// closer than the LAST entry of a full list (GraphBuilderNode::cutoff, graph/builder.rs:50-57), then `other` is pruned
template <class Dist>
__device__ void back_link(const Dist& P, const ListRef& other, uint32_t i, uint32_t ekey, uint32_t m_max,
                          const Scratch& s) {
  __shared__ uint32_t sh_go, sh_n;
  if ((threadIdx.x & 31) == 0) {
    const uint32_t c2 = *other.cnt;
    const uint32_t cutoff = c2 < m_max ? KEY_INF : ukey_of(other.dist[c2 - 1]);  // the LAST entry
    const bool add = ekey < cutoff;
    if (add) {
      for (uint32_t j = 0; j < c2; ++j) {
        s.lid[j] = other.ids[j];
        s.lk[j] = ukey_of(other.dist[j]);
      }
      s.lid[c2] = i;
      s.lk[c2] = ekey;
    }
    sh_go = add;
    sh_n = c2 + 1;
  }
  __syncwarp();
  const bool add = sh_go;
  const uint32_t c = sh_n;
  __syncwarp();
  if (add) prune_into(P, s.lid, s.lk, c, m_max, other, s);
}

// HNSW::index_vectors of partitions order[0 ..), taken largest first by a persistent grid of one-warp CTAs, each
// inserting its partition's nodes 1 .. n_p - 1 one after the other (insert_batch 1)
template <class Dist>
__global__ void __launch_bounds__(32)
hnsw_build_kernel(GraphDev g, const uint64_t* __restrict__ part_offsets, const uint32_t* __restrict__ order, int nparts,
                  uint32_t* __restrict__ next, const Dist proto, uint32_t efc, int32_t lo, int32_t hi,
                  uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B, uint32_t LB, uint32_t TW,
                  uint32_t QW) {
  __shared__ uint32_t sh_part;
  const int lane = threadIdx.x & 31;
  if (!Dist::TABLE) TW = 0;
  if (!Dist::QUERY) QW = 0;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, LB, TW, QW), nmax, E, B, LB, TW, QW);
  for (;;) {
    if (lane == 0) sh_part = atomicAdd(next, 1u);
    __syncwarp();
    const uint32_t t = sh_part;
    __syncwarp();
    if (t >= (uint32_t)nparts) return;
    const uint32_t p = order[t];
    Dist P = proto;
    P.bind(part_offsets[p], (uint32_t)(part_offsets[p + 1] - part_offsets[p]));
    for (uint32_t i = 1; i < P.n; ++i) {  // HnswBuilder::insert (builder.rs:396-463)
      insert_search(g, P, i, efc, lo, hi, s);
      const int target = (int)g.nlev[P.off + i] - 1;
      for (int level = 0; level <= target; ++level) {  // the back-links, level by level, in pruned-list order
        const uint32_t m_max = level == 0 ? 2 * g.m : g.m;
        const ListRef mine = list_of(g, P.off + i, level);
        const uint32_t cm = *mine.cnt;
        for (uint32_t e = 0; e < cm; ++e)
          back_link(P, list_of(g, P.off + mine.ids[e], level), i, ukey_of(mine.dist[e]), m_max, s);
      }
    }
  }
}

// ---- the batched build (insert_batch B >= 2): rounds of concurrent inserts --------------------------------------
// A round inserts nodes s0 .. s0 + W - 1 of every partition order[0 .. nparts) (each clipped to its rows), item t
// being node s0 + t % W of partition order[t / W].  Phase 1 (hnsw_round_search_kernel) runs every item's
// insert_search over the graph as the round found it: no list names a node of the round yet, so it reads lists of
// nodes < s0 only and writes only the round's own lists.  Phase 2 applies the back-links as if the round's nodes
// had linked back one after the other in ascending order: a list (j, level) receives at most one entry per node, and
// lists are independent, so each target list takes its entries in ascending node order, distinct lists in parallel.
// hnsw_round_link_kernel chains every back-link onto its target list (head[list] -> rec_next ...) and names each
// target list once in `touched`; hnsw_round_apply_kernel gives each touched list to one warp, which orders the
// chain by node and applies back_link entry by entry.

struct RoundBufs {
  uint32_t* counters;  // [0] the next phase-1 item, [1] records, [2] touched lists
  uint32_t* head;      // [n + n_up] the last record of each list's chain, NONE when empty
  uint32_t *rec_i, *rec_key, *rec_next;
  uint32_t* touched;   // [3][..]: partition, node, level of each touched list
};

// the list number of (global row, level): level 0 by row, the upper levels after every level-0 list
__device__ __forceinline__ uint64_t list_number(const GraphDev& g, uint64_t n, uint64_t row, int level) {
  return level == 0 ? row : n + g.up_base[row] + (level - 1);
}

template <class Dist>
__global__ void __launch_bounds__(32)
hnsw_round_search_kernel(GraphDev g, const uint64_t* __restrict__ part_offsets, const uint32_t* __restrict__ order,
                         uint32_t nparts, uint32_t s0, uint32_t W, RoundBufs rb, const Dist proto, uint32_t efc,
                         int32_t lo, int32_t hi, uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B,
                         uint32_t LB, uint32_t TW, uint32_t QW) {
  __shared__ uint32_t sh_t;
  const int lane = threadIdx.x & 31;
  if (!Dist::TABLE) TW = 0;
  if (!Dist::QUERY) QW = 0;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, LB, TW, QW), nmax, E, B, LB, TW, QW);
  const uint32_t items = nparts * W;
  for (;;) {
    if (lane == 0) sh_t = atomicAdd(rb.counters, 1u);
    __syncwarp();
    const uint32_t t = sh_t;
    __syncwarp();
    if (t >= items) return;
    const uint32_t p = order[t / W], i = s0 + t % W;
    Dist P = proto;
    P.bind(part_offsets[p], (uint32_t)(part_offsets[p + 1] - part_offsets[p]));
    if (i < P.n) insert_search(g, P, i, efc, lo, hi, s);
  }
}

// one thread per item: every entry of the item's lists becomes a record on its target list's chain
__global__ void hnsw_round_link_kernel(GraphDev g, uint64_t n, const uint64_t* __restrict__ part_offsets,
                                       const uint32_t* __restrict__ order, uint32_t nparts, uint32_t s0, uint32_t W,
                                       RoundBufs rb) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)nparts * W) return;
  const uint32_t p = order[t / W], i = s0 + (uint32_t)(t % W);
  const uint64_t off = part_offsets[p];
  if (i >= part_offsets[p + 1] - off) return;
  const int target = (int)g.nlev[off + i] - 1;
  for (int level = 0; level <= target; ++level) {
    const ListRef mine = list_of(g, off + i, level);
    const uint32_t cm = *mine.cnt;
    for (uint32_t e = 0; e < cm; ++e) {
      const uint32_t eid = mine.ids[e];
      const uint32_t r = atomicAdd(rb.counters + 1, 1u);
      rb.rec_i[r] = i;
      rb.rec_key[r] = ukey_of(mine.dist[e]);
      const uint32_t prev = atomicExch(rb.head + list_number(g, n, off + eid, level), r);
      rb.rec_next[r] = prev;
      if (prev == NONE) {  // the first record of this list: name the list once
        const uint32_t u = atomicAdd(rb.counters + 2, 1u);
        rb.touched[3 * (uint64_t)u] = p;
        rb.touched[3 * (uint64_t)u + 1] = eid;
        rb.touched[3 * (uint64_t)u + 2] = (uint32_t)level;
      }
    }
  }
}

// one warp per touched list: its chain ordered by node (each node appears once), then back_link in that order; the
// list's chain head goes back to NONE for the next round
template <class Dist>
__global__ void __launch_bounds__(32)
hnsw_round_apply_kernel(GraphDev g, uint64_t n, const uint64_t* __restrict__ part_offsets, RoundBufs rb,
                        const Dist proto, uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B,
                        uint32_t LB, uint32_t TW, uint32_t QW) {
  __shared__ uint32_t sh_c;
  const int lane = threadIdx.x & 31;
  if (!Dist::TABLE) TW = 0;
  if (!Dist::QUERY) QW = 0;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, LB, TW, QW), nmax, E, B, LB, TW, QW);
  const uint32_t nt = rb.counters[2];
  for (uint32_t u = blockIdx.x; u < nt; u += gridDim.x) {
    const uint32_t p = rb.touched[3 * (uint64_t)u], j = rb.touched[3 * (uint64_t)u + 1];
    const int level = (int)rb.touched[3 * (uint64_t)u + 2];
    Dist P = proto;
    P.bind(part_offsets[p], (uint32_t)(part_offsets[p + 1] - part_offsets[p]));
    const uint64_t ln = list_number(g, n, P.off + j, level);
    if (lane == 0) {  // the chain, at most one record per node of the round (< n_p <= nmax), into ck
      uint32_t c = 0;
      for (uint32_t r = rb.head[ln]; r != NONE; r = rb.rec_next[r]) s.ck[c++] = r;
      rb.head[ln] = NONE;
      sh_c = c;
    }
    __syncwarp();
    const uint32_t c = sh_c;
    __syncwarp();
    for (uint32_t a = lane; a < c; a += 32) {  // rank by node: the nodes are distinct, so the ranks are a permutation
      const uint32_t ra = s.ck[a], ia = rb.rec_i[ra];
      uint32_t rank = 0;
      for (uint32_t b = 0; b < c; ++b) rank += rb.rec_i[s.ck[b]] < ia;
      s.cid[rank] = ra;
    }
    __syncwarp();
    const ListRef other = list_of(g, P.off + j, level);
    const uint32_t m_max = level == 0 ? 2 * g.m : g.m;
    for (uint32_t k = 0; k < c; ++k) {
      const uint32_t r = s.cid[k];
      back_link(P, other, rb.rec_i[r], rb.rec_key[r], m_max, s);
    }
  }
}

// HNSW::search of every slot: partition id >= K or an empty partition -> no rows; the prefilter's flat branch when
// fewer than 10 % of the partition's rows are allowed (builder.rs:715-725), search_inner otherwise
template <class Dist>
__global__ void __launch_bounds__(32)
hnsw_search_kernel(GraphDev g, uint64_t nslots, int np, const uint32_t* __restrict__ probe_ids,
                   const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ acnt, const Dist proto,
                   const uint64_t* __restrict__ row_ids, uint32_t ef0, int kc, ScanFilter flt0,
                   float* __restrict__ cand_d, uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt,
                   uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B, uint32_t TW, uint32_t QW,
                   const QueryParam* __restrict__ qp) {
  __shared__ uint32_t sh_n;
  const int lane = threadIdx.x & 31;
  if (!Dist::TABLE) TW = 0;
  if (!Dist::QUERY) QW = 0;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, 0, TW, QW), nmax, E, B, 0, TW, QW);
  for (uint64_t slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
    const uint64_t qi = slot / np;
    const uint32_t p = probe_ids[slot];
    // the query's own k', ef, filter and allowed-row counts with per-query values (kc is then the lists' stride)
    const int kq = qp ? qp[qi].k : kc;
    const uint32_t ef = qp ? qp[qi].ef : ef0;
    const ScanFilter flt = qp ? qp[qi].flt : flt0;
    const uint32_t* __restrict__ ac = qp ? qp[qi].acnt : acnt;
    Dist P = proto;
    P.bind(offsets[p], (uint32_t)(offsets[p + 1] - offsets[p]));
    if (P.n == 0) {  // an empty partition returns no rows (builder.rs:695-697)
      if (lane == 0) cand_cnt[slot] = 0;
      continue;
    }
    const typename Dist::Ctx q = P.query_ctx(qi, p, s);  // dist_calculator(query)
    uint32_t R;
    if (flt.allow && ac[p] < (uint32_t)((uint64_t)P.n * 10 / 100)) {
      // HNSW::flat_search (builder.rs:238-280): allowed rows in node order, kept when lower < d <= upper.  Lane 0 drives
      // the reference's heap over the partition's rows, 32 distances at a time; this branch only runs when fewer than
      // 10 % of the rows are allowed.
      uint32_t len = 0;
      for (uint32_t c0 = 0; c0 < P.n; c0 += 32) {
        const uint32_t j = c0 + lane;
        if (j < P.n && allowed(flt.allow, P.off + j)) s.bk[lane] = P.key(q, j);
        __syncwarp();
        if (lane == 0) {
          for (uint32_t t = 0; t < 32 && c0 + t < P.n; ++t) {
            if (!allowed(flt.allow, P.off + c0 + t)) continue;
            const uint32_t key = s.bk[t];
            const int32_t sk = (int32_t)(key ^ 0x80000000u);
            if (sk <= flt.lo_key || sk > flt.hi_key) continue;
            if (len < (uint32_t)kq) {
              rheap_push(s.rk, s.rid, len, key, c0 + t);
            } else if (key < s.rk[0]) {
              rheap_pop(s.rk, s.rid, len);
              rheap_push(s.rk, s.rid, len, key, c0 + t);
            }
          }
        }
        __syncwarp();
      }
      if (lane == 0) {
        rheap_into_sorted(s.rk, s.rid, len);
        sh_n = len;
      }
      __syncwarp();
      R = sh_n;
      __syncwarp();
    } else {  // search_inner (builder.rs:164-201): greedy descent to level 0 inclusive, then the beam search
      uint32_t ep = 0, ekey = P.key(q, 0);
      for (int level = g.max_level - 1; level >= 0; --level) greedy(g, P, q, level, ep, ekey, s);
      R = beam_search(g, P, q, 0, ep, ekey, ef, flt.allow, flt.lo_key, flt.hi_key, s);
      R = min(R, (uint32_t)kq);
    }
    for (uint32_t j = lane; j < R; j += 32) {
      cand_d[slot * kc + j] = float_of(s.rk[j]);
      cand_id[slot * kc + j] = row_ids[P.off + s.rid[j]];
    }
    if (lane == 0) cand_cnt[slot] = R;
    __syncwarp();
  }
}

int32_t key_of_host(float f) { return host_total_key(f); }

}  // namespace

void hnsw_level_thresholds(int m, int max_level, uint64_t* thr) {
  const uint64_t two32 = 1ull << 32;
  uint64_t pw = 1;  // m^l, saturated above 2^32
  for (int l = 0; l < max_level; ++l) {
    thr[l] = two32 / pw;
    pw = pw > two32 ? pw : pw * (uint64_t)m;
  }
}

// One kept partition of a rebuilt graph: its level-0 block (rows, 2m per row) and its upper block (rows, m per row),
// each contiguous in both layouts because nodes are in storage order and upper rows are compact.
struct SpliceSpan {
  uint64_t old_row, new_row, rows, old_up, new_up, up_rows;
};

// copies every kept partition's blocks from the old graph to their new offsets (blockIdx.x = the partition, the
// y blocks and the threads stride over its words); neighbour ids are partition-local, so nothing is rewritten
__global__ void hnsw_splice_kernel(const SpliceSpan* __restrict__ spans, int m, const uint32_t* __restrict__ cnt0,
                                   const uint32_t* __restrict__ nbr0, const float* __restrict__ dst0,
                                   const uint32_t* __restrict__ cntu, const uint32_t* __restrict__ nbru,
                                   const float* __restrict__ dstu, uint32_t* __restrict__ ocnt0,
                                   uint32_t* __restrict__ onbr0, float* __restrict__ odst0, uint32_t* __restrict__ ocntu,
                                   uint32_t* __restrict__ onbru, float* __restrict__ odstu) {
  const SpliceSpan sp = spans[blockIdx.x];
  const uint64_t t0 = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x, st = (uint64_t)gridDim.y * blockDim.x;
  const uint64_t w0 = sp.rows * 2 * (uint64_t)m, wu = sp.up_rows * (uint64_t)m;
  for (uint64_t i = t0; i < sp.rows; i += st) ocnt0[sp.new_row + i] = cnt0[sp.old_row + i];
  for (uint64_t i = t0; i < w0; i += st) {
    onbr0[sp.new_row * 2 * m + i] = nbr0[sp.old_row * 2 * m + i];
    odst0[sp.new_row * 2 * m + i] = dst0[sp.old_row * 2 * m + i];
  }
  for (uint64_t i = t0; i < sp.up_rows; i += st) ocntu[sp.new_up + i] = cntu[sp.old_up + i];
  for (uint64_t i = t0; i < wu; i += st) {
    onbru[sp.new_up * m + i] = nbru[sp.old_up * m + i];
    odstu[sp.new_up * m + i] = dstu[sp.old_up * m + i];
  }
}

// the buffers of the layout for n rows, n_up upper rows and a largest partition of nmax rows (each at least 1 entry)
static void alloc_layout(HnswGraph& g, uint64_t n, uint64_t n_up, uint64_t nmax) {
  const uint64_t m = (uint64_t)g.m;
  g.max_part = nmax;
  g.n_up = n_up;
  g.nlev.alloc(std::max<uint64_t>(n, 1));
  g.up_base.alloc(std::max<uint64_t>(n, 1));
  g.cnt0.alloc(std::max<uint64_t>(n, 1));
  g.nbr0.alloc(std::max<uint64_t>(n * 2 * m, 1));
  g.dst0.alloc(std::max<uint64_t>(n * 2 * m, 1));
  g.cntu.alloc(std::max<uint64_t>(n_up, 1));
  g.nbru.alloc(std::max<uint64_t>(n_up * m, 1));
  g.dstu.alloc(std::max<uint64_t>(n_up * m, 1));
}

// the levels and the empty lists of every partition's graph, then the build kernels with policy P and its table and
// query words TW / QW in each warp's scratch.  With `keep`, a kept partition's nodes take their levels from the old
// graph (a loaded graph has no seed) and its lists are spliced in; only the other partitions with at least 2 rows are
// built.  max_part and the upper rows are counted over the whole new layout.
template <class Dist>
static void build_graphs(HnswGraph& g, const uint64_t* part_offsets, int K, uint64_t seed, const HnswKeep* keep,
                         const Dist& P, uint32_t TW, uint32_t QW) {
  std::vector<uint64_t> off(K + 1);
  d2h(off.data(), part_offsets, (size_t)K + 1);
  std::vector<uint8_t> old_lev;
  if (keep) {
    LB2_REQUIRE(keep->old && keep->src.size() == (size_t)K && !keep->old_off.empty(), "%s: bad kept-graph table", g.kind);
    old_lev.resize(keep->old_off.back());
    if (!old_lev.empty()) d2h(old_lev.data(), keep->old->nlev.p, old_lev.size());
  }
  sync_stream();
  // the first upper row of every old node's partition: the old upper rows are compact in storage order
  std::vector<uint64_t> old_up;
  if (keep) {
    const size_t ok = keep->old_off.size() - 1;
    old_up.assign(ok + 1, 0);
    for (size_t q = 0; q < ok; ++q) {
      uint64_t u = 0;
      for (uint64_t r = keep->old_off[q]; r < keep->old_off[q + 1]; ++r) u += old_lev[r] - 1;
      old_up[q + 1] = old_up[q] + u;
    }
  }
  const uint64_t n = off[K];
  std::vector<uint64_t> thr(g.max_level);
  hnsw_level_thresholds(g.m, g.max_level, thr.data());
  std::vector<uint8_t> nlev(n);
  std::vector<uint32_t> up_base(n);
  uint64_t n_up = 0, nmax = 0;
  std::vector<uint32_t> order;
  std::vector<SpliceSpan> spans;
  for (int p = 0; p < K; ++p) {
    const uint64_t np_ = off[p + 1] - off[p];
    nmax = std::max(nmax, np_);
    const int64_t q = keep ? keep->src[p] : -1;
    if (q >= 0) {
      LB2_REQUIRE(keep->old_off[q + 1] - keep->old_off[q] == np_, "%s: kept partition %d changed size", g.kind, p);
      if (np_) spans.push_back({keep->old_off[q], off[p], np_, old_up[q], n_up, old_up[q + 1] - old_up[q]});
    } else if (np_ >= 2) {
      order.push_back((uint32_t)p);
    }
    for (uint64_t i = 0; i < np_; ++i) {
      int L = g.max_level;  // node 0: every level (builder.rs:368-370)
      if (q >= 0) {
        L = old_lev[keep->old_off[q] + i];
      } else if (i > 0) {
        const uint64_t u = hnsw_level_draw(seed, (uint32_t)p, (uint32_t)i);
        L = 1;
        for (int l = 1; l < g.max_level; ++l) L += u < thr[l] ? 1 : 0;
      }
      nlev[off[p] + i] = (uint8_t)L;
      up_base[off[p] + i] = (uint32_t)n_up;
      n_up += (uint64_t)(L - 1);
      LB2_REQUIRE(n_up < 0xffffffffull, "%s: more than 2^32 - 1 upper-level rows", g.kind);
    }
  }
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    return off[a + 1] - off[a] > off[b + 1] - off[b];
  });
  alloc_layout(g, n, n_up, nmax);
  if (n) {
    h2d(g.nlev.p, nlev.data(), n);
    h2d(g.up_base.p, up_base.data(), n);
  }
  g.cnt0.zero();
  g.cntu.zero();
  g.nbr0.zero();  // unused list slots export as zeros
  g.dst0.zero();
  g.nbru.zero();
  g.dstu.zero();
  if (!spans.empty()) {
    DevBuf<SpliceSpan> dspans(spans.size());
    h2d(dspans.p, spans.data(), spans.size());
    const HnswGraph& o = *keep->old;
    LB2_LAUNCH("hnsw_splice", hnsw_splice_kernel, dim3((unsigned)spans.size(), 8), 256, 0, (const SpliceSpan*)dspans.p,
               g.m, o.cnt0.p, o.nbr0.p, o.dst0.p, o.cntu.p, o.nbru.p, o.dstu.p, g.cnt0.p, g.nbr0.p, g.dst0.p, g.cntu.p,
               g.nbru.p, g.dstu.p);
    sync_stream();  // dspans is freed on return
  }
  if (order.empty()) {
    sync_stream();
    return;
  }
  const uint32_t E = (uint32_t)g.ef_construction, B = 2 * (uint32_t)g.m + 1, LB = std::max(E, B);
  const size_t words = scratch_words(nmax, E, B, LB, TW, QW);
  // one warp per work item, at most 32 per SM, and no more warps than 512 MB of scratch holds
  const size_t fit = std::max<size_t>(1, (512ull << 20) / (words * 4));
  DevBuf<uint32_t> dorder(order.size());
  h2d(dorder.p, order.data(), order.size());
  const int32_t lo = key_of_host(-3.40282347e+38f), hi = key_of_host(3.40282347e+38f);  // f32::MIN, f32::MAX
  const uint32_t batch = std::max<uint32_t>(g.insert_batch, 1);
  // LB2_HNSW_ROUNDS=1: insert_batch 1 through the round driver too (the same graph; for timing it against the serial
  // kernel).  Read on every call.
  const char* env_rounds = getenv("LB2_HNSW_ROUNDS");
  if (batch == 1 && !(env_rounds && *env_rounds && *env_rounds != '0')) {
    const unsigned nct = (unsigned)std::min<size_t>({order.size(), (size_t)ctx().num_sms * 32, fit});
    DevBuf<uint32_t> scratch(words * nct), next(1);
    next.zero();
    LB2_LAUNCH("hnsw_build", hnsw_build_kernel<Dist>, nct, 32, 0, dev_view(g), part_offsets, dorder.p,
               (int)order.size(), next.p, P, E, lo, hi, scratch.p, nmax, E, B, LB, TW, QW);
    sync_stream();
    return;
  }
  // The rounds: starting at s = 1, a round inserts nodes s .. s + min(batch, s) - 1 of every partition that has them,
  // so rounds hold 1, 2, 4, .. nodes, then `batch`.  `order` is largest first, so a round's partitions are a prefix.
  // Size the round buffers by the largest round: its items, and the entries its nodes' lists can hold.
  struct Round {
    uint32_t s0, W, nparts;
  };
  std::vector<Round> rounds;
  uint64_t max_items = 0, max_recs = 0;
  {
    const uint64_t top = off[order[0] + 1] - off[order[0]];
    uint32_t np_r = (uint32_t)order.size();
    for (uint64_t s0 = 1; s0 < top;) {
      const uint64_t W = std::min<uint64_t>(batch, s0);
      while (np_r > 0 && off[order[np_r - 1] + 1] - off[order[np_r - 1]] <= s0) --np_r;
      uint64_t recs = 0;
      for (uint32_t t = 0; t < np_r; ++t) {
        const uint64_t a = off[order[t]], np_ = off[order[t] + 1] - a;
        for (uint64_t i = s0; i < std::min(np_, s0 + W); ++i) recs += 2 * (uint64_t)g.m + (uint64_t)g.m * (nlev[a + i] - 1);
      }
      rounds.push_back({(uint32_t)s0, (uint32_t)W, np_r});
      max_items = std::max(max_items, (uint64_t)np_r * W);
      max_recs = std::max(max_recs, recs);
      s0 += W;
    }
  }
  LB2_REQUIRE(max_items < 0xffffffffull && max_recs < 0xffffffffull, "%s: a round of more than 2^32 - 1 back-links",
              g.kind);
  const unsigned nct = (unsigned)std::min<size_t>({(size_t)max_items, (size_t)ctx().num_sms * 32, fit});
  DevBuf<uint32_t> scratch(words * nct), counters(3), head(n + n_up), rec_i(max_recs), rec_key(max_recs),
      rec_next(max_recs), touched(3 * max_recs);
  LB2_CUDA(cudaMemsetAsync(head.p, 0xff, head.n * sizeof(uint32_t), ctx().stream));  // every chain empty (NONE)
  const RoundBufs rb{counters.p, head.p, rec_i.p, rec_key.p, rec_next.p, touched.p};
  for (const Round& r : rounds) {
    const uint64_t items = (uint64_t)r.nparts * r.W;
    counters.zero();
    LB2_LAUNCH("hnsw_round_search", hnsw_round_search_kernel<Dist>, (unsigned)std::min<uint64_t>(items, nct), 32, 0,
               dev_view(g), part_offsets, dorder.p, r.nparts, r.s0, r.W, rb, P, E, lo, hi, scratch.p, nmax, E, B, LB,
               TW, QW);
    LB2_LAUNCH("hnsw_round_link", hnsw_round_link_kernel, (unsigned)cdiv(items, 128), 128, 0, dev_view(g), n,
               part_offsets, dorder.p, r.nparts, r.s0, r.W, rb);
    LB2_LAUNCH("hnsw_round_apply", hnsw_round_apply_kernel<Dist>, nct, 32, 0, dev_view(g), n, part_offsets, rb, P,
               scratch.p, nmax, E, B, LB, TW, QW);
  }
  sync_stream();
}

// the words of a PQ warp's table (M x 2^nbits) and of a PQ or flat warp's query / row (d, kept 16-byte aligned)
static uint32_t pq_table_words(int M, int nbits) { return (uint32_t)M << nbits; }
static uint32_t query_words(int d) { return (uint32_t)(d + 3) & ~3u; }

// The distance policy of ix's graphs, the one place it is chosen: f(P, TW, QW) with P over ix's payload and model and
// TW / QW its table and query words in each warp's scratch.  s: the search (nullptr: the build), whose P holds its
// queries (f32, normalised under cosine) and the SQ query codes `qcodes` from query 0 on (at_slab moves them).
//  * SQ: r2 = (upper - lower)^2 (inverse_scalar_dist, sq.rs:279-287); cosine is L2 on the normalised vectors' codes.
//  * PQ: cosine is L2 (the storage's distance type, pq/storage.rs:465-468); dist_between of 16-bit rows under dot
//    takes 32 lanes (dot.rs:78-83,133), every other case 16.  The search never calls `between`, so it takes the f32
//    rule: one rule per (metric, nbits).
//  * FLAT: every distance, cosine included, is the IVF_FLAT scan's rule for the metric and the stored element type.
template <class F>
static void with_policy(const lb2_index& ix, const IvfSearch* s, const uint8_t* qcodes, F&& f) {
  const int d = ix.d, M = ix.M, nbits = ix.nbits;
  const float* queries = s ? s->queries : nullptr;
  switch (ix.kind) {
    case IndexKind::SQ: {
      const float rf = (float)(ix.sq_upper - ix.sq_lower);
      auto go = [&](auto m) {
        SqDist<decltype(m)::value> P{};
        P.base = ix.codes.p;
        P.qcodes = qcodes;
        P.d = d;
        P.r2 = rf * rf;
        f(P, 0u, 0u);
      };
      if (ix.metric == METRIC_DOT) go(std::integral_constant<int, METRIC_DOT>{});
      else go(std::integral_constant<int, METRIC_L2>{});
      break;
    }
    case IndexKind::PQ: {
      auto go = [&](auto m, auto rule) {
        auto with_bits = [&](auto b) {
          PqDist<decltype(m)::value, decltype(b)::value, decltype(rule)::value> P{};
          P.base = ix.codes.p;
          P.codebook = ix.codebook.p;
          P.queries = queries;
          P.centroids = ix.centroids.p;
          P.d = d;
          P.M = M;
          P.ds = d / M;
          P.cw = nbits == 4 ? M / 2 : M;
          f(P, pq_table_words(M, nbits), query_words(d));
        };
        if (nbits == 4) with_bits(std::integral_constant<int, 4>{});
        else with_bits(std::integral_constant<int, 8>{});
      };
      const lb2_dtype rule_dtype = s ? LB2_F32 : ix.dtype;
      if (ix.metric != METRIC_DOT)
        go(std::integral_constant<int, METRIC_L2>{}, std::integral_constant<int, RULE_LANES16>{});
      else if (rule_dtype == LB2_F16 || rule_dtype == LB2_BF16)
        go(std::integral_constant<int, METRIC_DOT>{}, std::integral_constant<int, RULE_DOT32>{});
      else
        go(std::integral_constant<int, METRIC_DOT>{}, std::integral_constant<int, RULE_LANES16>{});
      break;
    }
    case IndexKind::FLAT:
      dispatch_metric_elem<false>(ix.metric, (int)ix.vdtype(), [&](auto m, auto e) {
        using T = typename decltype(e)::type;
        FlatDist<decltype(m)::value, T> P{};
        P.base = reinterpret_cast<const T*>(ix.vectors.p);
        P.queries = queries;
        P.d = d;
        f(P, 0u, query_words(d));
      });
      break;
    case IndexKind::RQ:  // no IVF_RQ index has a graph
      break;
  }
}

void hnsw_build(HnswGraph& g, const lb2_index& ix, uint64_t seed, const HnswKeep* keep) {
  with_policy(ix, nullptr, nullptr, [&](const auto& P, uint32_t TW, uint32_t QW) {
    build_graphs(g, ix.part_offsets.p, ix.K, seed, keep, P, TW, QW);
  });
}

void hnsw_build_rows(HnswGraph& g, const float* rows, uint64_t n, int d, int metric, uint64_t seed) {
  LB2_REQUIRE(d % 4 == 0, "%s: the graph's rows need a dimension that is a multiple of 4, d = %d", g.kind, d);
  const uint64_t off[2] = {0, n};
  DevBuf<uint64_t> doff(2);
  h2d(doff.p, off, 2);
  auto go = [&](auto m) {
    FlatDist<decltype(m)::value, float> P{};
    P.base = rows;
    P.d = d;
    build_graphs(g, doff.p, 1, seed, nullptr, P, 0u, query_words(d));
  };
  if (metric == METRIC_DOT) go(std::integral_constant<int, METRIC_DOT>{});
  else go(std::integral_constant<int, METRIC_L2>{});
}

// caller memory (host or device) -> host
template <class T>
static std::vector<T> fetch(const T* src, size_t count) {
  std::vector<T> h(count);
  if (count) LB2_CUDA(cudaMemcpyAsync(h.data(), src, count * sizeof(T), cudaMemcpyDefault, ctx().stream));
  sync_stream();
  return h;
}

// a list naming one node twice would be expanded once here and twice by beam_search's filter-then-process loop
static void no_duplicates(const char* kind, const uint32_t* ids, uint32_t c, uint64_t row, int level) {
  for (uint32_t a = 0; a < c; ++a)
    for (uint32_t b = a + 1; b < c; ++b)
      LB2_REQUIRE(ids[a] != ids[b], "%s: row %llu lists node %u twice at level %d", kind, (unsigned long long)row,
                  ids[a], level);
}

void hnsw_load(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* levels, const uint32_t* counts0,
               const uint32_t* nbr0, const float* dist0, const uint32_t* counts_up, const uint32_t* nbr_up,
               const float* dist_up) {
  const std::vector<uint64_t> off = fetch(part_offsets, (size_t)K + 1);
  const uint64_t n = off[K], m = (uint64_t)g.m;
  LB2_REQUIRE(n == 0 || (levels && counts0 && nbr0 && dist0), "null argument");
  const std::vector<uint8_t> lv = fetch(levels, n);
  std::vector<uint32_t> up_base(n);
  uint64_t n_up = 0, nmax = 0;
  for (int p = 0; p < K; ++p) {
    nmax = std::max(nmax, off[p + 1] - off[p]);
    for (uint64_t r = off[p]; r < off[p + 1]; ++r) {
      const int L = lv[r];
      LB2_REQUIRE(L >= 1 && L <= g.max_level && (r > off[p] || L == g.max_level),
                  "%s: row %llu has %d levels (node 0 of a partition has max_level = %d, the others 1 .. %d)", g.kind,
                  (unsigned long long)r, L, g.max_level, g.max_level);
      up_base[r] = (uint32_t)n_up;
      n_up += (uint64_t)(L - 1);
      LB2_REQUIRE(n_up < 0xffffffffull, "%s: more than 2^32 - 1 upper-level rows", g.kind);
    }
  }
  LB2_REQUIRE(n_up == 0 || (counts_up && nbr_up && dist_up), "null argument");
  const std::vector<uint32_t> c0 = fetch(counts0, n), n0 = fetch(nbr0, n * 2 * m), cu = fetch(counts_up, n_up),
                              nu = fetch(nbr_up, n_up * m);
  for (int p = 0; p < K; ++p) {  // every neighbour is a node of the partition that has the level
    const uint64_t a = off[p], np_ = off[p + 1] - a;
    for (uint64_t r = a; r < off[p + 1]; ++r) {
      LB2_REQUIRE(c0[r] <= 2 * m, "%s: row %llu has %u level-0 neighbours (at most 2m = %llu)", g.kind,
                  (unsigned long long)r, c0[r], (unsigned long long)(2 * m));
      for (uint32_t j = 0; j < c0[r]; ++j)
        LB2_REQUIRE(n0[r * 2 * m + j] < np_, "%s: row %llu links to node %u of a %llu-row partition", g.kind,
                    (unsigned long long)r, n0[r * 2 * m + j], (unsigned long long)np_);
      no_duplicates(g.kind, &n0[r * 2 * m], c0[r], r, 0);
      for (int l = 1; l < lv[r]; ++l) {
        const uint64_t u = up_base[r] + (l - 1);
        LB2_REQUIRE(cu[u] <= m, "%s: row %llu has %u neighbours at level %d (at most m = %llu)", g.kind,
                    (unsigned long long)r, cu[u], l, (unsigned long long)m);
        for (uint32_t j = 0; j < cu[u]; ++j) {
          const uint32_t id = nu[u * m + j];
          LB2_REQUIRE(id < np_ && lv[a + id] > l, "%s: row %llu links at level %d to node %u, which lacks it", g.kind,
                      (unsigned long long)r, l, id);
        }
        no_duplicates(g.kind, &nu[u * m], cu[u], r, l);
      }
    }
  }
  alloc_layout(g, n, n_up, nmax);
  cudaStream_t st = ctx().stream;
  if (n) {
    h2d(g.nlev.p, lv.data(), n);
    h2d(g.up_base.p, up_base.data(), n);
    h2d(g.cnt0.p, c0.data(), n);
    h2d(g.nbr0.p, n0.data(), n * 2 * m);
    LB2_CUDA(cudaMemcpyAsync(g.dst0.p, dist0, sizeof(float) * n * 2 * m, cudaMemcpyDefault, st));
  }
  if (n_up) {
    h2d(g.cntu.p, cu.data(), n_up);
    h2d(g.nbru.p, nu.data(), n_up * m);
    LB2_CUDA(cudaMemcpyAsync(g.dstu.p, dist_up, sizeof(float) * n_up * m, cudaMemcpyDefault, st));
  }
  sync_stream();
}

// HNSW::search of every probed partition with policy P0 (its queries from the search's first on) and its table and
// query words TW / QW in each warp's scratch
template <class Dist>
static void search_graphs(const IvfSearch& s, const HnswGraph& g, uint32_t ef, const Dist& P0, uint32_t TW,
                          uint32_t QW) {
  const uint32_t kc = (uint32_t)s.k;
  if (ef == 0) ef = kc + kc / 2;
  // per-query values: every query's ef was resolved and checked by the caller, ef is the largest
  if (ef < kc && !s.qp) fail(LB2_INVALID_ARG, "%s: ef = %u must be greater than or equal to k = %u", g.kind, ef, kc);
  if (!ivf_search_begin(s, 0, "%zu", 0)) return;
  DevBuf<uint32_t> acnt;
  if (s.flt.allow && !s.qp) {  // `remained`: the allowed rows of each partition (builder.rs:715-718)
    acnt.alloc(s.K);
    partition_counts(s.part_offsets, s.K, s.flt.allow, 0xffffffffu, acnt.p);
  }
  const uint64_t nmax = std::max<uint64_t>(g.max_part, 1);
  const uint32_t E = std::max(ef, kc), B = std::max<uint32_t>(2 * (uint32_t)g.m, 32);
  const size_t words = scratch_words(nmax, E, B, 0, TW, QW);
  const uint64_t cap = std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx().num_sms * 32, (256ull << 20) / (words * 4)));
  DevBuf<uint32_t> scratch(words * cap);
  run_ivf_search(s, [&](const ScanSlots& sl) {
    const uint64_t nslots = sl.qn * sl.np;
    if (nslots == 0) return;
    const unsigned nct = (unsigned)std::min<uint64_t>(nslots, cap);
    Dist P = P0;
    P.at_slab(sl.q0);
    LB2_LAUNCH("hnsw_search", hnsw_search_kernel<Dist>, nct, 32, 0, dev_view(g), nslots, sl.np, sl.probe_ids,
               sl.offsets, acnt.p, P, s.row_ids, ef, (int)kc, s.flt, sl.cand_d, sl.cand_id, sl.cand_cnt, scratch.p,
               nmax, E, B, TW, QW, s.qp_at(sl.q0));
  });
}

void hnsw_search(const IvfSearch& s, const lb2_index& ix, const uint8_t* sq_query_codes, uint32_t ef) {
  with_policy(ix, &s, sq_query_codes, [&](const auto& P, uint32_t TW, uint32_t QW) {
    search_graphs(s, *ix.hnsw, ef, P, TW, QW);
  });
}

}  // namespace lb2
