// hnsw.cu -- IVF_HNSW_SQ: an HNSW graph per partition over the partition's SQ codes, built and searched on the device
// (lance-index/src/vector/hnsw/builder.rs, graph.rs, hnsw.rs, graph/builder.rs).
//
// Replaces  HNSW::index_vectors / HnswBuilder::insert      hnsw/builder.rs:386-507,742-775
//           select_neighbors_heuristic                   hnsw.rs:60-88
//           beam_search / greedy_search                  graph.rs:275-409
//           HNSW::search / search_inner / flat_search    hnsw/builder.rs:164-280,678-739
//
// Every distance is the SQ row rule of sq.cuh (query-to-row and row-to-row alike, sq/storage.rs:387-444,
// storage.rs:102-105): an integer sum times one constant, so the build is deterministic and bit-exact.
//
// One warp owns one partition (build) or one (query, partition) slot (search).  Its heaps and visited bitset live in
// a per-warp global scratch sized by the largest partition, so no partition is refused for its size.  Lane 0 runs
// the reference's serial heap and list updates in the reference's order; the 32 lanes compute the distances of a
// neighbour list or of a candidate's accepted neighbours, one row per lane.  Control decisions reach the other lanes through shared memory after a
// __syncwarp.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "exact.cuh"
#include "hnsw.cuh"
#include "ivf_search.cuh"
#include "probe.cuh"
#include "sq.cuh"
#include "topk.cuh"

namespace lb2 {

namespace {

constexpr uint32_t KEY_INF = 0xff800000u;  // unsigned order key of f32::INFINITY
constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ uint32_t ukey_of(float f) { return (uint32_t)total_order_key(f) ^ 0x80000000u; }
__device__ __forceinline__ float float_of(uint32_t uk) { return key_to_float((int32_t)(uk ^ 0x80000000u)); }

struct GraphDev {
  const uint8_t* nlev;
  const uint32_t* up_base;
  uint32_t *cnt0, *nbr0, *cntu, *nbru;
  float *dst0, *dstu;
  int m, max_level;
};
struct ListRef {
  uint32_t* cnt;
  uint32_t* ids;
  float* dist;
};
// the list of global row `row` at `level`
__device__ __forceinline__ ListRef list_of(const GraphDev& g, uint64_t row, int level) {
  if (level == 0) return {g.cnt0 + row, g.nbr0 + row * 2 * g.m, g.dst0 + row * 2 * g.m};
  const uint64_t r = (uint64_t)g.up_base[row] + (level - 1);
  return {g.cntu + r, g.nbru + r * g.m, g.dstu + r * g.m};
}

// one partition as a warp sees it
struct Part {
  const uint8_t* codes;  // the partition's first code row
  uint64_t off;          // its first storage position
  uint32_t n;
  int d;
  float r2;
};

// per-warp scratch (u32 words): vis[words(nmax)], candidate heap ck / cid [nmax + 1], result heap rk / rid [E + 1],
// batch bid / bk [B], list lid / lk / ord [LB], accepted aid / ak [B]
struct Scratch {
  uint32_t *vis, *ck, *cid, *rk, *rid, *bid, *bk, *lid, *lk, *ord, *aid, *ak;
};
__host__ __device__ inline size_t scratch_words(uint64_t nmax, uint32_t E, uint32_t B, uint32_t LB) {
  return (nmax + 31) / 32 + 2 * (nmax + 1) + 2 * ((size_t)E + 1) + 4 * (size_t)B + 3 * (size_t)LB;
}
__device__ inline Scratch scratch_at(uint32_t* base, uint64_t nmax, uint32_t E, uint32_t B, uint32_t LB) {
  Scratch s;
  s.vis = base;
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

// keys[j] = key(q, node ids[j]) for j < n, one node per lane; the ids must be visible to every lane
template <int METRIC>
__device__ __forceinline__ void warp_keys(const Part& P, const uint8_t* q, const uint32_t* ids, uint32_t n,
                                          uint32_t* keys) {
  for (uint32_t j = threadIdx.x & 31; j < n; j += 32) keys[j] = pair_key<METRIC>(q, P.codes + (uint64_t)ids[j] * P.d, P.d, P.r2);
  __syncwarp();
}

__device__ __forceinline__ bool allowed(const uint64_t* allow, uint64_t pos) {
  return allow == nullptr || ((allow[pos >> 6] >> (pos & 63)) & 1ull) != 0;
}

// greedy_search (graph.rs:375-409): neighbours in list order, strictly closer (f32 `<`) moves on
template <int METRIC>
__device__ void greedy(const GraphDev& g, const Part& P, const uint8_t* q, int level, uint32_t& cur, uint32_t& ckey,
                       const Scratch& s) {
  __shared__ uint32_t sh_cur, sh_key, sh_go;
  const int lane = threadIdx.x & 31;
  for (;;) {
    const ListRef L = list_of(g, P.off + cur, level);
    const uint32_t n = *L.cnt;
    warp_keys<METRIC>(P, q, L.ids, n, s.bk);
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
template <int METRIC>
__device__ uint32_t beam_search(const GraphDev& g, const Part& P, const uint8_t* q, int level, uint32_t ep,
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
    warp_keys<METRIC>(P, q, s.bid, n, s.bk);
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
template <int METRIC>
__device__ void prune_into(const Part& P, const uint32_t* ids, const uint32_t* keys, uint32_t c, uint32_t m_max,
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
    const uint8_t* urow = P.codes + (uint64_t)uid * P.d;
    for (uint32_t j = lane; j < na; j += 32)
      ok = ok && ukey < pair_key<METRIC>(urow, P.codes + (uint64_t)s.aid[j] * P.d, P.d, P.r2);
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
    for (uint32_t j = 0; j < na; ++j) {
      dst.ids[j] = s.aid[j];
      dst.dist[j] = float_of(s.ak[j]);
    }
    *dst.cnt = na;
  }
  __syncwarp();
}

// HNSW::index_vectors of partitions order[0 ..), taken largest first by a persistent grid of one-warp CTAs
template <int METRIC>
__global__ void __launch_bounds__(32)
hnsw_build_kernel(GraphDev g, const uint64_t* __restrict__ part_offsets, const uint32_t* __restrict__ order, int nparts,
                  uint32_t* __restrict__ next, const uint8_t* __restrict__ codes, int d, float r2, uint32_t efc,
                  int32_t lo, int32_t hi, uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B,
                  uint32_t LB) {
  __shared__ uint32_t sh_part, sh_go, sh_n;
  const int lane = threadIdx.x & 31;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, LB), nmax, E, B, LB);
  for (;;) {
    if (lane == 0) sh_part = atomicAdd(next, 1u);
    __syncwarp();
    const uint32_t t = sh_part;
    __syncwarp();
    if (t >= (uint32_t)nparts) return;
    const uint32_t p = order[t];
    Part P;
    P.off = part_offsets[p];
    P.n = (uint32_t)(part_offsets[p + 1] - P.off);
    P.codes = codes + P.off * d;
    P.d = d;
    P.r2 = r2;
    for (uint32_t i = 1; i < P.n; ++i) {  // HnswBuilder::insert (builder.rs:396-463)
      const uint8_t* q = P.codes + (uint64_t)i * d;
      const int target = (int)g.nlev[P.off + i] - 1;
      uint32_t ep = 0, ekey = pair_key<METRIC>(q, P.codes, d, r2);
      for (int level = g.max_level - 1; level > target; --level) greedy<METRIC>(g, P, q, level, ep, ekey, s);
      for (int level = target; level >= 0; --level) {
        const uint32_t R = beam_search<METRIC>(g, P, q, level, ep, ekey, efc, nullptr, lo, hi, s);
        ep = s.rid[0];
        ekey = s.rk[0];
        const uint32_t m_max = level == 0 ? 2 * g.m : g.m;
        prune_into<METRIC>(P, s.rid, s.rk, R, m_max, list_of(g, P.off + i, level), s);
      }
      for (int level = 0; level <= target; ++level) {  // the back-links, level by level, in pruned-list order
        const uint32_t m_max = level == 0 ? 2 * g.m : g.m;
        const ListRef mine = list_of(g, P.off + i, level);
        const uint32_t cm = *mine.cnt;
        for (uint32_t e = 0; e < cm; ++e) {
          const uint32_t eid = mine.ids[e];
          const ListRef other = list_of(g, P.off + eid, level);
          if (lane == 0) {
            const uint32_t ekey2 = ukey_of(mine.dist[e]);
            const uint32_t c2 = *other.cnt;
            const uint32_t cutoff = c2 < m_max ? KEY_INF : ukey_of(other.dist[c2 - 1]);  // the LAST entry
            const bool add = ekey2 < cutoff;
            if (add) {
              for (uint32_t j = 0; j < c2; ++j) {
                s.lid[j] = other.ids[j];
                s.lk[j] = ukey_of(other.dist[j]);
              }
              s.lid[c2] = i;
              s.lk[c2] = ekey2;
            }
            sh_go = add;
            sh_n = c2 + 1;
          }
          __syncwarp();
          const bool add = sh_go;
          const uint32_t c = sh_n;
          __syncwarp();
          if (add) prune_into<METRIC>(P, s.lid, s.lk, c, m_max, other, s);
        }
      }
    }
  }
}

// HNSW::search of every slot: partition id >= K or an empty partition -> no rows; the prefilter's flat branch when
// fewer than 10 % of the partition's rows are allowed (builder.rs:715-725), search_inner otherwise
template <int METRIC>
__global__ void __launch_bounds__(32)
hnsw_search_kernel(GraphDev g, uint64_t nslots, int np, const uint32_t* __restrict__ probe_ids,
                   const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ acnt,
                   const uint8_t* __restrict__ qcodes, const uint8_t* __restrict__ codes, int d, float r2,
                   const uint64_t* __restrict__ row_ids, uint32_t ef, int kc, ScanFilter flt,
                   float* __restrict__ cand_d, uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt,
                   uint32_t* __restrict__ scratch, uint64_t nmax, uint32_t E, uint32_t B) {
  __shared__ uint32_t sh_n;
  const int lane = threadIdx.x & 31;
  const Scratch s = scratch_at(scratch + blockIdx.x * scratch_words(nmax, E, B, 0), nmax, E, B, 0);
  for (uint64_t slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
    const uint64_t qi = slot / np;
    const uint32_t p = probe_ids[slot];
    Part P;
    P.off = offsets[p];
    P.n = (uint32_t)(offsets[p + 1] - P.off);
    P.codes = codes + P.off * d;
    P.d = d;
    P.r2 = r2;
    if (P.n == 0) {  // an empty partition returns no rows (builder.rs:695-697)
      if (lane == 0) cand_cnt[slot] = 0;
      continue;
    }
    const uint8_t* q = qcodes + qi * d;
    uint32_t R;
    if (flt.allow && acnt[p] < (uint32_t)((uint64_t)P.n * 10 / 100)) {
      // HNSW::flat_search (builder.rs:238-280): allowed rows in node order, kept when lower < d <= upper.  Lane 0 drives
      // the reference's heap over the partition's rows, 32 distances at a time; this branch only runs when fewer than
      // 10 % of the rows are allowed.
      uint32_t len = 0;
      for (uint32_t c0 = 0; c0 < P.n; c0 += 32) {
        const uint32_t j = c0 + lane;
        if (j < P.n && allowed(flt.allow, P.off + j)) s.bk[lane] = pair_key<METRIC>(q, P.codes + (uint64_t)j * d, d, r2);
        __syncwarp();
        if (lane == 0) {
          for (uint32_t t = 0; t < 32 && c0 + t < P.n; ++t) {
            if (!allowed(flt.allow, P.off + c0 + t)) continue;
            const uint32_t key = s.bk[t];
            const int32_t sk = (int32_t)(key ^ 0x80000000u);
            if (sk <= flt.lo_key || sk > flt.hi_key) continue;
            if (len < (uint32_t)kc) {
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
      uint32_t ep = 0, ekey = pair_key<METRIC>(q, P.codes, d, r2);
      for (int level = g.max_level - 1; level >= 0; --level) greedy<METRIC>(g, P, q, level, ep, ekey, s);
      R = beam_search<METRIC>(g, P, q, 0, ep, ekey, ef, flt.allow, flt.lo_key, flt.hi_key, s);
      R = min(R, (uint32_t)kc);
    }
    for (uint32_t j = lane; j < R; j += 32) {
      cand_d[slot * kc + j] = float_of(s.rk[j]);
      cand_id[slot * kc + j] = row_ids[P.off + s.rid[j]];
    }
    if (lane == 0) cand_cnt[slot] = R;
    __syncwarp();
  }
}

GraphDev dev_view(const HnswGraph& g) {
  return GraphDev{g.nlev.p, g.up_base.p, g.cnt0.p, g.nbr0.p, g.cntu.p, g.nbru.p, g.dst0.p, g.dstu.p, g.m, g.max_level};
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

void hnsw_build(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* codes, int d, int metric, float r2,
                uint64_t seed) {
  std::vector<uint64_t> off(K + 1);
  d2h(off.data(), part_offsets, (size_t)K + 1);
  sync_stream();
  const uint64_t n = off[K];
  std::vector<uint64_t> thr(g.max_level);
  hnsw_level_thresholds(g.m, g.max_level, thr.data());
  std::vector<uint8_t> nlev(n);
  std::vector<uint32_t> up_base(n);
  uint64_t n_up = 0, nmax = 0;
  std::vector<uint32_t> order;
  for (int p = 0; p < K; ++p) {
    const uint64_t np_ = off[p + 1] - off[p];
    nmax = std::max(nmax, np_);
    if (np_ >= 2) order.push_back((uint32_t)p);
    for (uint64_t i = 0; i < np_; ++i) {
      int L = g.max_level;  // node 0: every level (builder.rs:368-370)
      if (i > 0) {
        const uint64_t u = hnsw_level_draw(seed, (uint32_t)p, (uint32_t)i);
        L = 1;
        for (int l = 1; l < g.max_level; ++l) L += u < thr[l] ? 1 : 0;
      }
      nlev[off[p] + i] = (uint8_t)L;
      up_base[off[p] + i] = (uint32_t)n_up;
      n_up += (uint64_t)(L - 1);
      LB2_REQUIRE(n_up < 0xffffffffull, "IVF_HNSW_SQ: more than 2^32 - 1 upper-level rows");
    }
  }
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    return off[a + 1] - off[a] > off[b + 1] - off[b];
  });
  g.max_part = nmax;
  g.n_up = n_up;
  g.nlev.alloc(std::max<uint64_t>(n, 1));
  g.up_base.alloc(std::max<uint64_t>(n, 1));
  g.cnt0.alloc(std::max<uint64_t>(n, 1));
  g.nbr0.alloc(std::max<uint64_t>(n * 2 * g.m, 1));
  g.dst0.alloc(std::max<uint64_t>(n * 2 * g.m, 1));
  g.cntu.alloc(std::max<uint64_t>(n_up, 1));
  g.nbru.alloc(std::max<uint64_t>(n_up * g.m, 1));
  g.dstu.alloc(std::max<uint64_t>(n_up * g.m, 1));
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
  if (order.empty()) {
    sync_stream();
    return;
  }
  const uint32_t E = (uint32_t)g.ef_construction, B = 2 * (uint32_t)g.m + 1, LB = std::max(E, B);
  const size_t words = scratch_words(nmax, E, B, LB);
  // one warp per partition, at most 32 per SM, and no more warps than 512 MB of scratch holds
  const size_t fit = std::max<size_t>(1, (512ull << 20) / (words * 4));
  const unsigned nct = (unsigned)std::min<size_t>({order.size(), (size_t)ctx().num_sms * 32, fit});
  DevBuf<uint32_t> scratch(words * nct), dorder(order.size()), next(1);
  h2d(dorder.p, order.data(), order.size());
  next.zero();
  const int32_t lo = key_of_host(-3.40282347e+38f), hi = key_of_host(3.40282347e+38f);  // f32::MIN, f32::MAX
  auto launch = [&](auto kern) {
    LB2_LAUNCH("hnsw_build", kern, nct, 32, 0, dev_view(g), part_offsets, dorder.p, (int)order.size(), next.p, codes,
               d, r2, E, lo, hi, scratch.p, nmax, E, B, LB);
  };
  if (metric == METRIC_DOT) launch(hnsw_build_kernel<METRIC_DOT>);
  else launch(hnsw_build_kernel<METRIC_L2>);  // cosine: L2 on the normalised vectors' codes
  sync_stream();
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
static void no_duplicates(const uint32_t* ids, uint32_t c, uint64_t row, int level) {
  for (uint32_t a = 0; a < c; ++a)
    for (uint32_t b = a + 1; b < c; ++b)
      LB2_REQUIRE(ids[a] != ids[b], "IVF_HNSW_SQ: row %llu lists node %u twice at level %d", (unsigned long long)row,
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
                  "IVF_HNSW_SQ: row %llu has %d levels (node 0 of a partition has max_level = %d, the others 1 .. %d)",
                  (unsigned long long)r, L, g.max_level, g.max_level);
      up_base[r] = (uint32_t)n_up;
      n_up += (uint64_t)(L - 1);
      LB2_REQUIRE(n_up < 0xffffffffull, "IVF_HNSW_SQ: more than 2^32 - 1 upper-level rows");
    }
  }
  LB2_REQUIRE(n_up == 0 || (counts_up && nbr_up && dist_up), "null argument");
  const std::vector<uint32_t> c0 = fetch(counts0, n), n0 = fetch(nbr0, n * 2 * m), cu = fetch(counts_up, n_up),
                              nu = fetch(nbr_up, n_up * m);
  for (int p = 0; p < K; ++p) {  // every neighbour is a node of the partition that has the level
    const uint64_t a = off[p], np_ = off[p + 1] - a;
    for (uint64_t r = a; r < off[p + 1]; ++r) {
      LB2_REQUIRE(c0[r] <= 2 * m, "IVF_HNSW_SQ: row %llu has %u level-0 neighbours (at most 2m = %llu)",
                  (unsigned long long)r, c0[r], (unsigned long long)(2 * m));
      for (uint32_t j = 0; j < c0[r]; ++j)
        LB2_REQUIRE(n0[r * 2 * m + j] < np_, "IVF_HNSW_SQ: row %llu links to node %u of a %llu-row partition",
                    (unsigned long long)r, n0[r * 2 * m + j], (unsigned long long)np_);
      no_duplicates(&n0[r * 2 * m], c0[r], r, 0);
      for (int l = 1; l < lv[r]; ++l) {
        const uint64_t u = up_base[r] + (l - 1);
        LB2_REQUIRE(cu[u] <= m, "IVF_HNSW_SQ: row %llu has %u neighbours at level %d (at most m = %llu)",
                    (unsigned long long)r, cu[u], l, (unsigned long long)m);
        for (uint32_t j = 0; j < cu[u]; ++j) {
          const uint32_t id = nu[u * m + j];
          LB2_REQUIRE(id < np_ && lv[a + id] > l, "IVF_HNSW_SQ: row %llu links at level %d to node %u, which lacks it",
                      (unsigned long long)r, l, id);
        }
        no_duplicates(&nu[u * m], cu[u], r, l);
      }
    }
  }
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

void hnsw_search(const IvfSearch& s, const HnswGraph& g, const uint8_t* codes, float r2, const uint8_t* qcodes,
                 uint32_t ef) {
  const uint32_t kc = (uint32_t)s.k;
  if (ef == 0) ef = kc + kc / 2;
  if (ef < kc) fail(LB2_INVALID_ARG, "IVF_HNSW_SQ: ef = %u must be greater than or equal to k = %u", ef, kc);
  if (!ivf_search_begin(s, 0, "%zu", 0)) return;
  DevBuf<uint32_t> acnt;
  if (s.flt.allow) {  // `remained`: the allowed rows of each partition (builder.rs:715-718)
    acnt.alloc(s.K);
    partition_counts(s.part_offsets, s.K, s.flt.allow, 0xffffffffu, acnt.p);
  }
  const uint64_t nmax = std::max<uint64_t>(g.max_part, 1);
  const uint32_t E = std::max(ef, kc), B = std::max<uint32_t>(2 * (uint32_t)g.m, 32);
  const size_t words = scratch_words(nmax, E, B, 0);
  const uint64_t cap = std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx().num_sms * 32, (256ull << 20) / (words * 4)));
  DevBuf<uint32_t> scratch(words * cap);
  run_ivf_search(s, [&](const ScanSlots& sl) {
    const uint64_t nslots = sl.qn * sl.np;
    if (nslots == 0) return;
    const unsigned nct = (unsigned)std::min<uint64_t>(nslots, cap);
    auto launch = [&](auto kern) {
      LB2_LAUNCH("hnsw_search", kern, nct, 32, 0, dev_view(g), nslots, sl.np, sl.probe_ids, sl.offsets, acnt.p,
                 qcodes + sl.q0 * s.d, codes, s.d, r2, s.row_ids, ef, (int)kc, s.flt, sl.cand_d, sl.cand_id,
                 sl.cand_cnt, scratch.p, nmax, E, B);
    };
    if (s.metric == METRIC_DOT) launch(hnsw_search_kernel<METRIC_DOT>);
    else launch(hnsw_search_kernel<METRIC_L2>);
  });
}

}  // namespace lb2
