// ivf_search.cu -- the part of an IVF search that does not depend on the index kind: probe selection, the two
// skeletons (a fixed nprobes, or a probe rule) that drive a kind's scan, and the merges of candidate lists.
//
// Replaces  kmeans_find_partitions               lance-index/src/vector/kmeans.rs:1134-1158
//           SortExec(_distance,_rowid).fetch(k)  rust/lance/src/dataset/scanner.rs:3450-3466
#include <algorithm>

#include "assign.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "ivf_search.cuh"
#include "probe.cuh"
#include "topk.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// coarse probe selection: nprobes smallest (distance, id), ascending (kmeans.rs:1152-1157)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
select_probes_kernel(const float* __restrict__ all_dists, int K, int nprobes,
                     uint32_t* __restrict__ ids, float* __restrict__ dists) {
  const float* row = all_dists + (size_t)blockIdx.x * K;
  emit_ascending<128>(
      nprobes, K,
      [&](uint32_t c, int32_t& key, uint64_t& tie) {
        key = total_order_key(row[c]);
        tie = c;
        return true;
      },
      [&](uint32_t r, uint32_t c, int32_t, uint64_t) {
        ids[(size_t)blockIdx.x * nprobes + r] = c;
        dists[(size_t)blockIdx.x * nprobes + r] = row[c];
      });
}

// global merge per query: ascending (distance, row id), first k.  Candidate e of list pi of query qi sits
// at cand[pi * stride_p + qi * stride_q + e] (per-partition lists of one GPU: stride_p = k, stride_q = np * k;
// per-rank results gathered from a sharded index: stride_p = the rank stride, stride_q = k).
// A query may hold nl > np lists: they are merged in groups of np consecutive lists, output row qi * ng + g for group
// g (ng = ceil(nl / np)); nl = np is the plain merge.  Block b merges group b % ng of query b / ng.
// Lists of up to MERGE_RANK_MAX candidates in total are merged by RANK COUNTING in shared memory: every candidate
// counts the candidates that precede it in (distance, row id) order -- the pairs are unique -- and the ones with rank
// < k are the output, already in place.  (The k-round argmin below re-reads all candidates from global memory per
// round: 3.6 ms for 10 000 queries x 10 lists x k = 100; it remains for larger totals.)
constexpr int MERGE_RANK_MAX = 2048;
__global__ void __launch_bounds__(256)
merge_rank_kernel(const float* __restrict__ cand_d, const uint64_t* __restrict__ cand_id,
                  const uint32_t* __restrict__ cand_cnt, int np, int k, size_t stride_p_d, size_t stride_p_id,
                  size_t stride_q, size_t cnt_stride_p, size_t cnt_stride_q, int nl, uint64_t* __restrict__ out_id,
                  float* __restrict__ out_d, uint32_t* __restrict__ out_cnt, const QueryParam* __restrict__ qp) {
  extern __shared__ __align__(16) unsigned char mr_smem[];
  const int total = np * k;
  uint64_t* s_id = reinterpret_cast<uint64_t*>(mr_smem);             // [total]
  int32_t* s_key = reinterpret_cast<int32_t*>(s_id + total);         // [total]; invalid entries: key = INT_MAX, id = ~0
  __shared__ uint32_t s_valid;
  const size_t qi = blockIdx.x;
  const int ng = nl > np ? (nl + np - 1) / np : 1;
  const size_t q = qi / ng;
  const int first = (int)(qi % ng) * np;
  const int kq = qp ? qp[q].k : k;  // the query's own output length; the lists' stride stays k
  const int tid = threadIdx.x;
  if (tid == 0) s_valid = 0;
  __syncthreads();
  uint32_t myvalid = 0;
  for (int c = tid; c < total; c += 256) {
    const int pi = first + c / k, e = c % k;
    const bool ok = pi < nl && (uint32_t)e < cand_cnt[pi * cnt_stride_p + q * cnt_stride_q];
    s_key[c] = ok ? total_order_key(cand_d[pi * stride_p_d + q * stride_q + e]) : 0x7fffffff;
    s_id[c] = ok ? cand_id[pi * stride_p_id + q * stride_q + e] : ~0ull;
    myvalid += ok ? 1u : 0u;
  }
  if (myvalid) atomicAdd(&s_valid, myvalid);
  __syncthreads();
  for (int c = tid; c < total; c += 256) {
    const uint64_t id = s_id[c];
    if (id == ~0ull && s_key[c] == 0x7fffffff) continue;
    const int32_t key = s_key[c];
    int rank = 0;
    for (int j = 0; j < total; ++j) {
      const int32_t kj = s_key[j];
      rank += (kj < key || (kj == key && s_id[j] < id)) ? 1 : 0;
    }
    if (rank < kq) {
      out_id[qi * k + rank] = id;
      out_d[qi * k + rank] = key_to_float(key);
    }
  }
  const int r = min((uint32_t)kq, s_valid);
  for (int e = r + tid; e < k; e += 256) {
    out_id[qi * k + e] = ~0ull;
    out_d[qi * k + e] = __int_as_float(0x7f800000);
  }
  if (tid == 0 && out_cnt) out_cnt[qi] = r;
}

__global__ void __launch_bounds__(128)
merge_kernel(const float* __restrict__ cand_d, const uint64_t* __restrict__ cand_id,
             const uint32_t* __restrict__ cand_cnt, int np, int k, size_t stride_p_d, size_t stride_p_id,
             size_t stride_q, size_t cnt_stride_p, size_t cnt_stride_q, int nl, uint64_t* __restrict__ out_id,
             float* __restrict__ out_d, uint32_t* __restrict__ out_cnt, const QueryParam* __restrict__ qp) {
  const size_t qi = blockIdx.x;
  const int ng = nl > np ? (nl + np - 1) / np : 1;
  const size_t q = qi / ng;
  const int first = (int)(qi % ng) * np;
  const int tid = threadIdx.x;
  const int r = (int)emit_ascending<128>(
      qp ? qp[q].k : k, np * k,
      [&](uint32_t c, int32_t& key, uint64_t& id) {
        const int pi = first + c / k, e = c % k;
        if (pi >= nl || (uint32_t)e >= cand_cnt[pi * cnt_stride_p + q * cnt_stride_q]) return false;
        key = total_order_key(cand_d[pi * stride_p_d + q * stride_q + e]);
        id = cand_id[pi * stride_p_id + q * stride_q + e];
        return true;
      },
      [&](uint32_t r, uint32_t c, int32_t, uint64_t id) {
        out_id[qi * k + r] = id;
        out_d[qi * k + r] = cand_d[(first + c / k) * stride_p_d + q * stride_q + (c % k)];
      });
  for (int e = r + tid; e < k; e += 128) {
    out_id[qi * k + e] = ~0ull;
    out_d[qi * k + e] = __int_as_float(0x7f800000);
  }
  if (tid == 0 && out_cnt) out_cnt[qi] = r;
}

void find_partitions_f32(const float* centroids, int K, int d, int metric, const float* queries,
                         uint64_t nq, int nprobes, uint32_t* ids, float* dists) {
  if (nq == 0) return;
  DevBuf<float> all((size_t)nq * K);
  centroid_distances(queries, nq, d, centroids, K, metric, all.p);
  LB2_LAUNCH("select_probes", select_probes_kernel, (unsigned)nq, 128, 0, all.p, K, nprobes, ids, dists);
}

void merge_lists(const char* name, uint64_t nq, const float* cand_d, const uint64_t* cand_id, const uint32_t* cand_cnt,
                 int np, int k, size_t stride_p_d, size_t stride_p_id, size_t stride_q, size_t cnt_stride_p,
                 size_t cnt_stride_q, uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nl,
                 const QueryParam* qp) {
  if (nq == 0) return;
  if (nl < np) nl = np;
  const uint64_t blocks = nq * (uint64_t)(nl > np ? (nl + np - 1) / np : 1);
  const size_t total = (size_t)np * k;
  if (total <= (size_t)MERGE_RANK_MAX) {
    LB2_LAUNCH(name, merge_rank_kernel, (unsigned)blocks, 256, total * 12, cand_d, cand_id, cand_cnt, np, k, stride_p_d,
               stride_p_id, stride_q, cnt_stride_p, cnt_stride_q, nl, out_ids, out_dists, out_counts, qp);
  } else {
    LB2_LAUNCH(name, merge_kernel, (unsigned)blocks, 128, 0, cand_d, cand_id, cand_cnt, np, k, stride_p_d, stride_p_id,
               stride_q, cnt_stride_p, cnt_stride_q, nl, out_ids, out_dists, out_counts, qp);
  }
}

// nl lists per query, laid out [nq][nl][k] with counts [nq][nl]: groups of MERGE_RANK_MAX / k lists are merged by rank
// counting, level by level (one launch per level), until one merge of at most MERGE_RANK_MAX candidates is left
void merge_list_tree(const char* name, uint64_t nq, const float* cand_d, const uint64_t* cand_id,
                     const uint32_t* cand_cnt, int nl, int k, uint64_t* out_ids, float* out_dists,
                     uint32_t* out_counts) {
  if (nq == 0) return;
  const int G = std::max(2, MERGE_RANK_MAX / k);
  DevBuf<float> lvl_d[2];
  DevBuf<uint64_t> lvl_id[2];
  DevBuf<uint32_t> lvl_cnt[2];
  for (int cur = 0; nl > G; cur ^= 1) {
    const int ng = (nl + G - 1) / G;
    lvl_d[cur].alloc(nq * ng * k);
    lvl_id[cur].alloc(nq * ng * k);
    lvl_cnt[cur].alloc(nq * ng);
    merge_lists(name, nq, cand_d, cand_id, cand_cnt, G, k, (size_t)k, (size_t)k, (size_t)nl * k, 1, (size_t)nl,
                lvl_id[cur].p, lvl_d[cur].p, lvl_cnt[cur].p, nl);
    cand_d = lvl_d[cur].p;
    cand_id = lvl_id[cur].p;
    cand_cnt = lvl_cnt[cur].p;
    nl = ng;
  }
  merge_lists(name, nq, cand_d, cand_id, cand_cnt, nl, k, (size_t)k, (size_t)k, (size_t)nl * k, 1, (size_t)nl, out_ids,
              out_dists, out_counts);
}

// partitions are found with L2 on the (normalised) vectors for cosine (ivf.rs:149-185)
static int probe_metric(int metric) { return metric == METRIC_DOT ? METRIC_DOT : METRIC_L2; }

// part_offsets with one more, empty, partition K: the probe id of a slot that searches nothing
static void ext_offsets(const uint64_t* part_offsets, int K, DevBuf<uint64_t>& ext) {
  ext.alloc((size_t)K + 2);
  d2d(ext.p, part_offsets, (size_t)K + 1);
  d2d(ext.p + K + 1, part_offsets + K, 1);
}

// The IVF query skeleton: the np nearest partitions of every query, one candidate list of <= k per (query, probe)
// slot, the lists merged per query.  With per-query probe counts (s.qnp) np is the largest: a query's first qnp[q]
// of its np nearest are its own nearest qnp[q], and its other slots probe the empty partition K; a batch holds its
// candidate lists in sub-slabs of about 256 MB (scan, then merge, per sub-slab).
static void ivf_search(const IvfSearch& s, int np, ScanRef scan) {
  const uint64_t nq = s.nq;
  const int k = s.k;
  const uint64_t per_q = (uint64_t)np * k * 12 + 4ull * np;
  const uint64_t sub = s.qp ? std::max<uint64_t>(1, std::min<uint64_t>(nq, (256ull << 20) / per_q)) : nq;
  DevBuf<uint32_t> pids((size_t)nq * np), cand_cnt((size_t)sub * np);
  DevBuf<float> pd((size_t)nq * np), cand_d((size_t)sub * np * k);
  DevBuf<uint64_t> cand_id((size_t)sub * np * k);
  find_partitions_f32(s.centroids, s.K, s.d, probe_metric(s.metric), s.queries, nq, np, pids.p, pd.p);
  const uint64_t* offsets = s.part_offsets;
  DevBuf<uint64_t> ext;
  DevBuf<uint32_t> own_ids;
  DevBuf<float> own_pd;
  if (s.qnp) {
    ext_offsets(s.part_offsets, s.K, ext);
    own_ids.alloc((size_t)nq * np);
    own_pd.alloc((size_t)nq * np);
    gather_probes(nq, np, pids.p, pd.p, s.qnp, np, (uint32_t)s.K, own_ids.p, own_pd.p);
    std::swap(pids, own_ids);
    std::swap(pd, own_pd);
    offsets = ext.p;
  }
  for (uint64_t a = 0; a < nq; a += sub) {
    const uint64_t b = std::min(sub, nq - a);
    for (uint64_t q0 = a; q0 < a + b; q0 += SEARCH_SLAB) {
      const uint64_t c = q0 - a;  // the query's place in the sub-slab's lists
      scan({q0, std::min<uint64_t>(SEARCH_SLAB, a + b - q0), np, offsets, pids.p + q0 * np, pd.p + q0 * np,
            cand_d.p + c * np * k, cand_id.p + c * np * k, cand_cnt.p + c * np});
    }
    merge_lists("merge_topk", b, cand_d.p, cand_id.p, cand_cnt.p, np, k, (size_t)k, (size_t)k, (size_t)np * k,
                (size_t)1, (size_t)np, s.out_ids + a * k, s.out_dists + a * k, s.out_counts ? s.out_counts + a : nullptr,
                0, s.qp_at(a));
  }
}

// The same skeleton with a per-query probe count (probe.cu): per slab of queries every centroid distance is ranked
// (P = the first L = min(maximum_nprobes or K, K)), the cutoff fixes how many of P each query searches, and the scan
// runs over a grid as wide as the slab's largest count.  A query's slots past its own count hold the partition id K,
// which `ext_offsets` (part_offsets with one more empty partition) makes an empty partition for every scan kernel.
// With a mask the query may answer from (`pr.mask_ids`), every query gets one more slot: the shortcut list.
// With a range bound c_p depends on the distances: all L partitions are scanned, the cutoff reads the scan's list
// counts and empties the lists past it.  Candidate memory is bounded by sub-slabs of about 256 MB.
static void ivf_search_probed(const IvfSearch& s, ScanRef scan) {
  const ProbeRule& pr = *s.pr;
  const uint64_t nq = s.nq;
  const int K = s.K, d = s.d, kc = s.k;
  if (nq == 0) return;
  const int L = pr.max_np ? (int)std::min<uint32_t>(pr.max_np, (uint32_t)K) : K;
  // a batch scans every query's L partitions first when any of its queries has a range; the cutoff then takes a
  // ranged query's c_p from its list counts and every other query's from its prefilter's counts, as its own call does
  const bool by_scan = s.pr->qpr ? s.any_range : s.flt.range != 0;
  const int extra = pr.mask_ids ? 1 : 0;
  DevBuf<uint64_t> ext;
  ext_offsets(s.part_offsets, K, ext);
  DevBuf<uint32_t> cpart;
  if (!by_scan && !pr.qpr) {
    cpart.alloc(K);
    partition_counts(s.part_offsets, K, s.flt.allow, (uint32_t)kc, cpart.p);
  }
  // the ranking's buffers: distances, and two runs of packed words above one tile
  const uint64_t rank_bytes = (uint64_t)K * (K > RANK_TILE ? 20 : 4) + (uint64_t)L * 8;
  const uint64_t qs = std::max<uint64_t>(1, std::min<uint64_t>(SEARCH_SLAB, (256ull << 20) / rank_bytes));
  DevBuf<float> all(std::min(qs, nq) * K), pd(std::min(qs, nq) * L);
  DevBuf<uint32_t> pids(std::min(qs, nq) * L), nsearch(std::min(qs, nq)), shortcut(std::min(qs, nq)), nmax(1);
  for (uint64_t q0 = 0; q0 < nq; q0 += qs) {
    const uint64_t qn = std::min(qs, nq - q0);
    centroid_distances(s.queries + q0 * d, qn, d, s.centroids, K, probe_metric(s.metric), all.p);
    rank_probes(all.p, qn, K, L, pids.p, pd.p);
    uint32_t* nprobes_out = pr.nprobes_out ? pr.nprobes_out + q0 : nullptr;
    const QueryProbe* qpr = pr.qpr ? pr.qpr + q0 : nullptr;
    int np = L;
    if (!by_scan) {
      nmax.zero();
      probe_cutoff(pr, qn, L, pids.p, pd.p, cpart.p, nullptr, 0, nsearch.p, shortcut.p, nmax.p, nprobes_out, qpr);
      uint32_t h = 0;
      d2h(&h, nmax.p, 1);
      sync_stream();
      np = (int)h;
    }
    const int nl = np + extra;  // slots per query
    DevBuf<uint32_t> sp((size_t)qn * nl);
    DevBuf<float> spd((size_t)qn * nl);
    gather_probes(qn, L, pids.p, pd.p, by_scan ? nullptr : nsearch.p, nl, (uint32_t)K, sp.p, spd.p, qpr);
    const uint64_t per_q = (uint64_t)nl * kc * 12 + 4 * (uint64_t)nl;
    const uint64_t sub = std::max<uint64_t>(1, std::min<uint64_t>(qn, (256ull << 20) / per_q));
    DevBuf<float> cd(sub * nl * kc);
    DevBuf<uint64_t> cid(sub * nl * kc);
    DevBuf<uint32_t> ccnt(sub * nl);
    for (uint64_t a = 0; a < qn; a += sub) {
      const uint64_t b = std::min(sub, qn - a);
      scan({q0 + a, b, nl, ext.p, sp.p + a * nl, spd.p + a * nl, cd.p, cid.p, ccnt.p});
      if (by_scan)
        probe_cutoff(pr, b, L, pids.p + a * L, pd.p + a * L, nullptr, ccnt.p, nl, nsearch.p + a, shortcut.p + a,
                     nmax.p, nprobes_out ? nprobes_out + a : nullptr, qpr ? qpr + a : nullptr);
      if (extra)
        shortcut_lists(b, shortcut.p + a, pr.mask_ids, pr.num_mask_ids, nl, kc, cd.p, cid.p, ccnt.p,
                       qpr ? qpr + a : nullptr);
      merge_lists("merge_topk", b, cd.p, cid.p, ccnt.p, nl, kc, (size_t)kc, (size_t)kc, (size_t)nl * kc, (size_t)1,
                  (size_t)nl, s.out_ids + (q0 + a) * kc, s.out_dists + (q0 + a) * kc,
                  s.out_counts ? s.out_counts + q0 + a : nullptr, 0, s.qp_at(q0 + a));
    }
  }
}

void run_ivf_search(const IvfSearch& s, ScanRef scan) {
  if (s.pr)
    ivf_search_probed(s, scan);
  else
    ivf_search(s, s.nprobes < s.K ? s.nprobes : s.K, scan);
}

bool ivf_search_begin(const IvfSearch& s, size_t need, const char* refusal, size_t refusal_arg) {
  if (s.nq == 0 || s.k == 0) return false;
  if (s.k > 1024) fail(LB2_UNSUPPORTED, "k (incl. refine factor) > 1024 is not implemented");
  if (need > ctx().smem_optin) fail(LB2_UNSUPPORTED, refusal, refusal_arg);
  return true;
}

// Row-sharded index (SURVEY 8e search (ii)): every rank has searched its own shard; the per-rank top-k lists
// are exchanged in ONE collective and merged on every rank by (_distance, _rowid), the order of the
// reference's final SortExec (rust/lance/src/dataset/scanner.rs:3450-3466).  ids / dists / counts: this
// rank's [nq][k] / [nq] results on the device; outputs likewise.
void merge_sharded_topk(const uint64_t* ids, const float* dists, const uint32_t* counts, uint64_t nq, int k,
                        uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
  Comm* c = current_comm();
  const int nr = c ? c->nranks : 1;
  const size_t id_bytes = (size_t)nq * k * 8, d_bytes = ((size_t)nq * k * 4 + 7) / 8 * 8, c_bytes = ((size_t)nq * 4 + 7) / 8 * 8;
  const size_t S = id_bytes + d_bytes + c_bytes;
  DevBuf<uint8_t> blob(S), gathered(S * nr);
  LB2_CUDA(cudaMemcpyAsync(blob.p, ids, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, ctx().stream));
  LB2_CUDA(cudaMemcpyAsync(blob.p + id_bytes, dists, (size_t)nq * k * 4, cudaMemcpyDeviceToDevice, ctx().stream));
  LB2_CUDA(cudaMemcpyAsync(blob.p + id_bytes + d_bytes, counts, (size_t)nq * 4, cudaMemcpyDeviceToDevice, ctx().stream));
  comm_allgather_bytes(blob.p, gathered.p, S);
  merge_lists("merge_sharded_topk", nq, reinterpret_cast<const float*>(gathered.p + id_bytes),
              reinterpret_cast<const uint64_t*>(gathered.p), reinterpret_cast<const uint32_t*>(gathered.p + id_bytes + d_bytes),
              nr, k, S / 4, S / 8, (size_t)k, S / 4, (size_t)1, out_ids, out_dists, out_counts);
  sync_stream();  // the exchange buffers are freed on return
}

}  // namespace lb2
