// topk.cuh -- the exact top-k of one slot (one (query, probed partition) pair, or one distance array), for every
// kernel that selects: a scan includes this header, writes a fill step that turns rows into order keys, and calls
// slot_topk.  Also the ordered emission (emit_ascending) the probe selection, the merges and the refine use.
//
// Replaces  FlatIndex::search heap top-k         lance-index/src/vector/flat/index.rs:82-177
//
// Everything here is __forceinline__, inline or a template and declares its __shared__ scratch itself: the library
// is built without relocatable device code, so each kernel gets its own copy.
#pragma once
#include <stdint.h>

#include "exact.cuh"
#include "ivf_search.cuh"

namespace lb2 {

// prefilter (PreFilter::mask, lance-index/src/prefilter.rs:27-51; FlatIndex::search :129-165): one bit
// per STORAGE position (partition-sorted order); a cleared bit removes the row from the scan.  Filtered
// rows get the maximal key, so they can only surface when fewer than k allowed rows exist, and the
// output stage drops them by re-testing the bit.
__device__ __forceinline__ bool row_allowed(const uint64_t* __restrict__ allow, uint64_t pos) {
  return allow == nullptr || ((allow[pos >> 6] >> (pos & 63)) & 1ull) != 0;
}
// range query (flat/index.rs:100-115): a row enters the heap iff lower <= dist < upper in f32::total_cmp
// order; an absent bound is f32::MIN / f32::MAX (NOT -inf / +inf), exactly as the reference unwraps them
__device__ __forceinline__ bool key_in_range(const ScanFilter& f, int32_t key) {
  return !f.range || (key >= f.lo_key && key < f.hi_key);
}

// ---- Rust std BinaryHeap<OrderedNode> restated (alloc::collections::binary_heap: push = sift_up,
// pop = swap with the last + sift_down_to_bottom + sift_up) on (unsigned order key, position) pairs.
// OrderedNode compares by distance only (graph.rs:117-121), so WHICH of several rows tied at the k-th
// distance survives FlatIndex::search's `if root.dist > dist { pop; push }` loop (flat/index.rs:116-126)
// depends on this exact sift order.  The parallel selections below return the k smallest (distance,
// position) pairs, which is the same SET unless more rows tie at the k-th distance than fit; exactly
// then (detected by selecting k + 1) the slot is replayed sequentially through this heap.
__device__ __forceinline__ void rheap_sift_up(uint32_t* hk, uint32_t* hp, uint32_t pos) {
  const uint32_t ek = hk[pos], ep = hp[pos];
  while (pos > 0) {
    const uint32_t parent = (pos - 1) >> 1;
    if (ek <= hk[parent]) break;
    hk[pos] = hk[parent];
    hp[pos] = hp[parent];
    pos = parent;
  }
  hk[pos] = ek;
  hp[pos] = ep;
}
__device__ __forceinline__ void rheap_push(uint32_t* hk, uint32_t* hp, uint32_t& len, uint32_t key, uint32_t pos) {
  hk[len] = key;
  hp[len] = pos;
  rheap_sift_up(hk, hp, len);
  ++len;
}
__device__ __forceinline__ void rheap_pop(uint32_t* hk, uint32_t* hp, uint32_t& len) {
  --len;
  if (len == 0) return;
  const uint32_t ek = hk[len], ep = hp[len];  // the last element moves to the root, then sinks to the bottom
  uint32_t pos = 0, child = 1;
  const uint32_t end = len;
  while (child + 1 < end) {
    if (hk[child] <= hk[child + 1]) child += 1;
    hk[pos] = hk[child];
    hp[pos] = hp[child];
    pos = child;
    child = 2 * pos + 1;
  }
  if (child + 1 == end) {
    hk[pos] = hk[child];
    hp[pos] = hp[child];
    pos = child;
  }
  hk[pos] = ek;
  hp[pos] = ep;
  rheap_sift_up(hk, hp, pos);
}
// BinaryHeap::into_sorted_vec: the heap sort (swap the root with the last, then sift_down_range(0, end)); the
// heap's arrays end ascending, and the order among equal keys is the reference's
__device__ __forceinline__ void rheap_into_sorted(uint32_t* hk, uint32_t* hp, uint32_t len) {
  for (uint32_t end = len; end > 1;) {
    --end;
    const uint32_t ek = hk[end], ep = hp[end];
    hk[end] = hk[0];
    hp[end] = hp[0];
    uint32_t pos = 0, child = 1;
    bool placed = false;
    while (child + 1 < end) {
      if (hk[child] <= hk[child + 1]) child += 1;
      if (ek >= hk[child]) { placed = true; break; }
      hk[pos] = hk[child];
      hp[pos] = hp[child];
      pos = child;
      child = 2 * pos + 1;
    }
    if (!placed && child + 1 == end && ek < hk[child]) {
      hk[pos] = hk[child];
      hp[pos] = hp[child];
      pos = child;
    }
    hk[pos] = ek;
    hp[pos] = ep;
  }
}
// FlatIndex::search's insertion rule for one row (flat/index.rs:116-126); keys are unsigned order keys
__device__ __forceinline__ void rheap_offer(uint32_t* hk, uint32_t* hp, uint32_t& len, uint32_t k, uint32_t key,
                                            uint32_t pos) {
  if (len < k) {
    rheap_push(hk, hp, len, key, pos);
  } else if (hk[0] > key) {
    rheap_pop(hk, hp, len);
    rheap_push(hk, hp, len, key, pos);
  }
}

// ------------------------------------------------------------------------------------------------
// block-level helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool ki_less(int32_t k1, uint64_t i1, int32_t k2, uint64_t i2) {
  return k1 < k2 || (k1 == k2 && i1 < i2);
}

// argmin over (key, tie) proposed by every thread of a 256/128-thread block; returns the winning
// thread id (all threads get it).  Threads with nothing to propose pass has=false.
template <int NT>
__device__ inline int block_argmin(bool has, int32_t key, uint64_t tie, int32_t* s_key,
                                   uint64_t* s_tie, int* s_tid) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int who = has ? tid : -1;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const int32_t ok = __shfl_xor_sync(0xffffffffu, key, off);
    const uint64_t ot = __shfl_xor_sync(0xffffffffu, tie, off);
    const int ow = __shfl_xor_sync(0xffffffffu, who, off);
    if (ow >= 0 && (who < 0 || ki_less(ok, ot, key, tie))) {
      key = ok; tie = ot; who = ow;
    }
  }
  if (lane == 0) { s_key[warp] = key; s_tie[warp] = tie; s_tid[warp] = who; }
  __syncthreads();
  if (tid == 0) {
    int bw = s_tid[0];
    int32_t bk = s_key[0];
    uint64_t bt = s_tie[0];
    for (int w = 1; w < NT / 32; ++w)
      if (s_tid[w] >= 0 && (bw < 0 || ki_less(s_key[w], s_tie[w], bk, bt))) {
        bw = s_tid[w]; bk = s_key[w]; bt = s_tie[w];
      }
    s_tid[NT / 32] = bw;
  }
  __syncthreads();
  const int winner = s_tid[NT / 32];
  __syncthreads();
  return winner;
}

// Ordered emission: round r finds the smallest (key, tie) strictly after round r - 1's among the candidates
// i in [0, n) for which cand(i, key, tie) returns true, and emit(r, i, key, tie) runs on the thread that proposed
// it.  Stops after `rounds` rounds or when no candidate is left; returns the number of rounds that emitted.
template <int NT, class Cand, class Emit>
__device__ __forceinline__ uint32_t emit_ascending(uint32_t rounds, uint32_t n, Cand cand, Emit emit) {
  __shared__ int32_t s_key[NT / 32];
  __shared__ uint64_t s_tie[NT / 32];
  __shared__ int s_tid[NT / 32 + 1];
  __shared__ int32_t prev_key;
  __shared__ uint64_t prev_tie;
  const int tid = threadIdx.x;
  uint32_t r = 0;
  for (; r < rounds; ++r) {
    int32_t bk = 0;
    uint64_t bt = 0;
    uint32_t bi = 0;
    bool has = false;
    const int32_t pk = r ? prev_key : 0;
    const uint64_t pt = r ? prev_tie : 0;
    for (uint32_t i = tid; i < n; i += NT) {
      int32_t key;
      uint64_t tie;
      if (!cand(i, key, tie) || (r && !ki_less(pk, pt, key, tie))) continue;  // none, or already emitted
      if (!has || ki_less(key, tie, bk, bt)) { bk = key; bt = tie; bi = i; has = true; }
    }
    const int w = block_argmin<NT>(has, bk, bt, s_key, s_tie, s_tid);
    if (w < 0) break;
    if (tid == w) {
      prev_key = bk;
      prev_tie = bt;
      emit(r, bi, bk, bt);
    }
    __syncthreads();
  }
  return r;
}

// rows whose keys a slot holds in shared memory at a time; the winners of a chunk join the next chunk's candidate pool
constexpr int SCAN_CHUNK = 4096;

__device__ __forceinline__ float key_to_float(int32_t key) {
  return __int_as_float(key ^ (int32_t)((uint32_t)(key >> 31) >> 1));
}

// ------------------------------------------------------------------------------------------------
// Exact top-k of one slot (16 < k <= 1024 in the PQ scan, every k in the IVF_FLAT scan and lb2_flat_topk), 256
// threads.  A row's distance is an unsigned order key (unsigned order == f32::total_cmp order); the caller's fill
// step writes the keys of rows [c0, c0 + clen) to ukey.  Per chunk of SCAN_CHUNK rows the kk = k + 1 smallest
// (key, position) pairs of the chunk and the winners carried from earlier chunks are found by a 4-pass MSB radix
// select over shared-memory keys (256-bin histograms): everything below the kk-th key is kept, ties AT it are
// resolved by position (earliest rows survive).  Selecting one more than asked for exposes ties that overflow the
// k-th place; those slots are replayed through the reference's heap.
// ------------------------------------------------------------------------------------------------
// shared memory of one slot (u32 words): ukey[SCAN_CHUNK + kk] (a chunk's keys, then the carried winners' keys),
// cpos[kk] (the carried winners' positions), nkey[kk] / npos[kk] (the next winners; the result; the replay heap)
__host__ __device__ constexpr size_t slot_smem_bytes(int k) {
  return sizeof(uint32_t) * (SCAN_CHUNK + 4 * (size_t)(k + 1));
}
struct SlotSmem {
  uint32_t *ukey, *cpos, *nkey, *npos;
  __device__ SlotSmem(void* base, int kk)
      : ukey(static_cast<uint32_t*>(base)), cpos(ukey + SCAN_CHUNK + kk), nkey(cpos + kk), npos(nkey + kk) {}
};

// a row the prefilter (bit at off + row) or the range removes
__device__ __forceinline__ bool slot_excluded(const ScanFilter& f, uint64_t off, uint32_t row, uint32_t ukey) {
  return !row_allowed(f.allow, off + row) || !key_in_range(f, (int32_t)(ukey ^ 0x80000000u));
}

// The kk smallest (key, position) pairs of rows [0, n); excluded rows take the maximal key, so they only surface when
// fewer than kk rows are left.  Returns their number; they are left unordered at ukey[SCAN_CHUNK ..) / cpos.
// max_admitted: some admitted row has the maximal key too (a NaN distance), so it ties with the excluded rows.
template <class Fill>
__device__ __forceinline__ uint32_t slot_select(const SlotSmem& s, uint32_t n, uint32_t kk, const ScanFilter& flt, uint64_t off,
                                Fill fill, bool& max_admitted) {
  __shared__ uint32_t hist[256], s_wsum[8];
  __shared__ uint32_t s_prefix, s_need, s_eq, s_out, s_maxadm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool filtering = flt.allow != nullptr || flt.range;
  uint32_t nw = 0;
  // once kk winners are carried, a chunk row whose key is >= lim (>= the kk-th carried key) cannot enter: kk
  // carried winners precede it in (key, position) order.  Such rows are left out of the pool.
  uint32_t lim = 0xffffffffu;
  bool full = false;
  if (tid == 0) s_maxadm = 0;  // ordered before any store by the barrier after the first fill
  for (uint32_t c0 = 0; c0 < n; c0 += SCAN_CHUNK) {
    const uint32_t clen = min((uint32_t)SCAN_CHUNK, n - c0);
    fill(c0, clen);
    __syncthreads();
    if (filtering) {
      for (uint32_t j = tid; j < clen; j += 256) {
        if (slot_excluded(flt, off, c0 + j, s.ukey[j])) s.ukey[j] = 0xffffffffu;
        else if (s.ukey[j] == 0xffffffffu) s_maxadm = 1;
      }
      __syncthreads();
    }
    // pool element i: i < clen -> (ukey[i], c0 + i), else the carried winner i - clen at ukey[SCAN_CHUNK ..)
    const uint32_t pool = clen + nw;
    auto key_at = [&](uint32_t i) { return i < clen ? s.ukey[i] : s.ukey[SCAN_CHUNK + (i - clen)]; };
    auto pos_at = [&](uint32_t i) { return i < clen ? c0 + i : s.cpos[i - clen]; };
    auto pooled = [&](uint32_t i, uint32_t kv) { return !full || i >= clen || kv < lim; };
    if (pool <= kk) {
      for (uint32_t i = tid; i < pool; i += 256) { s.nkey[i] = key_at(i); s.npos[i] = pos_at(i); }
      __syncthreads();
      for (uint32_t i = tid; i < pool; i += 256) { s.ukey[SCAN_CHUNK + i] = s.nkey[i]; s.cpos[i] = s.npos[i]; }
      nw = pool;
      full = nw == kk;
      __syncthreads();
      continue;
    }
    if (tid == 0) { s_prefix = 0; s_need = kk; }
    uint32_t mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
      hist[tid] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix, need = s_need;
      for (uint32_t i = tid; i < pool; i += 256) {
        const uint32_t kv = key_at(i);
        if (pooled(i, kv) && (kv & mask) == prefix) atomicAdd(&hist[(kv >> shift) & 255u], 1u);
      }
      __syncthreads();
      // the bin of the need-th key: the one whose inclusive prefix sum first reaches `need` (bin = thread)
      const uint32_t h = hist[tid];
      uint32_t cum = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, cum, o);
        if (lane >= o) cum += v;
      }
      if (lane == 31) s_wsum[warp] = cum;
      __syncthreads();
      for (int w = 0; w < warp; ++w) cum += s_wsum[w];
      if (cum >= need && cum - h < need) {
        s_need = need - (cum - h);
        s_prefix = prefix | ((uint32_t)tid << shift);
        s_eq = h;
      }
      mask |= 0xffu << shift;
      __syncthreads();
    }
    const uint32_t T = s_prefix, need = s_need, eq = s_eq;  // take all keys < T and `need` of the `eq` keys == T
    if (tid == 0) s_out = 0;
    __syncthreads();
    for (uint32_t i = tid; i < pool; i += 256) {
      const uint32_t kv = key_at(i);
      if (pooled(i, kv) && (kv < T || (kv == T && eq == need))) {
        const uint32_t at = atomicAdd(&s_out, 1u);
        s.nkey[at] = kv;
        s.npos[at] = pos_at(i);
      }
    }
    __syncthreads();
    if (eq != need)  // ties at the last key: the `need` smallest positions survive (rare)
      emit_ascending<256>(
          need, pool,
          [&](uint32_t i, int32_t& key, uint64_t& tie) {
            const uint32_t kv = key_at(i);
            key = 0;
            tie = pos_at(i);
            return kv == T && pooled(i, kv);
          },
          [&](uint32_t, uint32_t, int32_t, uint64_t tie) {
            const uint32_t at = s_out;
            s.nkey[at] = T;
            s.npos[at] = (uint32_t)tie;
            s_out = at + 1;
          });
    const uint32_t got = s_out;  // == kk
    __syncthreads();
    for (uint32_t i = tid; i < got; i += 256) { s.ukey[SCAN_CHUNK + i] = s.nkey[i]; s.cpos[i] = s.npos[i]; }
    nw = got;
    full = true;
    lim = T;
    __syncthreads();
  }
  max_admitted = n > 0 && s_maxadm != 0;  // every pass of the loop ends in a barrier
  return nw;
}

// The finish, on the nw <= kk winners in (key, position) order: excluded winners at the end are dropped (they carry
// the maximal key; an admitted row whose key is the maximal one, e.g. a NaN distance, keeps the excluded winners before
// it).  If kk winners remain and the last two share a key, more rows tie at the k-th distance than fit and the
// reference's heap decides: returns false.  So it does when excluded winners were dropped from the end of a full
// selection while an admitted row shares their key (max_admitted): admitted rows behind the kk may then belong in the
// result.  Otherwise leaves the admitted winners among the first k at nkey / npos (unordered), sets *cnt and returns
// true.
__device__ __forceinline__ bool slot_finish(const SlotSmem& s, uint32_t nw, uint32_t kk, bool max_admitted,
                            const ScanFilter& flt, uint64_t off, uint32_t* cnt) {
  __shared__ uint32_t s_kept, s_max, s_maxcnt, s_last, s_mid, s_out;
  const int tid = threadIdx.x;
  if (tid == 0) { s_kept = 0; s_max = 0; s_maxcnt = 0; s_last = 0; s_mid = 0; s_out = 0; }
  __syncthreads();
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key)) continue;
    atomicAdd(&s_kept, 1u);
    atomicMax(&s_max, key);
    if (key == 0xffffffffu) atomicMax(&s_last, pos + 1);  // 1 + the last admitted position at the maximal key
  }
  __syncthreads();
  const uint32_t mx = s_max, last = s_last;
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key)) {
      if (pos + 1 < last) atomicAdd(&s_mid, 1u);  // excluded, but in front of an admitted winner
    } else if (key == mx) {
      atomicAdd(&s_maxcnt, 1u);
    }
  }
  __syncthreads();
  const uint32_t kept = s_kept, mid = s_mid;
  const bool at_k = kept + mid == kk;
  if (at_k && s_maxcnt + mid >= 2) return false;  // block-uniform
  if (nw == kk && !at_k && max_admitted) return false;
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key) || (at_k && key == mx)) continue;  // at_k: the (k+1)-th is the unique max
    const uint32_t at = atomicAdd(&s_out, 1u);
    s.nkey[at] = key;
    s.npos[at] = pos;
  }
  __syncthreads();
  *cnt = s_out;
  return true;
}

// The reference's own loop (flat/index.rs:116-165): rows in storage order, keys filled one chunk ahead of the single
// thread that drives the heap.  Leaves the heap's content at nkey / npos and returns its size.
template <class Fill>
__device__ __forceinline__ uint32_t slot_replay(const SlotSmem& s, uint32_t n, uint32_t k, const ScanFilter& flt, uint64_t off,
                                Fill fill) {
  __shared__ uint32_t s_len;
  const bool filtering = flt.allow != nullptr || flt.range;
  uint32_t len = 0;
  for (uint32_t c0 = 0; c0 < n; c0 += SCAN_CHUNK) {
    const uint32_t clen = min((uint32_t)SCAN_CHUNK, n - c0);
    fill(c0, clen);
    __syncthreads();
    if (threadIdx.x == 0) {
      for (uint32_t j = 0; j < clen; ++j) {
        const uint32_t key = s.ukey[j];
        if (filtering && slot_excluded(flt, off, c0 + j, key)) continue;
        rheap_offer(s.nkey, s.npos, len, k, key, c0 + j);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) s_len = len;
  __syncthreads();
  return s_len;
}

// The exact top-k of a slot of n rows: <= k winners at nkey / npos (unordered); returns their number.  replay: go
// straight to the heap loop.
template <class Fill>
__device__ __forceinline__ uint32_t slot_topk(const SlotSmem& s, uint32_t n, int k, const ScanFilter& flt, uint64_t off, bool replay,
                              Fill fill) {
  if (!replay) {
    uint32_t cnt;
    bool max_admitted;
    const uint32_t nw = slot_select(s, n, k + 1, flt, off, fill, max_admitted);
    if (slot_finish(s, nw, k + 1, max_admitted, flt, off, &cnt)) return cnt;
    __syncthreads();
  }
  return slot_replay(s, n, k, flt, off, fill);
}

// a slot's winners -> its candidate list (unordered)
__device__ __forceinline__ void write_slot(const SlotSmem& s, uint32_t cnt, size_t slot, int k, uint64_t off,
                                           const uint64_t* __restrict__ row_ids, float* __restrict__ cand_d,
                                           uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt) {
  for (uint32_t i = threadIdx.x; i < cnt; i += 256) {
    cand_d[slot * k + i] = key_to_float((int32_t)(s.nkey[i] ^ 0x80000000u));
    cand_id[slot * k + i] = row_ids[off + s.npos[i]];
  }
  if (threadIdx.x == 0) cand_cnt[slot] = cnt;
}

// the partition slot (query blockIdx.y, or qlist[blockIdx.y] for a grid over a group of queries; probe blockIdx.x)
// scans: false, with an empty candidate list, when it has no rows
__device__ __forceinline__ bool slot_partition(const uint32_t* __restrict__ probe_ids, int np,
                                               const uint64_t* __restrict__ part_offsets, uint32_t* __restrict__ cand_cnt,
                                               size_t& qi, size_t& slot, uint32_t& p, uint64_t& off, uint32_t& n_p,
                                               const uint32_t* __restrict__ qlist = nullptr) {
  const int pi = blockIdx.x;
  qi = qlist ? qlist[blockIdx.y] : blockIdx.y;
  p = probe_ids[qi * np + pi];
  off = part_offsets[p];
  n_p = (uint32_t)(part_offsets[p + 1] - off);
  slot = qi * np + pi;
  if (n_p == 0) {
    if (threadIdx.x == 0) cand_cnt[slot] = 0;
    return false;
  }
  return true;
}

// the k' and the filter of query qi (slab-relative): its own with per-query values (qp, of the slab), else the search's
__device__ __forceinline__ int query_k(const QueryParam* __restrict__ qp, size_t qi, int k) { return qp ? qp[qi].k : k; }
__device__ __forceinline__ ScanFilter query_filter(const QueryParam* __restrict__ qp, size_t qi, const ScanFilter& f) {
  return qp ? qp[qi].flt : f;
}

}  // namespace lb2
