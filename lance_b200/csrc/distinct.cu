// distinct.cu -- the distinct row ids of a batch's candidate lists and every slot's position among them
// (lb2_index_search_candidates): one radix sort and one unique over the batch's slots, then a binary search per slot.
// The caller takes each distinct row once, in row-address order.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <climits>

#include "common.cuh"
#include "scan.cuh"

namespace lb2 {

// m = the unique count without the UINT64_MAX of the unused slots (the largest key, so the last if present)
__global__ void distinct_count_kernel(const uint64_t* __restrict__ distinct, const int64_t* __restrict__ nsel,
                                      uint64_t* __restrict__ m) {
  const int64_t s = *nsel;
  *m = (uint64_t)s - (s > 0 && distinct[s - 1] == ~0ull ? 1 : 0);
}

// the sort keys: values at or above limit are unused slots, as UINT64_MAX
__global__ void distinct_keys_kernel(const uint64_t* __restrict__ ids, uint64_t n, uint64_t limit,
                                     uint64_t* __restrict__ keys) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = ids[i] < limit ? ids[i] : ~0ull;
}

__global__ void distinct_positions_kernel(const uint64_t* __restrict__ ids, uint64_t n,
                                          const uint64_t* __restrict__ distinct, const uint64_t* __restrict__ m,
                                          uint64_t* __restrict__ positions) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t v = ids[i];
  if (v == ~0ull) {
    positions[i] = ~0ull;
    return;
  }
  uint64_t lo = 0, hi = *m;  // v is one of them
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (distinct[mid] < v) lo = mid + 1; else hi = mid;
  }
  positions[i] = lo;
}

void distinct_ids(const uint64_t* ids, uint64_t n, uint64_t* distinct, uint64_t* num_distinct, uint64_t* positions,
                  uint64_t limit) {
  if (n > (uint64_t)INT_MAX) fail(LB2_UNSUPPORTED, "%llu candidate slots: more than 2^31 - 1 is not implemented",
                                  (unsigned long long)n);
  cudaStream_t st = ctx().stream;
  LB2_CUDA(cudaMemsetAsync(distinct, 0xff, n * sizeof(uint64_t), st));
  if (n == 0) {
    LB2_CUDA(cudaMemsetAsync(num_distinct, 0, sizeof(uint64_t), st));
    return;
  }
  DevBuf<uint64_t> keys(n), sorted(n);
  LB2_LAUNCH("distinct_keys", distinct_keys_kernel, cdiv(n, 256), 256, 0, ids, n, limit, keys.p);
  ids = keys.p;
  DevBuf<int64_t> nsel(1);
  size_t sort_bytes = 0, uniq_bytes = 0;
  LB2_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, ids, sorted.p, (int)n, 0, 64, st));
  LB2_CUDA(cub::DeviceSelect::Unique(nullptr, uniq_bytes, sorted.p, distinct, nsel.p, (int)n, st));
  DevBuf<uint8_t> tmp(std::max(sort_bytes, uniq_bytes));
  {
    LaunchScope ls("distinct_sort");
    LB2_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, sort_bytes, ids, sorted.p, (int)n, 0, 64, st));
  }
  {
    LaunchScope ls("distinct_unique");
    LB2_CUDA(cub::DeviceSelect::Unique(tmp.p, uniq_bytes, sorted.p, distinct, nsel.p, (int)n, st));
  }
  LB2_LAUNCH("distinct_count", distinct_count_kernel, 1, 1, 0, distinct, nsel.p, num_distinct);
  LB2_LAUNCH("distinct_positions", distinct_positions_kernel, cdiv(n, 256), 256, 0, ids, n, distinct, num_distinct,
             positions);
}

}  // namespace lb2
