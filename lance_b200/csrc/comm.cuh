// comm.cuh -- optional multi-GPU communicator (one process per GPU).  NCCL is loaded with dlopen at
// lb2_comm_init time so that liblance_b200.so has no hard NCCL dependency.
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"
namespace lb2 {
struct Comm {
  void* handle = nullptr;  // ncclComm_t
  int rank = 0, nranks = 1;
};
Comm* current_comm();  // nullptr when lb2_comm_init has not been called on this thread
Comm* comm_swap(Comm* c);  // install c (may be nullptr) as this thread's communicator, return the previous one
// rank count of the current communicator (1 without one)
inline uint64_t comm_nranks() { const Comm* c = current_comm(); return c ? c->nranks : 1; }
enum class RedOp { Sum, Max };
// in-place all-reduce on the library's stream
void comm_allreduce_f32(float* buf, size_t count, RedOp op);
void comm_allreduce_f64(double* buf, size_t count, RedOp op);
void comm_allreduce_u32(uint32_t* buf, size_t count, RedOp op);
void comm_broadcast_bytes(void* buf, size_t bytes, int root);
// out[r * bytes ..] = rank r's `in`: one collective whose result every rank reduces in the same (rank) order
void comm_allgather_bytes(const void* in, void* out, size_t bytes);
// this rank's bytes for peer r: send + send_off[r] (send_bytes[r]); peer r's bytes land at recv + recv_off[r]
void comm_alltoallv_bytes(const void* send, const size_t* send_off, const size_t* send_bytes, void* recv,
                          const size_t* recv_off, const size_t* recv_bytes);
// element-wise sum of a few host-side counters over the ranks of the current communicator (identity on one GPU)
void sum_over_ranks(std::vector<uint32_t>& v);
}  // namespace lb2
