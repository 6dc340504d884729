// comm.cu -- NCCL plumbing for the sharded k-means (SURVEY.md section 8e): every rank holds a row
// shard of the training sample, the per-cluster partial sums / counts / losses are all-reduced over
// NVLink once per Lloyd iteration, and every rank then applies the same deterministic epilogue.
#include "comm.cuh"

#include <dlfcn.h>

namespace lb2 {

namespace {
// minimal NCCL ABI (nccl.h): only what we call
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclSuccess = 0 };
enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5,
       ncclFloat16 = 6, ncclFloat32 = 7, ncclFloat64 = 8 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 };

struct Api {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
Api& api() {
  static Api a;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      a.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (a.lib) break;
    }
    if (!a.lib) return;
    a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(a.lib, "ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))dlsym(a.lib, "ncclCommInitRank");
    a.CommDestroy = (decltype(a.CommDestroy))dlsym(a.lib, "ncclCommDestroy");
    a.AllReduce = (decltype(a.AllReduce))dlsym(a.lib, "ncclAllReduce");
    a.Broadcast = (decltype(a.Broadcast))dlsym(a.lib, "ncclBroadcast");
    a.AllGather = (decltype(a.AllGather))dlsym(a.lib, "ncclAllGather");
    a.Send = (decltype(a.Send))dlsym(a.lib, "ncclSend");
    a.Recv = (decltype(a.Recv))dlsym(a.lib, "ncclRecv");
    a.GroupStart = (decltype(a.GroupStart))dlsym(a.lib, "ncclGroupStart");
    a.GroupEnd = (decltype(a.GroupEnd))dlsym(a.lib, "ncclGroupEnd");
    a.GetErrorString = (decltype(a.GetErrorString))dlsym(a.lib, "ncclGetErrorString");
  });
  if (!a.lib || !a.GetUniqueId || !a.CommInitRank || !a.AllReduce || !a.Broadcast || !a.AllGather)
    fail(LB2_NCCL_ERROR, "NCCL (libnccl.so.2) could not be loaded: %s", dlerror() ? dlerror() : "missing symbols");
  return a;
}
void nccl_check(ncclResult_t r, const char* what) {
  if (r != ncclSuccess)
    fail(LB2_NCCL_ERROR, "%s failed: %s", what, api().GetErrorString ? api().GetErrorString(r) : "nccl error");
}
thread_local Comm* g_comm = nullptr;
}  // namespace

Comm* current_comm() { return g_comm; }
Comm* comm_swap(Comm* c) {
  Comm* prev = g_comm;
  g_comm = c;
  return prev;
}

static void allreduce(void* buf, size_t count, int dtype, RedOp op) {
  Comm* c = g_comm;
  if (!c || c->nranks <= 1 || count == 0) return;
  nccl_check(api().AllReduce(buf, buf, count, dtype, op == RedOp::Sum ? ncclSum : ncclMax,
                             (ncclComm_t)c->handle, ctx().stream), "ncclAllReduce");
  ctx().launches++;  // NCCL's reduction kernel
}
void comm_allreduce_f32(float* buf, size_t count, RedOp op) { allreduce(buf, count, ncclFloat32, op); }
void comm_allreduce_f64(double* buf, size_t count, RedOp op) { allreduce(buf, count, ncclFloat64, op); }
void comm_allreduce_u32(uint32_t* buf, size_t count, RedOp op) { allreduce(buf, count, ncclUint32, op); }
// out[r * bytes ..] = rank r's `in` (every rank ends with the same buffer, in rank order)
void comm_allgather_bytes(const void* in, void* out, size_t bytes) {
  Comm* c = g_comm;
  if (!c || c->nranks <= 1 || bytes == 0) {
    if (bytes && in != out) LB2_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, ctx().stream));
    return;
  }
  nccl_check(api().AllGather(in, out, bytes, ncclUint8, (ncclComm_t)c->handle, ctx().stream), "ncclAllGather");
  ctx().launches++;
}
// all-to-all with per-peer sizes (one grouped send/recv over NVLink): this rank's bytes for peer r start at
// send + send_off[r], the bytes from peer r land at recv + recv_off[r]
void comm_alltoallv_bytes(const void* send, const size_t* send_off, const size_t* send_bytes, void* recv,
                          const size_t* recv_off, const size_t* recv_bytes) {
  Comm* c = g_comm;
  const int G = c ? c->nranks : 1, me = c ? c->rank : 0;
  if (G <= 1) {
    if (send_bytes[0])
      LB2_CUDA(cudaMemcpyAsync((char*)recv + recv_off[0], (const char*)send + send_off[0], send_bytes[0],
                               cudaMemcpyDeviceToDevice, ctx().stream));
    return;
  }
  if (!api().Send || !api().Recv || !api().GroupStart || !api().GroupEnd)
    fail(LB2_NCCL_ERROR, "this NCCL has no ncclSend / ncclRecv");
  nccl_check(api().GroupStart(), "ncclGroupStart");
  for (int r = 0; r < G; ++r) {
    if (r == me) continue;
    if (send_bytes[r])
      nccl_check(api().Send((const char*)send + send_off[r], send_bytes[r], ncclUint8, r, (ncclComm_t)c->handle, ctx().stream), "ncclSend");
    if (recv_bytes[r])
      nccl_check(api().Recv((char*)recv + recv_off[r], recv_bytes[r], ncclUint8, r, (ncclComm_t)c->handle, ctx().stream), "ncclRecv");
  }
  nccl_check(api().GroupEnd(), "ncclGroupEnd");
  if (send_bytes[me])
    LB2_CUDA(cudaMemcpyAsync((char*)recv + recv_off[me], (const char*)send + send_off[me], send_bytes[me],
                             cudaMemcpyDeviceToDevice, ctx().stream));
  ctx().launches++;
}
void comm_broadcast_bytes(void* buf, size_t bytes, int root) {
  Comm* c = g_comm;
  if (!c || c->nranks <= 1 || bytes == 0) return;
  nccl_check(api().Broadcast(buf, buf, bytes, ncclUint8, root, (ncclComm_t)c->handle, ctx().stream), "ncclBroadcast");
}
void sum_over_ranks(std::vector<uint32_t>& v) {
  Comm* cm = current_comm();
  if (!cm || cm->nranks <= 1 || v.empty()) return;
  DevBuf<uint32_t> d(v.size());
  h2d(d.p, v.data(), v.size());
  comm_allreduce_u32(d.p, v.size(), RedOp::Sum);
  d2h(v.data(), d.p, v.size());
  sync_stream();
}

}  // namespace lb2

using namespace lb2;

extern "C" {

lb2_status lb2_comm_unique_id(void* unique_id_128) {
  LB2_API_BEGIN
  LB2_REQUIRE(unique_id_128, "null argument");
  ncclUniqueId id;
  nccl_check(api().GetUniqueId(&id), "ncclGetUniqueId");
  memcpy(unique_id_128, &id, sizeof(id));
  LB2_API_END
}

lb2_status lb2_comm_init(const void* unique_id_128, int rank, int nranks) {
  LB2_API_BEGIN
  LB2_REQUIRE(unique_id_128 && nranks >= 1 && rank >= 0 && rank < nranks, "bad communicator arguments");
  ctx();
  if (g_comm) fail(LB2_INVALID_ARG, "communicator already initialised on this thread");
  ncclUniqueId id;
  memcpy(&id, unique_id_128, sizeof(id));
  ncclComm_t comm = nullptr;
  nccl_check(api().CommInitRank(&comm, nranks, id, rank), "ncclCommInitRank");
  g_comm = new Comm();
  g_comm->handle = comm;
  g_comm->rank = rank;
  g_comm->nranks = nranks;
  LB2_API_END
}

lb2_status lb2_comm_destroy(void) {
  LB2_API_BEGIN
  if (g_comm) {
    sync_stream();
    if (api().CommDestroy) api().CommDestroy((ncclComm_t)g_comm->handle);
    delete g_comm;
    g_comm = nullptr;
  }
  LB2_API_END
}

}  // extern "C"
