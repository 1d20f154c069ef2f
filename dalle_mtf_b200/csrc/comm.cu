// D1 — hand-driven NCCL behind the C ABI: communicator + comm stream + event plumbing for the bucketed gradient
// all-reduce (and the reduce-scatter / all-gather pair of the optimiser-state-sharded configuration).
//
// Replaces the all-reduce mesh-tensorflow inserts per variable when it lowers a gradient whose batch_dim was reduced
// (src/optimizers.py:34, src/model_fns.py:189) and tf.tpu.CrossShardOptimizer's gradient mean (src/model_fns_tf.py:61):
// one process per GPU, ONE communicator over the GPUs of the box, buckets of the flat fp32 gradient buffer reduced in
// place on a dedicated stream while backward keeps running on the compute stream.
//
// libnccl is resolved at run time (dlopen; the path of torch's bundled libnccl.so.2 is passed in by the host code) so
// that libdalle_b200.so has no link-time dependency on it and single-GPU runs never load it.  The header the structs
// come from (ncclConfig_t) is the one shipped next to that library (NCCL 2.28).
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>

#include "common.cuh"

namespace db200 {
namespace {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRankConfig)(ncclComm_t*, int, ncclUniqueId, int, ncclConfig_t*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*ReduceScatter)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t,
                                cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommRegister)(const ncclComm_t, void*, size_t, void**) = nullptr;
  ncclResult_t (*CommDeregister)(const ncclComm_t, void*) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

int load_nccl(const char* path) {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.handle) return DB200_OK;
  void* h = nullptr;
  if (path && path[0]) h = dlopen(path, RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return set_error(DB200_E_UNSUPPORTED, "cannot load libnccl.so.2 (%s)", dlerror());
#define DB200_SYM(field, name)                                                      \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(h, name));          \
  if (!g_nccl.field) return set_error(DB200_E_UNSUPPORTED, "libnccl lacks %s", name)
  DB200_SYM(GetUniqueId, "ncclGetUniqueId");
  DB200_SYM(CommInitRankConfig, "ncclCommInitRankConfig");
  DB200_SYM(CommDestroy, "ncclCommDestroy");
  DB200_SYM(AllReduce, "ncclAllReduce");
  DB200_SYM(ReduceScatter, "ncclReduceScatter");
  DB200_SYM(AllGather, "ncclAllGather");
  DB200_SYM(GetVersion, "ncclGetVersion");
  DB200_SYM(GetErrorString, "ncclGetErrorString");
#undef DB200_SYM
  // optional (2.19+): user-buffer registration
  g_nccl.CommRegister = reinterpret_cast<decltype(g_nccl.CommRegister)>(dlsym(h, "ncclCommRegister"));
  g_nccl.CommDeregister = reinterpret_cast<decltype(g_nccl.CommDeregister)>(dlsym(h, "ncclCommDeregister"));
  g_nccl.handle = h;
  return DB200_OK;
}

#define DB200_NCCL(call)                                                                                  \
  do {                                                                                                    \
    ncclResult_t r__ = (call);                                                                            \
    if (r__ != ncclSuccess)                                                                               \
      return set_error(DB200_E_CUDA, "%s failed: %s", #call, g_nccl.GetErrorString(r__));                 \
  } while (0)

}  // namespace
}  // namespace db200

using namespace db200;

struct db200_comm {
  ncclComm_t comm = nullptr;
  cudaStream_t stream = nullptr;   // the communication stream (highest priority: collectives are latency-critical)
  cudaEvent_t ready = nullptr;     // recorded on the compute stream: "this bucket's gradients are final"
  cudaEvent_t done = nullptr;      // recorded on the comm stream: "every launched collective has finished"
  int device = 0, rank = 0, world = 1;
  int pending = 0;
  void* reg[8] = {nullptr};
  int n_reg = 0;
};

extern "C" int db200_comm_load_nccl(const char* libnccl_path) { return load_nccl(libnccl_path); }

extern "C" int db200_comm_unique_id(void* id_out, size_t bytes) {
  DB200_REQUIRE(id_out && bytes >= sizeof(ncclUniqueId), DB200_E_INVALID, "comm_unique_id: need a %zu-byte buffer",
                sizeof(ncclUniqueId));
  int rc = load_nccl(nullptr);
  if (rc != DB200_OK) return rc;
  DB200_NCCL(g_nccl.GetUniqueId(reinterpret_cast<ncclUniqueId*>(id_out)));
  return DB200_OK;
}

extern "C" int db200_comm_create(int device, int rank, int world, const void* unique_id, int max_ctas,
                                 db200_comm** out) {
  DB200_REQUIRE(out && unique_id && world >= 1 && rank >= 0 && rank < world, DB200_E_INVALID,
                "comm_create: bad rank %d / world %d or NULL argument", rank, world);
  int rc = load_nccl(nullptr);
  if (rc != DB200_OK) return rc;
  DB200_CUDA(cudaSetDevice(device));
  db200_comm* c = new db200_comm();
  c->device = device; c->rank = rank; c->world = world;
  ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
  cfg.blocking = 1;
  // Cap the CTAs NCCL may occupy: the persistent wgmma GEMM grids of backward run concurrently with the bucket
  // collectives, and every SM NCCL holds is one the one-CTA-per-SM grids wait for.
  if (max_ctas > 0) cfg.maxCTAs = max_ctas;
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  ncclResult_t r = g_nccl.CommInitRankConfig(&c->comm, world, id, rank, &cfg);
  if (r != ncclSuccess) {
    delete c;
    return set_error(DB200_E_CUDA, "ncclCommInitRankConfig failed: %s", g_nccl.GetErrorString(r));
  }
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  DB200_CUDA(cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, hi));
  DB200_CUDA(cudaEventCreateWithFlags(&c->ready, cudaEventDisableTiming));
  DB200_CUDA(cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming));
  *out = c;
  return DB200_OK;
}

extern "C" int db200_comm_destroy(db200_comm* c) {
  if (!c) return DB200_OK;
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (int i = 0; i < c->n_reg; ++i)
    if (g_nccl.CommDeregister && c->reg[i]) g_nccl.CommDeregister(c->comm, c->reg[i]);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  if (c->ready) cudaEventDestroy(c->ready);
  if (c->done) cudaEventDestroy(c->done);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return DB200_OK;
}

// Registers a long-lived buffer (the flat gradient buffer) with the communicator so that NCCL can skip its staging
// copies (and use NVLS user buffers where the allocation allows it).  Best effort: 1 is stored in *registered on success.
extern "C" int db200_comm_register(db200_comm* c, void* buf, size_t bytes, int* registered) {
  DB200_REQUIRE(c && buf, DB200_E_INVALID, "comm_register: NULL argument");
  if (registered) *registered = 0;
  if (!g_nccl.CommRegister || c->n_reg >= 8) return DB200_OK;
  void* h = nullptr;
  if (g_nccl.CommRegister(c->comm, buf, bytes, &h) == ncclSuccess && h) {
    c->reg[c->n_reg++] = h;
    if (registered) *registered = 1;
  }
  return DB200_OK;
}

static ncclDataType_t nccl_dtype(int dtype) { return dtype == DB200_BF16 ? ncclBfloat16 : ncclFloat32; }

// In-place SUM all-reduce of buf[0..count) on the comm stream, ordered after everything already enqueued on
// `compute_stream` (the kernels that produced the bucket) and NOT blocking that stream: backward continues.
extern "C" int db200_bucket_allreduce_launch(db200_comm* c, db200_stream_t compute_stream_, void* buf, size_t count,
                                             int dtype) {
  DB200_REQUIRE(c && buf, DB200_E_INVALID, "bucket_allreduce_launch: NULL argument");
  DB200_REQUIRE(dtype == DB200_F32 || dtype == DB200_BF16, DB200_E_UNSUPPORTED, "bucket_allreduce: dtype %d", dtype);
  if (count == 0 || c->world == 1) return DB200_OK;
  cudaStream_t compute = reinterpret_cast<cudaStream_t>(compute_stream_);
  DB200_CUDA(cudaEventRecord(c->ready, compute));
  DB200_CUDA(cudaStreamWaitEvent(c->stream, c->ready, 0));
  DB200_NCCL(g_nccl.AllReduce(buf, buf, count, nccl_dtype(dtype), ncclSum, c->comm, c->stream));
  c->pending = 1;
  return DB200_OK;
}

// ZeRO-1 pair: SUM reduce-scatter of send[0 .. world*count_per_rank) into recv[0..count_per_rank) (this rank's shard),
// and the all-gather of the updated shards.  Same ordering rules as the all-reduce.
extern "C" int db200_bucket_reduce_scatter_launch(db200_comm* c, db200_stream_t compute_stream_, const void* send,
                                                  void* recv, size_t count_per_rank, int dtype) {
  DB200_REQUIRE(c && send && recv, DB200_E_INVALID, "bucket_reduce_scatter_launch: NULL argument");
  if (count_per_rank == 0) return DB200_OK;
  cudaStream_t compute = reinterpret_cast<cudaStream_t>(compute_stream_);
  DB200_CUDA(cudaEventRecord(c->ready, compute));
  DB200_CUDA(cudaStreamWaitEvent(c->stream, c->ready, 0));
  DB200_NCCL(g_nccl.ReduceScatter(send, recv, count_per_rank, nccl_dtype(dtype), ncclSum, c->comm, c->stream));
  c->pending = 1;
  return DB200_OK;
}

extern "C" int db200_bucket_all_gather_launch(db200_comm* c, db200_stream_t compute_stream_, const void* send,
                                              void* recv, size_t count_per_rank, int dtype) {
  DB200_REQUIRE(c && send && recv, DB200_E_INVALID, "bucket_all_gather_launch: NULL argument");
  if (count_per_rank == 0) return DB200_OK;
  cudaStream_t compute = reinterpret_cast<cudaStream_t>(compute_stream_);
  DB200_CUDA(cudaEventRecord(c->ready, compute));
  DB200_CUDA(cudaStreamWaitEvent(c->stream, c->ready, 0));
  DB200_NCCL(g_nccl.AllGather(send, recv, count_per_rank, nccl_dtype(dtype), c->comm, c->stream));
  c->pending = 1;
  return DB200_OK;
}

// Makes `compute_stream` wait (on the device, no host block) for every collective launched so far.
extern "C" int db200_bucket_allreduce_wait(db200_comm* c, db200_stream_t compute_stream_) {
  DB200_REQUIRE(c, DB200_E_INVALID, "bucket_allreduce_wait: NULL communicator");
  if (!c->pending) return DB200_OK;
  cudaStream_t compute = reinterpret_cast<cudaStream_t>(compute_stream_);
  DB200_CUDA(cudaEventRecord(c->done, c->stream));
  DB200_CUDA(cudaStreamWaitEvent(compute, c->done, 0));
  c->pending = 0;
  return DB200_OK;
}

extern "C" int db200_comm_info(db200_comm* c, int* rank, int* world, int* nccl_version) {
  DB200_REQUIRE(c, DB200_E_INVALID, "comm_info: NULL communicator");
  if (rank) *rank = c->rank;
  if (world) *world = c->world;
  if (nccl_version) g_nccl.GetVersion(nccl_version);
  return DB200_OK;
}
