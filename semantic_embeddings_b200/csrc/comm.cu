// Data-parallel gradient exchange inside the C-ABI (SURVEY.md section 8b/8e): one NCCL communicator per process
// (one process per GPU), sum all-reduce of ranges of the flat gradient buffer on a dedicated stream so that the plan
// runner can overlap bucket k's exchange with the backward pass of the layers below it and capture everything -- forward,
// backward, all-reduce, optimizer -- in ONE CUDA graph.  Replaces keras.utils.multi_gpu_model's tower merge
// (learn_image_embeddings.py:133,148): per-sample losses are pre-scaled by 1/global_batch, so the SUM is the gradient of
// the global mean.
// NCCL is resolved at run time from the libnccl.so.2 the process already holds (PyTorch links it): no link-time
// dependency, and a host without NCCL only loses se_comm_init (single-GPU paths never call it).
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include "common.cuh"

namespace se {

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  const char* (*GetErrorString)(ncclResult_t);
  bool ok;
};

static NcclApi load_nccl() {
  NcclApi api = {};
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);          // the copy PyTorch already loaded
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (h) {
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
    api.GroupStart = (decltype(api.GroupStart))dlsym(h, "ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))dlsym(h, "ncclGroupEnd");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce && api.GroupStart && api.GroupEnd;
  }
  return api;
}

static NcclApi* nccl_api() {
  static NcclApi api = load_nccl();
  return &api;
}

static ncclComm_t g_comm = nullptr;
static int g_rank = 0, g_world = 1;
static cudaStream_t g_comm_stream = nullptr;
static cudaEvent_t g_comm_event = nullptr;   // orders the communication stream against se_run_ops' streams

static int nccl_fail(const char* what, ncclResult_t r) {
  NcclApi* a = nccl_api();
  set_error("%s: %s", what, a->GetErrorString ? a->GetErrorString(r) : "NCCL error");
  return SE_ERR_CUDA;
}

cudaStream_t comm_stream() { return g_comm_stream; }
cudaEvent_t comm_event() { return g_comm_event; }
bool comm_ready() { return g_comm != nullptr; }

// sum all-reduce (in place) of `nranges` element ranges of a float buffer on stream `st`, one NCCL group
int comm_allreduce_ranges(float* base, const long long* off, const long long* cnt, int nranges, cudaStream_t st) {
  NcclApi* a = nccl_api();
  if (!g_comm) { set_error("se_allreduce: no communicator (call se_comm_init)"); return SE_ERR_ARG; }
  ncclResult_t r = a->GroupStart();
  if (r != ncclSuccess) return nccl_fail("ncclGroupStart", r);
  for (int k = 0; k < nranges; ++k) {
    if (cnt[k] <= 0) continue;
    r = a->AllReduce(base + off[k], base + off[k], (size_t)cnt[k], ncclFloat32, ncclSum, g_comm, st);
    if (r != ncclSuccess) { a->GroupEnd(); return nccl_fail("ncclAllReduce", r); }
  }
  r = a->GroupEnd();
  if (r != ncclSuccess) return nccl_fail("ncclGroupEnd", r);
  count_launch(1);
  return SE_OK;
}

}  // namespace se

using namespace se;

extern "C" int se_comm_unique_id(void* id_out, int bytes) {
  SE_REQUIRE(id_out && bytes >= (int)sizeof(ncclUniqueId), "need a 128-byte buffer");
  NcclApi* a = nccl_api();
  if (!a->ok) { set_error("se_comm_unique_id: libnccl.so.2 is not available in this process"); return SE_ERR_UNSUPPORTED; }
  ncclUniqueId id;
  ncclResult_t r = a->GetUniqueId(&id);
  if (r != ncclSuccess) return nccl_fail("ncclGetUniqueId", r);
  memcpy(id_out, &id, sizeof(id));
  return SE_OK;
}

extern "C" int se_comm_init(int rank, int world, const void* unique_id, int bytes) {
  SE_REQUIRE(unique_id && bytes >= (int)sizeof(ncclUniqueId) && world >= 1 && rank >= 0 && rank < world, "bad arguments");
  NcclApi* a = nccl_api();
  if (!a->ok) { set_error("se_comm_init: libnccl.so.2 is not available in this process"); return SE_ERR_UNSUPPORTED; }
  if (g_comm) { set_error("se_comm_init: a communicator already exists (se_comm_destroy first)"); return SE_ERR_ARG; }
  if (!g_comm_stream) {   // the stream and event outlive a communicator: se_comm_destroy keeps them for the next one
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (cudaStreamCreateWithPriority(&g_comm_stream, cudaStreamNonBlocking, hi) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_comm_event, cudaEventDisableTiming) != cudaSuccess) {
      g_comm_stream = nullptr;
      set_error("se_comm_init: cannot create the communication stream");
      return SE_ERR_CUDA;
    }
  }
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  ncclResult_t r = a->CommInitRank(&g_comm, world, id, rank);
  if (r != ncclSuccess) { g_comm = nullptr; return nccl_fail("ncclCommInitRank", r); }
  g_rank = rank; g_world = world;
  return SE_OK;
}

extern "C" int se_comm_world(void) { return g_comm ? g_world : 1; }

extern "C" int se_allreduce_sum(float* buf, int64_t n, void* stream) {
  SE_REQUIRE(buf && n > 0, "bad arguments");
  const long long off = 0, cnt = n;
  return comm_allreduce_ranges(buf, &off, &cnt, 1, as_stream(stream));
}

extern "C" int se_comm_destroy(void) {
  if (g_comm) {
    NcclApi* a = nccl_api();
    a->CommDestroy(g_comm);
    g_comm = nullptr;
    g_world = 1;
    g_rank = 0;
  }
  return SE_OK;
}
