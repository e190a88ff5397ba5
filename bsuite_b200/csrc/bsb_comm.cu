// Multi-GPU log points inside the C ABI (SURVEY.md 2.1d / 8e): the ONE collective of the path -- an all-gather of the
// per-rank Logging sums -- for callers that have no torch.distributed (any FFI host).  NCCL is resolved at run time
// with dlopen (no link-time dependency: single-GPU users never load it); the five entry points used are declared
// here from NCCL's public, stable C API.
//
// A log point = one reduction kernel on the caller's stream (bsb_sum_episode_stats_many, or bsb_sum_setting_stats for
// one row per setting) + ncclAllGather on a side stream the communicator owns, fenced by events in both directions,
// so the caller's stream goes on stepping.
#include <dlfcn.h>

#include <cstdlib>
#include <cstring>

#include "bsb_env.h"

using namespace bsb;

namespace {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;                       // ncclSuccess == 0
const int kNcclFloat64 = 8;                     // ncclDataType_t::ncclFloat64 / ncclDouble

struct NcclApi {
  void* handle;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  const char* (*GetErrorString)(ncclResult_t);
};

NcclApi g_nccl = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};

int load_nccl() {
  if (g_nccl.handle) return BSB_OK;
  const char* names[3] = {getenv("BSB_NCCL_LIBRARY"), "libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (int k = 0; k < 3 && !h; ++k)
    if (names[k] && names[k][0]) h = dlopen(names[k], RTLD_NOW | RTLD_LOCAL);
  if (!h) return fail(BSB_UNSUPPORTED, "NCCL not found: set BSB_NCCL_LIBRARY to libnccl.so.2 (needed for multi-GPU log points only)");
  NcclApi api;
  api.handle = h;
  api.GetUniqueId = reinterpret_cast<ncclResult_t (*)(ncclUniqueId*)>(dlsym(h, "ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<ncclResult_t (*)(ncclComm_t*, int, ncclUniqueId, int)>(dlsym(h, "ncclCommInitRank"));
  api.AllGather = reinterpret_cast<ncclResult_t (*)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t)>(dlsym(h, "ncclAllGather"));
  api.CommDestroy = reinterpret_cast<ncclResult_t (*)(ncclComm_t)>(dlsym(h, "ncclCommDestroy"));
  api.GetErrorString = reinterpret_cast<const char* (*)(ncclResult_t)>(dlsym(h, "ncclGetErrorString"));
  if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.CommDestroy || !api.GetErrorString) {
    dlclose(h);
    return fail(BSB_UNSUPPORTED, "the NCCL library lacks a required symbol");
  }
  g_nccl = api;
  return BSB_OK;
}

#define BSB_NCCL(expr)                                                                                    \
  do {                                                                                                    \
    ncclResult_t r__ = (expr);                                                                            \
    if (r__ != 0) return fail(BSB_CUDA_ERROR, std::string(#expr) + ": " + g_nccl.GetErrorString(r__));    \
  } while (0)

struct DeviceScope {
  int prev;
  explicit DeviceScope(int dev) : prev(0) { cudaGetDevice(&prev); cudaSetDevice(dev); }
  ~DeviceScope() { cudaSetDevice(prev); }
};

}  // namespace

struct bsb_comm {
  ncclComm_t comm;
  int rank, world, device;
  cudaStream_t side;            // the all-gather rides here
  cudaEvent_t ready, done;      // reduction finished on the caller's stream / gather finished on the side stream
  bool issued;
};

extern "C" {

int32_t bsb_comm_unique_id(uint8_t* id) {
  if (!id) return fail(BSB_INVALID_ARGUMENT, "null argument");
  { int rc = load_nccl(); if (rc != BSB_OK) return rc; }
  ncclUniqueId uid;
  BSB_NCCL(g_nccl.GetUniqueId(&uid));
  static_assert(sizeof(uid) == BSB_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  memcpy(id, &uid, sizeof(uid));
  return BSB_OK;
}

int32_t bsb_comm_create(const uint8_t* id, int32_t rank, int32_t world, int32_t device, bsb_comm** out) {
  if (!id || !out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (world < 1 || rank < 0 || rank >= world || device < 0) return fail(BSB_INVALID_ARGUMENT, "bad rank / world / device");
  { int rc = load_nccl(); if (rc != BSB_OK) return rc; }
  DeviceScope scope(device);
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  bsb_comm* c = new bsb_comm();
  c->comm = nullptr; c->rank = rank; c->world = world; c->device = device; c->side = nullptr; c->ready = c->done = nullptr; c->issued = false;
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, uid, rank);
  if (r != 0) { delete c; return fail(BSB_CUDA_ERROR, std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r)); }
  if (cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ready, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming) != cudaSuccess) {
    bsb_comm_destroy(c);
    return fail(BSB_CUDA_ERROR, "stream / event creation failed");
  }
  *out = c;
  return BSB_OK;
}

int32_t bsb_comm_destroy(bsb_comm* comm) {
  if (!comm) return BSB_OK;
  DeviceScope scope(comm->device);
  if (comm->side) { cudaStreamSynchronize(comm->side); cudaStreamDestroy(comm->side); }
  if (comm->ready) cudaEventDestroy(comm->ready);
  if (comm->done) cudaEventDestroy(comm->done);
  if (comm->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm->comm);
  delete comm;
  return BSB_OK;
}

int32_t bsb_comm_world(const bsb_comm* comm, int32_t* rank, int32_t* world) {
  if (!comm || !rank || !world) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *rank = comm->rank; *world = comm->world;
  return BSB_OK;
}

// bsb_log_point (one row per handle) and bsb_log_point_settings (one row per setting).
static int32_t log_point(bsb_comm* comm, bsb_env* const* envs, int32_t count, bool per_setting, double* local,
                         double* gathered, void* stream) {
  if (!comm || !envs || !local || !gathered || count <= 0) return fail(BSB_INVALID_ARGUMENT, "bad arguments");
  DeviceScope scope(comm->device);
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  // the previous gather may still be reading `local` / writing `gathered`: the reduction must not overtake it
  if (comm->issued) BSB_CUDA(cudaStreamWaitEvent(caller, comm->done, 0));
  int rc = per_setting ? bsb_sum_setting_stats(envs, count, local, stream)
                       : bsb_sum_episode_stats_many(envs, count, local, stream);
  if (rc != BSB_OK) return rc;
  size_t rows = 0;                      // the reduction has checked every handle
  for (int32_t k = 0; k < count; ++k) rows += per_setting ? (size_t)envs[k]->n_settings : 1;
  BSB_CUDA(cudaEventRecord(comm->ready, caller));
  BSB_CUDA(cudaStreamWaitEvent(comm->side, comm->ready, 0));
  BSB_NCCL(g_nccl.AllGather(local, gathered, rows * 5, kNcclFloat64, comm->comm, comm->side));
  BSB_CUDA(cudaEventRecord(comm->done, comm->side));
  comm->issued = true;
  return BSB_OK;
}

int32_t bsb_log_point(bsb_comm* comm, bsb_env* const* envs, int32_t count, double* local, double* gathered, void* stream) {
  return log_point(comm, envs, count, false, local, gathered, stream);
}

int32_t bsb_log_point_settings(bsb_comm* comm, bsb_env* const* envs, int32_t count, double* local, double* gathered,
                               void* stream) {
  return log_point(comm, envs, count, true, local, gathered, stream);
}

int32_t bsb_comm_wait(bsb_comm* comm, void* stream) {
  if (!comm) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (!comm->issued) return BSB_OK;
  DeviceScope scope(comm->device);
  BSB_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), comm->done, 0));
  return BSB_OK;
}

}  // extern "C"
