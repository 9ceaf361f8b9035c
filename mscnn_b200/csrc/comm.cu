// Multi-GPU exchange of the detection forward path (SURVEY.md 8(e); include/mscnn_b200.h "multi-GPU").
//
// Images are independent, so the path shards by image with NO data-path collective; the one exchange is an all-gather
// of the final detections at the end of a step.  The reference has no multi-GPU inference at all (its P2PSync is
// training-only, src/caffe/parallel.cpp:421-439); what this file matches is its threading model: one Caffe context
// per host thread (boost::thread_specific_ptr, src/caffe/common.cpp:13-22), here one communicator rank per thread
// (mscnn_comm_init_all) or per process (mscnn_comm_init_rank).
//
// ONE ncclAllGather per step: each rank's payload carries its per-image counts in a header in front of the compacted
// rows (pack_image_rows, box_output.cu), so no second collective for the counts.  The collective runs on
// the communicator's own stream: it waits (on the device) for the producer stream's tail and the producer goes on
// with the next step's trunk, so step k's gather overlaps step k + 1's convolutions.
//
// NCCL is bound at run time (dlopen): the library keeps no link dependency, and inside a process that already
// carries an NCCL (torch's) the same instance is used.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "mscnn_b200.h"

namespace {

struct NcclApi {
  ncclResult_t (*GetVersion)(int*);
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  const char* (*GetErrorString)(ncclResult_t);
  void* handle;
  bool ok;
};

NcclApi g_api;
std::once_flag g_api_once;

void load_api() {
  memset(&g_api, 0, sizeof(g_api));
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // an NCCL already in the process (torch's) wins
  if (!h) {
    if (const char* e = getenv("MSCNN_NCCL_LIB")) h = dlopen(e, RTLD_NOW | RTLD_GLOBAL);
  }
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    fprintf(stderr, "mscnn_comm: cannot load libnccl.so.2 (%s); set MSCNN_NCCL_LIB\n", dlerror());
    return;
  }
  g_api.handle = h;
#define BIND(field, sym)                                                   \
  *reinterpret_cast<void**>(&g_api.field) = dlsym(h, sym);                 \
  if (!g_api.field) {                                                      \
    fprintf(stderr, "mscnn_comm: %s missing from libnccl\n", sym);         \
    return;                                                                \
  }
  BIND(GetVersion, "ncclGetVersion")
  BIND(GetUniqueId, "ncclGetUniqueId")
  BIND(CommInitRank, "ncclCommInitRank")
  BIND(CommInitAll, "ncclCommInitAll")
  BIND(CommDestroy, "ncclCommDestroy")
  BIND(AllGather, "ncclAllGather")
  BIND(GetErrorString, "ncclGetErrorString")
#undef BIND
  g_api.ok = true;
}

NcclApi* api() {
  std::call_once(g_api_once, load_api);
  return g_api.ok ? &g_api : nullptr;
}

struct Comm {
  ncclComm_t comm = nullptr;
  int nranks = 0, rank = 0, device = 0;
  cudaStream_t stream = nullptr;            // the collective's own stream
  cudaEvent_t produced = nullptr;           // producer stream's tail -> collective
  cudaEvent_t done = nullptr;               // collective finished
  bool done_valid = false;
  // device time of the last kTimed collectives (start / end on the communicator's stream): the collective's own
  // duration INCLUDING its wait for the slowest peer -- what the scaling analysis needs (mscnn_comm_gather_times)
  static constexpr int kTimed = 64;
  cudaEvent_t t0[kTimed] = {}, t1[kTimed] = {};
  unsigned long long issued = 0;
};

int nccl_fail(const char* what, ncclResult_t r) {
  fprintf(stderr, "mscnn_comm: %s: %s\n", what, g_api.GetErrorString ? g_api.GetErrorString(r) : "?");
  return MSCNN_ERR_CUDA;
}

int finish_init(Comm* c) {
  if (cudaSetDevice(c->device) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (cudaEventCreateWithFlags(&c->produced, cudaEventDisableTiming) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming) != cudaSuccess) return MSCNN_ERR_CUDA;
  for (int i = 0; i < Comm::kTimed; ++i)
    if (cudaEventCreate(&c->t0[i]) != cudaSuccess || cudaEventCreate(&c->t1[i]) != cudaSuccess) return MSCNN_ERR_CUDA;
  return MSCNN_OK;
}

}  // namespace

extern "C" {

int mscnn_comm_nccl_version(void) {
  NcclApi* a = api();
  int v = 0;
  if (!a || a->GetVersion(&v) != ncclSuccess) return 0;
  return v;
}

int mscnn_comm_get_unique_id(void* id128) {
  NcclApi* a = api();
  if (!a || !id128) return MSCNN_ERR_INVALID;
  static_assert(sizeof(ncclUniqueId) == MSCNN_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  const ncclResult_t r = a->GetUniqueId(&id);
  if (r != ncclSuccess) return nccl_fail("ncclGetUniqueId", r);
  memcpy(id128, &id, sizeof(id));
  return MSCNN_OK;
}

int mscnn_comm_init_rank(void** comm_out, int nranks, int rank, const void* id128) {
  NcclApi* a = api();
  if (!a || !comm_out || !id128 || nranks <= 0 || rank < 0 || rank >= nranks) return MSCNN_ERR_INVALID;
  Comm* c = new Comm();
  c->nranks = nranks;
  c->rank = rank;
  if (cudaGetDevice(&c->device) != cudaSuccess) { delete c; return MSCNN_ERR_CUDA; }
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  const ncclResult_t r = a->CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) { delete c; return nccl_fail("ncclCommInitRank", r); }
  const int rc = finish_init(c);
  if (rc) { mscnn_comm_destroy(c); return rc; }
  *comm_out = c;
  return MSCNN_OK;
}

int mscnn_comm_init_all(void** comms_out, int ndev, const int* devices) {
  NcclApi* a = api();
  if (!a || !comms_out || ndev <= 0 || ndev > 64) return MSCNN_ERR_INVALID;
  ncclComm_t raw[64];
  int devs[64];
  for (int i = 0; i < ndev; ++i) devs[i] = devices ? devices[i] : i;
  int prev = 0;
  cudaGetDevice(&prev);
  const ncclResult_t r = a->CommInitAll(raw, ndev, devs);
  if (r != ncclSuccess) return nccl_fail("ncclCommInitAll", r);
  int rc = MSCNN_OK;
  for (int i = 0; i < ndev; ++i) {
    Comm* c = new Comm();
    c->comm = raw[i];
    c->nranks = ndev;
    c->rank = i;
    c->device = devs[i];
    comms_out[i] = c;
    const int rci = finish_init(c);
    if (rci) rc = rci;
  }
  cudaSetDevice(prev);
  return rc;
}

int mscnn_comm_destroy(void* comm) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c) return MSCNN_OK;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->comm && api()) g_api.CommDestroy(c->comm);
  if (c->produced) cudaEventDestroy(c->produced);
  if (c->done) cudaEventDestroy(c->done);
  for (int i = 0; i < Comm::kTimed; ++i) {
    if (c->t0[i]) cudaEventDestroy(c->t0[i]);
    if (c->t1[i]) cudaEventDestroy(c->t1[i]);
  }
  if (c->stream) cudaStreamDestroy(c->stream);
  cudaSetDevice(prev);
  delete c;
  return MSCNN_OK;
}

int mscnn_comm_info(void* comm, int* nranks, int* rank, int* device) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c) return MSCNN_ERR_INVALID;
  if (nranks) *nranks = c->nranks;
  if (rank) *rank = c->rank;
  if (device) *device = c->device;
  return MSCNN_OK;
}

int mscnn_comm_stream_wait(void* comm, void* stream) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c) return MSCNN_ERR_INVALID;
  if (!c->done_valid) return MSCNN_OK;
  return cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), c->done, 0) == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}

int mscnn_comm_synchronize(void* comm) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c) return MSCNN_ERR_INVALID;
  if (!c->done_valid) return MSCNN_OK;
  return cudaEventSynchronize(c->done) == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}

// In-place all-gather: rank r's `floats_per_rank` floats sit at buf_all + r * floats_per_rank and were (or are being)
// written on `producer_stream`.  Runs on the communicator's stream behind the producer's current tail.
int mscnn_comm_all_gather(void* comm, float* buf_all, size_t floats_per_rank, void* producer_stream) {
  Comm* c = static_cast<Comm*>(comm);
  NcclApi* a = api();
  if (!c || !a || !buf_all || floats_per_rank == 0) return MSCNN_ERR_INVALID;
  if (cudaEventRecord(c->produced, static_cast<cudaStream_t>(producer_stream)) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (cudaStreamWaitEvent(c->stream, c->produced, 0) != cudaSuccess) return MSCNN_ERR_CUDA;
  const int slot = static_cast<int>(c->issued % Comm::kTimed);
  cudaEventRecord(c->t0[slot], c->stream);
  const ncclResult_t r = a->AllGather(buf_all + (size_t)c->rank * floats_per_rank, buf_all, floats_per_rank, ncclFloat32,
                                      c->comm, c->stream);
  if (r != ncclSuccess) return nccl_fail("ncclAllGather", r);
  cudaEventRecord(c->t1[slot], c->stream);
  ++c->issued;
  if (cudaEventRecord(c->done, c->stream) != cudaSuccess) return MSCNN_ERR_CUDA;
  c->done_valid = true;
  return MSCNN_OK;
}

// Device durations (ms) of the most recent collectives, oldest first; returns how many were written (<= cap, <= 64).
// Waits for the last one.
int mscnn_comm_gather_times(void* comm, float* host_ms, int cap) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c || !host_ms || cap <= 0) return MSCNN_ERR_INVALID;
  if (c->done_valid && cudaEventSynchronize(c->done) != cudaSuccess) return MSCNN_ERR_CUDA;
  const unsigned long long have = c->issued < (unsigned long long)Comm::kTimed ? c->issued : Comm::kTimed;
  const int n = static_cast<int>(have < (unsigned long long)cap ? have : cap);
  for (int i = 0; i < n; ++i) {
    const int slot = static_cast<int>((c->issued - n + i) % Comm::kTimed);
    if (cudaEventElapsedTime(&host_ms[i], c->t0[slot], c->t1[slot]) != cudaSuccess) return MSCNN_ERR_CUDA;
  }
  return n;
}

}  // extern "C"
