// Peer-memory exchange of the final detections over NVLink (include/mscnn_b200.h "Peer-memory exchange").
//
// Every rank owns one device allocation: G generations of [flags: one word per rank][data: nranks x payload].  The
// post-process kernel of rank r stores its packed detections directly into slot r of EVERY rank's buffer (its own and,
// through peer-mapped pointers, the others') and then publishes the step's sequence number in word r of every rank's
// flag array (detect_push_packed_kernel, box_output.cu).  Receiving = cuStreamWaitValue32 on the local flag words: a
// stream memory operation, no kernel.  Nothing rendezvouses: a sender never waits for a receiver, the exchange costs no
// launch and holds no SM.  Step s uses generation s mod G; a rank may consume the payloads of step s (on the stream it
// waited on) until it issues its push of step s + 1, and a sender reuses a generation only after every peer has pushed
// step s - G + 1, i.e. has finished with step s - G.  G > 2 lets the ranks drift apart by up to G - 1 steps: per-step
// times jitter by several percent under the power cap, and ranks that must meet EVERY step pay E[max over ranks] per
// step, ranks that only
// have to stay within G steps pay it once per G steps.
//
// Peers in the same process (one host thread per GPU): cudaDeviceEnablePeerAccess + plain pointers
// (mscnn_xchg_connect_local).  Peers in other processes: cudaIpcGetMemHandle / cudaIpcOpenMemHandle; the 64-byte handles
// travel by whatever the host has (torch.distributed in mscnn_b200/parallel.py).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "mscnn_b200.h"
#include "xchg.h"

namespace {

struct Xchg {
  int nranks = 0, rank = 0, device = 0;
  size_t per = 0;            // floats per rank payload
  unsigned int gens = 2;     // generations G
  size_t gen_bytes = 0;      // bytes of one generation: flags (256 B aligned) + data
  size_t flag_bytes = 0;
  char* local = nullptr;     // 2 generations + the done counter
  char* peer[mscnn::kMaxPushRanks] = {};   // base of every rank's allocation as seen from this device
  bool opened_ipc[mscnn::kMaxPushRanks] = {};
  unsigned int seq = 0;      // sequence number of the last push
};

float* gen_data(char* base, const Xchg* x, unsigned gen) { return reinterpret_cast<float*>(base + gen * x->gen_bytes + x->flag_bytes); }
unsigned int* gen_flags(char* base, const Xchg* x, unsigned gen) { return reinterpret_cast<unsigned int*>(base + gen * x->gen_bytes); }

PFN_cuStreamWaitValue32_v11070 wait_value_fn() {
  static PFN_cuStreamWaitValue32_v11070 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuStreamWaitValue32_v11070>(p);
    else
      fprintf(stderr, "mscnn_xchg: cuStreamWaitValue32 entry point unavailable\n");
  });
  return fn;
}

}  // namespace

extern "C" {

int mscnn_xchg_create(void** out, int nranks, int rank, size_t floats_per_rank, int generations) {
  if (!out || nranks < 1 || nranks > mscnn::kMaxPushRanks || rank < 0 || rank >= nranks || floats_per_rank == 0 ||
      generations < 2 || generations > 1024)
    return MSCNN_ERR_INVALID;
  Xchg* x = new Xchg();
  x->gens = (unsigned)generations;
  x->nranks = nranks;
  x->rank = rank;
  x->per = floats_per_rank;
  x->flag_bytes = 256;
  x->gen_bytes = (x->flag_bytes + (size_t)nranks * floats_per_rank * sizeof(float) + 255) & ~(size_t)255;
  if (cudaGetDevice(&x->device) != cudaSuccess) { delete x; return MSCNN_ERR_CUDA; }
  const size_t total = x->gens * x->gen_bytes + 256;
  if (cudaMalloc(&x->local, total) != cudaSuccess) { delete x; return MSCNN_ERR_NOMEM; }
  if (cudaMemset(x->local, 0, total) != cudaSuccess) { cudaFree(x->local); delete x; return MSCNN_ERR_CUDA; }
  x->peer[rank] = x->local;
  *out = x;
  return MSCNN_OK;
}

int mscnn_xchg_destroy(void* xv) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x) return MSCNN_OK;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(x->device);
  cudaDeviceSynchronize();
  for (int p = 0; p < x->nranks; ++p)
    if (x->opened_ipc[p] && x->peer[p]) cudaIpcCloseMemHandle(x->peer[p]);
  if (x->local) cudaFree(x->local);
  cudaSetDevice(prev);
  delete x;
  return MSCNN_OK;
}

int mscnn_xchg_ipc_handle(void* xv, void* handle64) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x || !handle64) return MSCNN_ERR_INVALID;
  static_assert(sizeof(cudaIpcMemHandle_t) == MSCNN_XCHG_HANDLE_BYTES, "cudaIpcMemHandle_t size");
  cudaIpcMemHandle_t h;
  if (cudaIpcGetMemHandle(&h, x->local) != cudaSuccess) {
    fprintf(stderr, "mscnn_xchg: cudaIpcGetMemHandle: %s\n", cudaGetErrorString(cudaGetLastError()));
    return MSCNN_ERR_CUDA;
  }
  memcpy(handle64, &h, sizeof(h));
  return MSCNN_OK;
}

int mscnn_xchg_open_peer_ipc(void* xv, int peer, const void* handle64) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x || !handle64 || peer < 0 || peer >= x->nranks || peer == x->rank) return MSCNN_ERR_INVALID;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  void* p = nullptr;
  if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
    fprintf(stderr, "mscnn_xchg: cudaIpcOpenMemHandle(rank %d): %s\n", peer, cudaGetErrorString(cudaGetLastError()));
    return MSCNN_ERR_CUDA;
  }
  x->peer[peer] = static_cast<char*>(p);
  x->opened_ipc[peer] = true;
  return MSCNN_OK;
}

// Same process, one exchange object per device: enable peer access both ways and hand out the pointers.
int mscnn_xchg_connect_local(void** xs, int n) {
  if (!xs || n < 1 || n > mscnn::kMaxPushRanks) return MSCNN_ERR_INVALID;
  int prev = 0;
  cudaGetDevice(&prev);
  for (int i = 0; i < n; ++i) {
    Xchg* a = static_cast<Xchg*>(xs[i]);
    if (!a || a->nranks != n || a->rank != i) return MSCNN_ERR_INVALID;
    cudaSetDevice(a->device);
    for (int j = 0; j < n; ++j) {
      Xchg* b = static_cast<Xchg*>(xs[j]);
      if (i == j) continue;
      if (a->device != b->device) {
        const cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
          fprintf(stderr, "mscnn_xchg: peer access %d -> %d: %s\n", a->device, b->device, cudaGetErrorString(e));
          cudaSetDevice(prev);
          return MSCNN_ERR_CUDA;
        }
        cudaGetLastError();
      }
      a->peer[j] = b->local;
    }
  }
  cudaSetDevice(prev);
  return MSCNN_OK;
}

int mscnn_xchg_info(void* xv, int* nranks, int* rank, size_t* floats_per_rank) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x) return MSCNN_ERR_INVALID;
  if (nranks) *nranks = x->nranks;
  if (rank) *rank = x->rank;
  if (floats_per_rank) *floats_per_rank = x->per;
  return MSCNN_OK;
}

// The gathered payloads of the last push: [nranks][floats_per_rank] on this device (valid after mscnn_xchg_wait).
const float* mscnn_xchg_buffer(void* xv) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x || x->seq == 0) return nullptr;
  return gen_data(x->local, x, x->seq % x->gens);
}

static int wait_seq(Xchg* x, unsigned int seq, void* stream) {
  if (seq == 0) return MSCNN_OK;
  PFN_cuStreamWaitValue32_v11070 wait = wait_value_fn();
  if (!wait) return MSCNN_ERR_CUDA;
  unsigned int* flags = gen_flags(x->local, x, seq % x->gens);
  for (int p = 0; p < x->nranks; ++p) {
    const CUresult r = wait(static_cast<CUstream>(stream), reinterpret_cast<CUdeviceptr>(flags + p), seq,
                            CU_STREAM_WAIT_VALUE_GEQ);
    if (r != CUDA_SUCCESS) {
      fprintf(stderr, "mscnn_xchg: cuStreamWaitValue32 rc=%d\n", (int)r);
      return MSCNN_ERR_CUDA;
    }
  }
  return MSCNN_OK;
}

// `stream` waits (on the device, no kernel) until every rank's payload of the last push has landed here.
int mscnn_xchg_wait(void* xv, void* stream) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x) return MSCNN_ERR_INVALID;
  return wait_seq(x, x->seq, stream);
}

// Post-process on raw blobs + fused push (the Net facade's mscnn_net_detect_push wraps this).  Flow control: the push of
// step s first makes the stream wait for every peer's payload of step s - G + 1 (long arrived in steady state): a peer
// that has pushed s - G + 1 has finished consuming step s - G, whose generation this push overwrites.  Ranks stay
// within G - 1 steps of each other, and nobody ever spins on an SM.
int mscnn_detect_postprocess_push(const mscnn_detect_cfg* cfg, int N, const float* proposals_score, const float* cls_pred,
                                  const float* bbox_pred, const int* num_rois, void* workspace, size_t workspace_bytes,
                                  void* xv, void* stream) {
  return mscnn::xchg_detect_push(cfg, nullptr, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace,
                                 workspace_bytes, xv, nullptr, stream);
}

}  // extern "C"

int mscnn::xchg_detect_push(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                            const float* proposals_score, const float* cls_pred, const float* bbox_pred,
                            const int* num_rois, void* workspace, size_t workspace_bytes, void* xv, const float* geom,
                            void* stream) {
  Xchg* x = static_cast<Xchg*>(xv);
  if (!x) return MSCNN_ERR_INVALID;
  // every argument is checked (host only) before the flow-control wait below is queued
  size_t ws_need = 0;
  const int crc = classes ? mscnn_detect_classes_workspace_bytes(cfg, N, classes, &ws_need)
                          : mscnn_detect_workspace_bytes(cfg, N, &ws_need);
  if (crc != MSCNN_OK) return crc;
  const int slots = N * (classes ? classes->num_ids : 1);
  if (mscnn_detect_payload_floats(slots, cfg->max_rois_per_image) != x->per) return MSCNN_ERR_INVALID;
  for (int p = 0; p < x->nranks; ++p)
    if (!x->peer[p]) return MSCNN_ERR_INVALID;  // not connected yet
  const unsigned int seq = x->seq + 1, gen = seq % x->gens;
  if (seq >= x->gens) {
    const int wrc = wait_seq(x, seq - x->gens + 1, stream);
    if (wrc != MSCNN_OK) return wrc;
  }
  mscnn::PushTargets t;
  memset(&t, 0, sizeof(t));
  t.count = x->nranks;
  t.self = x->rank;
  for (int p = 0; p < x->nranks; ++p) {
    t.data[p] = gen_data(x->peer[p], x, gen) + (size_t)x->rank * x->per;
    t.flag[p] = gen_flags(x->peer[p], x, gen) + x->rank;
  }
  unsigned int* counter = reinterpret_cast<unsigned int*>(x->local + (size_t)x->gens * x->gen_bytes);
  const int rc = mscnn::detect_postprocess(false, cfg, classes, N, proposals_score, cls_pred, bbox_pred, num_rois,
                                           workspace, workspace_bytes, geom, mscnn::DetectOut::pushed(&t, seq, counter),
                                           stream);
  if (rc == MSCNN_OK) x->seq = seq;
  return rc;
}
