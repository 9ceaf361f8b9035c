// Peer-memory exchange of the packed final detections (xchg.cu, box_output.cu detect_push_packed_kernel).
#pragma once
#include <stddef.h>

#include "mscnn_b200.h"

namespace mscnn {

constexpr int kMaxPushRanks = 16;

// Kernel argument: where this rank's payload goes in every rank's gather buffer (peer-mapped device pointers) and the
// flag word of each rank that announces it.
struct PushTargets {
  float* data[kMaxPushRanks];
  unsigned int* flag[kMaxPushRanks];
  int count;
  int self;  // this rank: its slot of ITS OWN buffer is packed first, the others receive copies of it
};

int detect_postprocess_push(const mscnn_detect_cfg* cfg, int N, const float* proposals_score, const float* cls_pred,
                            const float* bbox_pred, const int* num_rois, void* workspace, size_t workspace_bytes,
                            const PushTargets* push, unsigned int seq, unsigned int* done_counter, const float* geom,
                            void* stream);

// mscnn_detect_postprocess_push with optional per-image geometry (HOST [N][4], NULL = the cfg's scalars): the Net
// facade's entry.
int xchg_detect_push(const mscnn_detect_cfg* cfg, int N, const float* proposals_score, const float* cls_pred,
                     const float* bbox_pred, const int* num_rois, void* workspace, size_t workspace_bytes, void* xchg,
                     const float* geom, void* stream);

}  // namespace mscnn
