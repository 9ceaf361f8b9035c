// Internal entries of the final-detection post-process (box_output.cu) and of the peer-memory exchange of its packed
// results (xchg.cu, box_output.cu detect_push_packed_kernel).
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

// The one output form of a post-process call: padded dets [N][max_rois_per_image][5] + det_counts [N], a packed
// payload (mscnn_detect_payload_floats), or a packed payload pushed to every rank (PushTargets, the step's sequence
// number and the exchange's done counter).
struct DetectOut {
  float* dets;
  int* det_counts;
  float* payload;
  const PushTargets* push;
  unsigned int seq;
  unsigned int* done_counter;
  static DetectOut padded(float* dets, int* det_counts) { return {dets, det_counts, nullptr, nullptr, 0, nullptr}; }
  static DetectOut packed(float* payload) { return {nullptr, nullptr, payload, nullptr, 0, nullptr}; }
  static DetectOut pushed(const PushTargets* push, unsigned int seq, unsigned int* done_counter) {
    return {nullptr, nullptr, nullptr, push, seq, done_counter};
  }
};

// The MS-CNN (cascade = false) or cascade (cascade = true) post-process of N images.  geom: HOST [N][4] = ratio_h,
// ratio_w, org_h, org_w per image, or NULL for the cfg's four scalars.  classes: NULL = cfg->cls_id alone without a
// detection threshold; otherwise the outputs hold N x classes->num_ids slots in image-major order.
int detect_postprocess(bool cascade, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                       const float* proposals_score, const float* cls_pred, const float* bbox_pred, const int* num_rois,
                       void* workspace, size_t workspace_bytes, const float* geom, const DetectOut& out, void* stream);

// mscnn_detect_postprocess_push with optional per-image geometry (HOST [N][4], NULL = the cfg's scalars) and class set
// (NULL = cfg->cls_id; the exchange must then carry mscnn_detect_payload_floats(N * num_ids, cap) floats per rank):
// the Net facade's entry.
int xchg_detect_push(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                     const float* proposals_score, const float* cls_pred, const float* bbox_pred, const int* num_rois,
                     void* workspace, size_t workspace_bytes, void* xchg, const float* geom, void* stream);

}  // namespace mscnn
