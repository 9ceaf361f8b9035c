// BoxOutput on the device: anchor decode + objectness score, per-image joint top-N over all
// scales, greedy NMS, and the [R,5] / [R,6] outputs -- without the host round trip the
// reference makes (BoxOutputLayer has only Forward_cpu:
// /root/reference/include/caffe/layers/box_output_layer.hpp:37-40, so GPU mode falls back to
// src/caffe/layers/box_output_layer.cpp:66-234 through layer.hpp:341-345).
//
// Parity notes (every discrete decision of the reference is reproduced bit for bit):
//   * all box arithmetic is fp32 with one rounding per operation (the file is compiled with
//     -fmad=false; the reference is scalar x86-64 code without FMA);
//   * exp() is evaluated in fp64 and rounded once to fp32, which agrees with glibc's expf (the
//     function the reference resolves to for Dtype=float) except on sub-ulp ties;
//   * ranking is std::sort with std::greater<pair<score,idx>> (box_output_layer.cpp:168): score
//     descending, ties broken by the LARGER candidate index.  Candidate indices grow with the
//     anchor scan order (scale j, then row-major position), so the 64-bit key
//     (orderable(score) << 32 | anchor_index) sorted descending gives the same permutation
//     (-0 and +0 compare equal there, so they share one key: score_key);
//   * NMS is nmsMax(greedy) over the top max_nms_num boxes of an image, all scales together
//     (box_output_layer.cpp:38-63,176-182), IoU by BoxIOU (util/math_functions.cpp:13-35) with
//     the strict `>` test.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "mscnn_b200.h"
#include "launch_count.h"
#include "xchg.h"

namespace mscnn {

struct DecodeScale {
  const float* data;  // [N][C][H][W]
  int height, width;
  int anchor_base;    // first anchor index of this scale inside an image
  float field_w, field_h, rate;
  float img_w, img_h;  // (float)(int)(width * rate)
};

struct DecodeParams {
  DecodeScale sc[MSCNN_MAX_SCALES];
  int num_scales, channels, cls_num, anchors_per_image;
  float fg_thr, min_xyr, max_xyr, min_whr, max_whr, min_size;
  int do_norm;
  float mean[4], stdv[4];
};

__device__ __forceinline__ uint32_t float_orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// The sort key of a score.  -0.0f and +0.0f get one key: fg + 0.0f is +0.0f for both (round to nearest), so a run of
// zero scores is ranked by the index word alone, as std::greater<pair<float,int>> (BoxOutput) and MATLAB's stable
// sort (final detections) rank it, where the raw bits would put every +0 above every -0.  The score written back from
// the key is therefore +0.0f for a zero score of either sign.
__device__ __forceinline__ uint32_t score_key(float f) { return float_orderable(f + 0.0f); }
__device__ __forceinline__ float orderable_float(uint32_t o) {
  const uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
  return __uint_as_float(u);
}
__device__ __forceinline__ float exp_ref(float x) { return static_cast<float>(exp(static_cast<double>(x))); }

// One thread per anchor; channel planes are read with unit stride across the warp.
// box_output_layer.cpp:107-163.
__global__ void box_decode_kernel(const DecodeParams p, int N, unsigned long long* __restrict__ keys,
                                  float4* __restrict__ boxes) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  if (a >= p.anchors_per_image) return;
  int j = 0;
#pragma unroll 1
  for (int s = 1; s < p.num_scales; ++s)
    if (a >= p.sc[s].anchor_base) j = s;
  const DecodeScale& S = p.sc[j];
  const int id = a - S.anchor_base;
  const int spatial = S.height * S.width;
  const float* x = S.data + (size_t)n * p.channels * spatial + id;
  const int h = id / S.width, w = id - h * S.width;

  float fg = -3.402823466e+38f;  // -FLT_MAX
  for (int k = 1; k < p.cls_num; ++k) {
    const float v = x[(size_t)k * spatial];
    fg = (fg < v) ? v : fg;  // std::max(fg, v)
  }
  fg = fg - x[0];
  unsigned long long key = 0ull;
  if (fg >= p.fg_thr) {
    const float* c = x + (size_t)p.cls_num * spatial;
    float bx = c[0], by = c[(size_t)spatial], bw = c[(size_t)2 * spatial], bh = c[(size_t)3 * spatial];
    if (p.do_norm) {
      bx = bx * p.stdv[0]; by = by * p.stdv[1]; bw = bw * p.stdv[2]; bh = bh * p.stdv[3];
      bx = bx + p.mean[0]; by = by + p.mean[1]; bw = bw + p.mean[2]; bh = bh + p.mean[3];
    }
    bx = (p.min_xyr < bx) ? bx : p.min_xyr; bx = (bx < p.max_xyr) ? bx : p.max_xyr;
    by = (p.min_xyr < by) ? by : p.min_xyr; by = (by < p.max_xyr) ? by : p.max_xyr;
    bx = bx * S.field_w + ((float)w + 0.5f) * S.rate;
    by = by * S.field_h + ((float)h + 0.5f) * S.rate;
    bw = (p.min_whr < bw) ? bw : p.min_whr; bw = (bw < p.max_whr) ? bw : p.max_whr;
    bh = (p.min_whr < bh) ? bh : p.min_whr; bh = (bh < p.max_whr) ? bh : p.max_whr;
    bw = S.field_w * exp_ref(bw);
    bh = S.field_h * exp_ref(bh);
    bx = bx - bw / 2.0f;
    by = by - bh / 2.0f;
    bx = (bx < 0.0f) ? 0.0f : bx;  // std::max(bbx, 0)
    by = (by < 0.0f) ? 0.0f : by;
    const float rw = S.img_w - bx, rh = S.img_h - by;
    bw = (rw < bw) ? rw : bw;  // std::min(bbw, img_width - bbx)
    bh = (rh < bh) ? rh : bh;
    if (bw >= p.min_size && bh >= p.min_size) {
      key = ((unsigned long long)score_key(fg) << 32) | (unsigned int)a;
      boxes[(size_t)n * p.anchors_per_image + a] = make_float4(bx, by, bw, bh);
    }
  }
  keys[(size_t)n * p.anchors_per_image + a] = key;
}

// ----------------------------------------------------------------------------------------
// Per image: the K largest keys (K = max_nms_num), sorted descending.  One 1024-thread CTA per
// image: byte-wise radix select of the K-th largest key, compaction of keys >= threshold into
// shared memory, bitonic sort.  box_output_layer.cpp:166-179.
constexpr int kTopkThreads = 1024;

// Bitonic sort of the shared keys sk[0 .. Kpad) into descending order (Kpad a power of two) by all kTopkThreads threads
// of the CTA, which have filled sk and synchronised before the call; it ends synchronised.
__device__ __forceinline__ void bitonic_sort_desc(unsigned long long* sk, int Kpad) {
  const int tid = threadIdx.x;
  for (int size = 2; size <= Kpad; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < (Kpad >> 1); i += kTopkThreads) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = sk[lo], b = sk[hi];
        if ((a < b) == desc) { sk[lo] = b; sk[hi] = a; }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(kTopkThreads)
box_topk_kernel(const unsigned long long* __restrict__ keys, const float4* __restrict__ boxes,
                int A, int K, int Kpad, float4* __restrict__ sorted_boxes,
                float* __restrict__ sorted_scores, int* __restrict__ counts) {
  extern __shared__ unsigned long long sk[];  // Kpad keys
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_remaining, s_valid, s_fill;
  const int n = blockIdx.x, tid = threadIdx.x;
  const unsigned long long* kk = keys + (size_t)n * A;

  if (tid == 0) { s_valid = 0; s_fill = 0; }
  __syncthreads();
  int local = 0;
  for (int i = tid; i < A; i += kTopkThreads) local += (kk[i] != 0ull);
  for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((tid & 31) == 0 && local) atomicAdd(&s_valid, local);
  __syncthreads();
  const int valid = s_valid;
  const int M = valid < K ? valid : K;
  unsigned long long thr = 1ull;  // all valid keys
  if (valid > K) {
    if (tid == 0) { s_prefix = 0ull; s_remaining = K; }
    __syncthreads();
    for (int byte = 7; byte >= 0; --byte) {
      for (int i = tid; i < 256; i += kTopkThreads) hist[i] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      for (int i = tid; i < A; i += kTopkThreads) {
        const unsigned long long k = kk[i];
        const bool match = (byte == 7) ? true : ((k >> (8 * (byte + 1))) == prefix);
        if (match && k != 0ull) atomicAdd(&hist[(unsigned)(k >> (8 * byte)) & 255u], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        int rem = s_remaining, d = 255;
        for (; d > 0; --d) {
          const int c = (int)hist[d];
          if (c >= rem) break;
          rem -= c;
        }
        s_remaining = rem;
        s_prefix = (prefix << 8) | (unsigned long long)d;
      }
      __syncthreads();
    }
    thr = s_prefix;  // the K-th largest key (keys are unique: the low word is the anchor index)
  }
  for (int i = tid; i < Kpad; i += kTopkThreads) sk[i] = 0ull;
  __syncthreads();
  for (int i = tid; i < A; i += kTopkThreads) {
    const unsigned long long k = kk[i];
    if (k >= thr && k != 0ull) {
      const int pos = atomicAdd(&s_fill, 1);
      if (pos < Kpad) sk[pos] = k;
    }
  }
  __syncthreads();
  bitonic_sort_desc(sk, Kpad);
  for (int i = tid; i < M; i += kTopkThreads) {
    const unsigned long long k = sk[i];
    const unsigned int a = (unsigned int)(k & 0xFFFFFFFFull);
    sorted_boxes[(size_t)n * Kpad + i] = boxes[(size_t)n * A + a];
    sorted_scores[(size_t)n * Kpad + i] = orderable_float((uint32_t)(k >> 32));
  }
  if (tid == 0) counts[n] = M;
}

// ----------------------------------------------------------------------------------------
// BoxIOU (util/math_functions.cpp:13-35), fp32, one rounding per operation.
__device__ __forceinline__ float box_iou_ref(const float4 a, const float4 b, int mode) {
  if (a.z <= 0.f || a.w <= 0.f || b.z <= 0.f || b.w <= 0.f) return 0.f;
  const float tlx = (a.x < b.x) ? b.x : a.x;
  const float tly = (a.y < b.y) ? b.y : a.y;
  const float ax2 = a.x + a.z, bx2 = b.x + b.z, ay2 = a.y + a.w, by2 = b.y + b.w;
  const float brx = (bx2 < ax2) ? bx2 : ax2;
  const float bry = (by2 < ay2) ? by2 : ay2;
  float over;
  if (tlx >= brx || tly >= bry) over = 0.f;
  else over = (brx - tlx) * (bry - tly);
  float u;
  if (mode == MSCNN_NMS_IOMU) {
    const float a1 = a.z * a.w, a2 = b.z * b.w;
    u = (a2 < a1) ? a2 : a1;
  } else if (mode == MSCNN_NMS_IOFU) {
    u = a.z * a.w;
  } else {
    u = a.z * a.w + b.z * b.w - over;
  }
  return over / u;
}

// bbNms.m:112-126 overlap test in double ('union' denominator).
__device__ __forceinline__ bool bbnms_overlaps(const float4 a, const float4 b, double overlap) {
  const double axs = a.x, axe = (double)a.x + (double)a.z, ays = a.y, aye = (double)a.y + (double)a.w;
  const double bxs = b.x, bxe = (double)b.x + (double)b.z, bys = b.y, bye = (double)b.y + (double)b.w;
  const double iw = fmin(axe, bxe) - fmax(axs, bxs);
  if (iw <= 0) return false;
  const double ih = fmin(aye, bye) - fmax(ays, bys);
  if (ih <= 0) return false;
  double o = iw * ih;
  const double u = (double)a.z * (double)a.w + (double)b.z * (double)b.w - o;
  o = o / u;
  return o > overlap;
}

// The suppression test of each NMS: BoxOutput's BoxIOU in fp32, the post-process's bbNms overlap in fp64.
struct BoxIouTest {
  float thr;
  int mode;
  __device__ __forceinline__ bool operator()(const float4 a, const float4 b) const { return box_iou_ref(a, b, mode) > thr; }
};
struct BbNmsTest {
  double overlap;
  __device__ __forceinline__ bool operator()(const float4 a, const float4 b) const { return bbnms_overlaps(a, b, overlap); }
};

// mask[n][i][cb] bit t  <=>  suppresses(box i, box cb*64+t)  and  cb*64+t > i
template <class Test>
__global__ void nms_mask_kernel(const float4* __restrict__ boxes, const int* __restrict__ counts,
                                int Kpad, int words, const Test suppresses,
                                unsigned long long* __restrict__ mask) {
  const int n = blockIdx.z, rb = blockIdx.y, cb = blockIdx.x;
  const int M = counts[n];
  if (cb < rb || rb * 64 >= M || cb * 64 >= M) return;
  __shared__ float4 cbox[64];
  const int t = threadIdx.x;
  const float4* bx = boxes + (size_t)n * Kpad;
  if (cb * 64 + t < M) cbox[t] = bx[cb * 64 + t];
  __syncthreads();
  const int i = rb * 64 + t;
  if (i >= M) return;
  const float4 me = bx[i];
  const int ncol = min(64, M - cb * 64);
  unsigned long long bits = 0ull;
  const int start = (rb == cb) ? t + 1 : 0;
  for (int c = start; c < ncol; ++c)
    if (suppresses(me, cbox[c])) bits |= (1ull << c);
  mask[((size_t)n * Kpad + i) * words + cb] = bits;
}

// Greedy scan (nmsMax with greedy=true, box_output_layer.cpp:46-56).  One CTA per image walks the boxes in blocks of
// 64.  The greedy order is a true dependence chain (box i survives iff no EARLIER SURVIVOR suppresses it), so the
// work per block is arranged around the chain:
//   * diagonal: warp 0 holds the block's 64 diagonal mask words in registers (lane l: rows l and l + 32) and resolves
//     the 64 intra-block decisions with shuffles -- no memory access on the chain;
//   * meanwhile warps 1..7 stage the NEXT block's mask rows in the other shared-memory buffer (coalesced);
//   * suppression of the later words: all 256 threads, thread (part, word) ORs the kept rows 8 part .. 8 part + 7 of
//     one word and merges with a shared-memory atomicOr (was: one warp, 64 dependent loads per thread);
//   * compaction of the survivors' indices by block-parallel prefix sums of the kept-bit popcounts.
constexpr int kScanThreads = 256;
__global__ void __launch_bounds__(kScanThreads)
nms_scan_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ counts, int Kpad,
                int words, int max_post, int* __restrict__ keep_idx, int* __restrict__ keep_count) {
  extern __shared__ unsigned long long tile[];  // 2 x [64][words]
  __shared__ unsigned long long remv[128];
  __shared__ unsigned long long kept[128];
  __shared__ int kept_off[129];
  __shared__ unsigned long long s_keptbits;
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int M = counts[n];
  const int nb = (M + 63) / 64;
  const unsigned long long* mk = mask + (size_t)n * Kpad * words;
  const int tile_words = 64 * words;
  for (int w = tid; w < 128; w += kScanThreads) { remv[w] = 0ull; kept[w] = 0ull; }
  // stage block b's rows (words b .. nb - 1 only: earlier words are never read) with threads [t0, t0 + nt)
  auto stage = [&](int b, unsigned long long* dst, int t0, int nt) {
    const int rows = min(64, M - b * 64);
    const int wcount = nb - b;
    for (int idx = tid - t0; idx < rows * wcount; idx += nt) {
      const int r = idx / wcount, w = b + idx - r * wcount;
      dst[r * words + w] = mk[(size_t)(b * 64 + r) * words + w];
    }
  };
  if (nb > 0) stage(0, tile, 0, kScanThreads);
  __syncthreads();
  for (int b = 0; b < nb; ++b) {
    const unsigned long long* cur_tile = tile + (b & 1) * tile_words;
    const int rows = min(64, M - b * 64);
    if (warp == 0) {
      const unsigned long long d0 = lane < rows ? cur_tile[lane * words + b] : 0ull;
      const unsigned long long d1 = lane + 32 < rows ? cur_tile[(lane + 32) * words + b] : 0ull;
      unsigned long long cur = remv[b], kb = 0ull;
#pragma unroll 8
      for (int i = 0; i < 64; ++i) {
        const unsigned long long wi = __shfl_sync(0xffffffffu, i < 32 ? d0 : d1, i & 31);
        if (i < rows && !((cur >> i) & 1ull)) {
          kb |= (1ull << i);
          cur |= wi;
        }
      }
      if (lane == 0) {
        s_keptbits = kb;
        kept[b] = kb;
      }
    } else if (b + 1 < nb) {
      stage(b + 1, tile + ((b + 1) & 1) * tile_words, 32, kScanThreads - 32);
    }
    __syncthreads();
    const unsigned long long kb = s_keptbits;
    const int part = tid >> 5;  // rows 8 part .. 8 part + 7
    const unsigned long long kpart = (kb >> (8 * part)) & 0xFFull;
    if (kpart) {
      for (int w = b + 1 + lane; w < nb; w += 32) {
        unsigned long long acc = 0ull;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if ((kpart >> i) & 1ull) acc |= cur_tile[(8 * part + i) * words + w];
        if (acc) atomicOr(&remv[w], acc);
      }
    }
    __syncthreads();
  }
  // survivors' indices in order: exclusive prefix of the per-block popcounts (nb <= 128)
  if (tid == 0) {
    int acc = 0;
    for (int b = 0; b < nb; ++b) { kept_off[b] = acc; acc += __popcll(kept[b]); }
    kept_off[nb] = acc;
    keep_count[n] = (max_post > 0 && acc > max_post) ? max_post : acc;
  }
  __syncthreads();
  for (int idx = tid; idx < nb * 64; idx += kScanThreads) {
    const int b = idx >> 6, i = idx & 63;
    const unsigned long long bits = kept[b];
    if ((bits >> i) & 1ull) {
      const int r = kept_off[b] + __popcll(bits & ((1ull << i) - 1ull));
      if (max_post <= 0 || r < max_post) keep_idx[(size_t)n * Kpad + r] = b * 64 + i;
    }
  }
}

// Concatenate the kept boxes of all images in batch order: top[0] rows [img x1 y1 x1+w y1+h],
// top[1] rows [... score] (box_output_layer.cpp:193-233); zero boxes -> dummy ROI / zero row.
__global__ void box_finalize_kernel(const float4* __restrict__ boxes, const float* __restrict__ scores,
                                    const int* __restrict__ keep_idx, const int* __restrict__ keep_count,
                                    int N, int Kpad, float* __restrict__ rois, float* __restrict__ rois_score,
                                    int* __restrict__ num_out) {
  // one CTA per image (was: one CTA for the whole batch, 61 us at batch 8): its row offset is the sum of the counts
  // of the images before it; the last CTA also knows the total and writes the counters
  const int n = blockIdx.x;
  __shared__ int s_off;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int m = 0; m < n; ++m) acc += keep_count[m];
    s_off = acc;
    num_out[2 + n] = keep_count[n];
    if (n == N - 1) {
      acc += keep_count[n];
      num_out[0] = acc > 0 ? acc : 1;  // rows in the output blobs (dummy row when empty)
      num_out[1] = acc;                // true number of proposals
      if (acc == 0) {
        rois[0] = 0.f; rois[1] = 1.f; rois[2] = 1.f; rois[3] = 10.f; rois[4] = 10.f;
        if (rois_score) for (int k = 0; k < 6; ++k) rois_score[k] = 0.f;
      }
    }
  }
  __syncthreads();
  const int off = s_off, cnt = keep_count[n];
  for (int r = threadIdx.x; r < cnt; r += blockDim.x) {
    const int src = keep_idx[(size_t)n * Kpad + r];
    const float4 b = boxes[(size_t)n * Kpad + src];
    const size_t o = (size_t)(off + r);
    const float x2 = b.x + b.z, y2 = b.y + b.w;
    rois[o * 5 + 0] = (float)n; rois[o * 5 + 1] = b.x; rois[o * 5 + 2] = b.y;
    rois[o * 5 + 3] = x2; rois[o * 5 + 4] = y2;
    if (rois_score) {
      rois_score[o * 6 + 0] = (float)n; rois_score[o * 6 + 1] = b.x; rois_score[o * 6 + 2] = b.y;
      rois_score[o * 6 + 3] = x2; rois_score[o * 6 + 4] = y2;
      rois_score[o * 6 + 5] = scores[(size_t)n * Kpad + src];
    }
  }
}

// ----------------------------------------------------------------------------------------
// Final detections: the MATLAB post-process that follows the Caffe net in the reference
// (examples/kitti_car/run_mscnn_detection.m:75-120 + utils/bbNms.m:112-126 nmsMax 'maxg').
// MATLAB evaluates the decode in single precision (matcaffe returns single, and single op double
// yields single) and the NMS in double on the converted singles; so do these kernels.
// The post-process runs over class SLOTS: slot s = n * num_ids + c is image n with class cls_ids[c] (image-major, so
// the per-slot outputs of N images x C classes read as [N][C] and the packed payload keeps its layout over N * C
// slots).  The single-class entries pass one id and det_thr <= 0.
struct DetectParams {
  int num_cls;
  int num_ids;
  int cls_ids[MSCNN_MAX_DETECT_CLASSES];  // 1-based like the MATLAB scripts
  float det_thr;                          // rows with prob < det_thr are dropped before the sort; -inf when off
  float mean[4], stdv[4];
  float proposal_thr;
};

// Per-image geometry [ratio_h, ratio_w, org_h, org_w] of the slots s0, s0 + 1, ... of one launch (one CTA each), by
// value in the kernel parameter block (1 KB).  The MATLAB drivers read each frame's size inside their loop
// (run_mscnn_detection.m:64-65, run_cascademscnn.m:77-80); a batch without per-image sizes repeats the cfg's four.
constexpr int kGeomPerLaunch = 64;
struct DetectGeom {
  int s0;
  float4 g[kGeomPerLaunch];
};

// One CTA per slot: decode every ROI of the slot's image for the slot's class, rank by probability (MATLAB sort
// 'descend' is stable: ties keep the lower row first), leave boxes sorted in `sboxes` / `sscores`.  With det_thr > 0
// rows below it are dropped first, as the WIDER drivers do before bbNms (examples/widerface/run_mscnn_detection.m:
// 139-143): 'maxg' NMS only lets a box suppress boxes ranked after it, and every row below the threshold ranks after
// every row at or above it, so dropping them before NMS equals dropping them from the unthresholded result.
// CASCADE = false: MS-CNN driver (run_mscnn_detection.m:75-116): prop = proposals_score [R][6],
//   cls = cls_pred logits [R][num_cls], bbox = bbox_pred deltas [R][4 num_cls].
// CASCADE = true: cascade driver (examples/kitti_car/run_cascademscnn.m:99-126): prop = the stage's
//   proposals [R][5], cls = its Softmax output [R][num_cls], bbox = its DecodeBBox output [R][5]
//   (already in net-input pixels); boxes are rescaled, clipped, converted to [x y w h] with the
//   MATLAB "+1" width convention and nothing is thresholded (det_thr = -1).
template <bool CASCADE>
__global__ void __launch_bounds__(kTopkThreads)
detect_decode_sort_kernel(const DetectParams p, const DetectGeom geom, const float* __restrict__ prop,
                          const float* __restrict__ cls,
                          const float* __restrict__ bbox,
                          const int* __restrict__ num_rois, int Kpad, float4* __restrict__ dboxes,
                          float4* __restrict__ sboxes, float* __restrict__ sscores,
                          int* __restrict__ counts) {
  extern __shared__ unsigned long long sk[];
  __shared__ int s_valid;
  const int s = geom.s0 + blockIdx.x, tid = threadIdx.x;
  const int n = s / p.num_ids, c = s - n * p.num_ids;
  int id = p.cls_ids[0] - 1;
#pragma unroll
  for (int k = 1; k < MSCNN_MAX_DETECT_CLASSES; ++k)  // static indices: the ids stay in the parameter bank
    if (c == k) id = p.cls_ids[k] - 1;
  const float4 gn = geom.g[blockIdx.x];
  const float ratio_h = gn.x, ratio_w = gn.y, org_h = gn.z, org_w = gn.w;
  int start = 0;
  for (int m = 0; m < n; ++m) start += num_rois[2 + m];
  int cnt = num_rois[2 + n];
  if (cnt > Kpad) cnt = Kpad;
  if (tid == 0) s_valid = 0;
  for (int i = tid; i < Kpad; i += kTopkThreads) sk[i] = 0ull;
  __syncthreads();
  for (int i = tid; i < cnt; i += kTopkThreads) {
    if (CASCADE) {
      const float* q = prop + (size_t)(start + i) * 5;
      const float qw = q[3] - q[1] + 1.f, qh = q[4] - q[2] + 1.f;  // run_cascademscnn.m:113-117
      if (qw == 0.f || qh == 0.f) continue;
      const float* b = bbox + (size_t)(start + i) * 5;
      float x1 = b[1] / ratio_w, y1 = b[2] / ratio_h, x2 = b[3] / ratio_w, y2 = b[4] / ratio_h;  // :101-102
      x1 = fmaxf(0.f, x1); y1 = fmaxf(0.f, y1);                                                    // :104
      x2 = fminf(x2, org_w); y2 = fminf(y2, org_h);                                                // :105
      const float w = x2 - x1 + 1.f, h = y2 - y1 + 1.f;                                                    // :106
      const float prob = cls[(size_t)(start + i) * p.num_cls + id];
      if (prob != prob) continue;  // bbNms: kp = bbs(:,5) > -inf drops NaN
      if (prob < p.det_thr) continue;  // widerface/run_cascademscnn.m:130-131
      dboxes[(size_t)s * Kpad + i] = make_float4(x1, y1, w, h);
      sk[i] = ((unsigned long long)score_key(prob) << 32) | (unsigned int)(0xFFFFFFFFu - (unsigned)i);
      atomicAdd(&s_valid, 1);
      continue;
    }
    const float* q = prop + (size_t)(start + i) * 6;
    const float px = q[1], py = q[2], pw = q[3] - q[1], ph = q[4] - q[2], psc = q[5];
    if (!(psc >= p.proposal_thr && pw != 0.f && ph != 0.f)) continue;
    const float* c = cls + (size_t)(start + i) * p.num_cls;
    const float* b = bbox + (size_t)(start + i) * 4 * p.num_cls + 4 * id;
    const float dx = b[0] * p.stdv[0] + p.mean[0], dy = b[1] * p.stdv[1] + p.mean[1];
    const float dw = b[2] * p.stdv[2] + p.mean[2], dh = b[3] * p.stdv[3] + p.mean[3];
    float sum = 0.f, mine = 0.f;
    for (int k = 0; k < p.num_cls; ++k) {
      const float e = exp_ref(c[k]);
      sum = sum + e;
      if (k == id) mine = e;
    }
    const float prob = mine / sum;
    const float cx = px + 0.5f * pw, cy = py + 0.5f * ph;
    float tx = dx * pw + cx, ty = dy * ph + cy;
    float tw = pw * exp_ref(dw), th = ph * exp_ref(dh);
    tx = tx - tw / 2.f; ty = ty - th / 2.f;
    tx = tx / ratio_w; tw = tw / ratio_w;
    ty = ty / ratio_h; th = th / ratio_h;
    tx = fmaxf(0.f, tx); ty = fmaxf(0.f, ty);
    tw = fminf(tw, org_w - tx); th = fminf(th, org_h - ty);
    if (prob != prob) continue;  // bbNms: kp = bbs(:,5) > -inf drops NaN
    if (prob < p.det_thr) continue;  // widerface/run_mscnn_detection.m:139-143
    dboxes[(size_t)s * Kpad + i] = make_float4(tx, ty, tw, th);
    sk[i] = ((unsigned long long)score_key(prob) << 32) | (unsigned int)(0xFFFFFFFFu - (unsigned)i);
    atomicAdd(&s_valid, 1);
  }
  __syncthreads();
  bitonic_sort_desc(sk, Kpad);
  const int M = s_valid;
  for (int i = tid; i < M; i += kTopkThreads) {
    const unsigned long long k = sk[i];
    const unsigned int src = 0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull);
    sboxes[(size_t)s * Kpad + i] = dboxes[(size_t)s * Kpad + src];
    sscores[(size_t)s * Kpad + i] = orderable_float((uint32_t)(k >> 32));
  }
  if (tid == 0) counts[s] = M;
}

// dets[n][r] = [x y w h prob], r < det_counts[n], in kept (score-descending) order.
__global__ void detect_write_kernel(const float4* __restrict__ sboxes, const float* __restrict__ sscores,
                                    const int* __restrict__ keep_idx, const int* __restrict__ keep_count,
                                    int Kpad, int cap, float* __restrict__ dets, int* __restrict__ det_counts) {
  const int n = blockIdx.x;
  int cnt = keep_count[n];
  if (cnt > cap) cnt = cap;
  for (int r = threadIdx.x; r < cnt; r += blockDim.x) {
    const int src = keep_idx[(size_t)n * Kpad + r];
    const float4 b = sboxes[(size_t)n * Kpad + src];
    float* o = dets + ((size_t)n * cap + r) * 5;
    o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = sscores[(size_t)n * Kpad + src];
  }
  if (threadIdx.x == 0) det_counts[n] = cnt;
}

// Packed form for the multi-GPU exchange (SURVEY.md 8(e): "fuse the device-side compaction that produces the send
// buffer with the post-process kernel"): payload = int32 header [N, total, counts[0..N)] padded to a multiple of 4
// words, then the kept rows of all images back to back, [total][5] = [x y w h prob] in image order.  One block per
// image; its row offset is the sum of the (capped) counts of the images before it.
struct PackedRows {
  int hdr, off, cnt;  // header words of the payload; this image's first row and row count
};
__device__ __forceinline__ PackedRows pack_image_rows(const float4* sboxes, const float* sscores, const int* keep_idx,
                                                      const int* keep_count, int Kpad, int cap, int N, float* payload) {
  const int n = blockIdx.x;
  int off = 0;
  for (int m = 0; m < n; ++m) off += min(keep_count[m], cap);
  const int cnt = min(keep_count[n], cap);
  const int hdr = (2 + N + 3) & ~3;
  int* head = reinterpret_cast<int*>(payload);
  float* rows = payload + hdr + (size_t)off * 5;
  for (int r = threadIdx.x; r < cnt; r += blockDim.x) {
    const int src = keep_idx[(size_t)n * Kpad + r];
    const float4 b = sboxes[(size_t)n * Kpad + src];
    float* o = rows + (size_t)r * 5;
    o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = sscores[(size_t)n * Kpad + src];
  }
  if (threadIdx.x == 0) {
    head[2 + n] = cnt;
    if (n == N - 1) {
      head[0] = N;
      head[1] = off + cnt;
    }
  }
  return PackedRows{hdr, off, cnt};
}

__global__ void detect_write_packed_kernel(const float4* __restrict__ sboxes, const float* __restrict__ sscores,
                                           const int* __restrict__ keep_idx, const int* __restrict__ keep_count,
                                           int Kpad, int cap, int N, float* __restrict__ payload) {
  pack_image_rows(sboxes, sscores, keep_idx, keep_count, Kpad, cap, N, payload);
}

// The same packing with the EXCHANGE FUSED IN (mscnn_net_detect_push): block n packs image n's rows into this rank's slot
// of its OWN gather buffer, then copies exactly that row range into the same slot of every other rank's buffer through
// peer-mapped pointers over NVLink with 16-byte coalesced stores (the unaligned ends with scalar ones); the last block to
// finish copies the header and publishes the step's sequence number in each rank's flag word (release at system scope).
// No collective kernel, no rendezvous: a rank never waits for a peer to send, and nothing but the receivers'
// cuStreamWaitValue32 ever waits to receive.  (Coalesced 16-byte stores instead of one 4-byte remote store per
// float: 16x fewer NVLink transactions; an ncclAllGather instead holds SMs spinning until the slowest peer joins.)
__global__ void detect_push_packed_kernel(const float4* __restrict__ sboxes, const float* __restrict__ sscores,
                                          const int* __restrict__ keep_idx, const int* __restrict__ keep_count,
                                          int Kpad, int cap, int N, mscnn::PushTargets t, unsigned int seq,
                                          unsigned int* __restrict__ done_counter) {
  const int tid = threadIdx.x, nt = blockDim.x;
  float* lbase = t.data[t.self];
  const PackedRows pr = pack_image_rows(sboxes, sscores, keep_idx, keep_count, Kpad, cap, N, lbase);
  const int hdr = pr.hdr, off = pr.off, cnt = pr.cnt;
  __syncthreads();
  // this block's rows = floats [f0, f1) of the slot; [a0, a1) is the 16-byte aligned middle (slot bases are aligned)
  const size_t f0 = (size_t)hdr + (size_t)off * 5, f1 = f0 + (size_t)cnt * 5;
  size_t a0 = (f0 + 3) & ~(size_t)3, a1 = f1 & ~(size_t)3;
  if (a0 > a1) a0 = a1 = f1;
  for (int d = 0; d < t.count; ++d) {
    if (d == t.self) continue;
    float* dbase = t.data[d];
    const float4* src4 = reinterpret_cast<const float4*>(lbase + a0);
    float4* dst4 = reinterpret_cast<float4*>(dbase + a0);
    const size_t n4 = (a1 - a0) / 4;
    for (size_t i = tid; i < n4; i += nt) dst4[i] = src4[i];
    for (size_t i = f0 + tid; i < a0 && i < f1; i += nt) dbase[i] = lbase[i];
    for (size_t i = (a1 > f0 ? a1 : f0) + tid; i < f1; i += nt) dbase[i] = lbase[i];
  }
  // publish: every block's stores are fenced at system scope; the last block to arrive copies the header (all blocks'
  // counts are in the local slot by then) and writes the flags
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (tid == 0) last = (atomicAdd(done_counter, 1u) == (unsigned)(N - 1));
  __syncthreads();
  if (last) {
    __threadfence();
    for (int d = 0; d < t.count; ++d) {
      if (d == t.self) continue;
      for (int i = tid; i < hdr; i += nt) t.data[d][i] = __ldcg(lbase + i);
    }
    __threadfence_system();
    __syncthreads();
    if (tid < t.count) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(t.flag[tid]), "r"(seq) : "memory");
    if (tid == 0) *done_counter = 0u;  // re-armed for the next launch (stream-ordered)
  }
}

static int next_pow2(int v) {
  int p = 64;
  while (p < v) p <<= 1;
  return p;
}

struct BoxWs {
  size_t keys, boxes, sboxes, sscores, counts, mask, keep_idx, keep_count, total;
};
static BoxWs plan_ws(int N, int A, int Kpad) {
  BoxWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~(size_t)255; return r; };
  w.keys = take((size_t)N * A * 8);
  w.boxes = take((size_t)N * A * 16);
  w.sboxes = take((size_t)N * Kpad * 16);
  w.sscores = take((size_t)N * Kpad * 4);
  w.counts = take((size_t)N * 4);
  w.mask = take((size_t)N * Kpad * (Kpad / 64) * 8);
  w.keep_idx = take((size_t)N * Kpad * 4);
  w.keep_count = take((size_t)N * 4);
  w.total = o;
  return w;
}

}  // namespace mscnn

using namespace mscnn;

static int box_cfg_check(const mscnn_box_output_cfg* c, int N, int* A_out, int* Kpad_out) {
  if (!c || N <= 0 || N > 1024 || c->num_scales <= 0 || c->num_scales > MSCNN_MAX_SCALES) return MSCNN_ERR_INVALID;
  if (c->channels < 6) return MSCNN_ERR_INVALID;
  // The reference treats max_nms_num == 0 as "no cap" (box_output_layer.cpp:176); the device
  // path needs a bound for its shared-memory sort and supports caps up to 8192.
  if (c->max_nms_num <= 0 || c->max_nms_num > 8192) return MSCNN_ERR_INVALID;
  long A = 0;
  for (int j = 0; j < c->num_scales; ++j) {
    if (c->height[j] <= 0 || c->width[j] <= 0) return MSCNN_ERR_INVALID;
    A += (long)c->height[j] * c->width[j];
  }
  if (A > (1l << 30)) return MSCNN_ERR_INVALID;
  *A_out = (int)A;
  *Kpad_out = next_pow2(c->max_nms_num);
  return MSCNN_OK;
}

extern "C" int mscnn_box_output_workspace_bytes(const mscnn_box_output_cfg* cfg, int N, size_t* bytes) {
  int A, Kpad;
  const int rc = box_cfg_check(cfg, N, &A, &Kpad);
  if (rc) return rc;
  if (!bytes) return MSCNN_ERR_INVALID;
  *bytes = plan_ws(N, A, Kpad).total;
  return MSCNN_OK;
}

extern "C" int mscnn_box_output_forward(const mscnn_box_output_cfg* cfg, int N, const float* const* maps,
                                        void* workspace, size_t workspace_bytes, float* proposals,
                                        float* proposals_score, int* num_out, void* stream_v) {
  cudaStream_t stream = (cudaStream_t)stream_v;
  int A, Kpad;
  int rc = box_cfg_check(cfg, N, &A, &Kpad);
  if (rc) return rc;
  if (!maps || !workspace || !proposals || !num_out) return MSCNN_ERR_INVALID;
  const BoxWs w = plan_ws(N, A, Kpad);
  if (workspace_bytes < w.total) return MSCNN_ERR_NOMEM;
  char* ws = (char*)workspace;

  DecodeParams p;
  p.num_scales = cfg->num_scales;
  p.channels = cfg->channels;
  p.cls_num = cfg->channels - 4;
  p.anchors_per_image = A;
  p.fg_thr = cfg->fg_thr;
  // box_output_layer.cpp:76-77, evaluated in fp32 like the reference (Dtype = float)
  p.min_whr = logf(1.0f / cfg->field_whr);
  p.max_whr = logf(cfg->field_whr);
  p.min_xyr = -1.0f / cfg->field_xyr;
  p.max_xyr = 1.0f / cfg->field_xyr;
  p.min_size = cfg->min_size;
  p.do_norm = cfg->do_bbox_norm;
  for (int k = 0; k < 4; ++k) { p.mean[k] = cfg->bbox_mean[k]; p.stdv[k] = cfg->bbox_std[k]; }
  int base = 0;
  for (int j = 0; j < cfg->num_scales; ++j) {
    DecodeScale& S = p.sc[j];
    if (!maps[j]) return MSCNN_ERR_INVALID;
    S.data = maps[j];
    S.height = cfg->height[j];
    S.width = cfg->width[j];
    S.anchor_base = base;
    S.field_w = cfg->field_w[j];
    S.field_h = cfg->field_h[j];
    S.rate = cfg->downsample_rate[j];
    // int img_width = width*downsample_rates[j]  (int * float -> float -> int), :115
    S.img_w = (float)(int)((float)S.width * S.rate);
    S.img_h = (float)(int)((float)S.height * S.rate);
    base += S.height * S.width;
  }
  unsigned long long* keys = (unsigned long long*)(ws + w.keys);
  float4* boxes = (float4*)(ws + w.boxes);
  float4* sboxes = (float4*)(ws + w.sboxes);
  float* sscores = (float*)(ws + w.sscores);
  int* counts = (int*)(ws + w.counts);
  unsigned long long* mask = (unsigned long long*)(ws + w.mask);
  int* keep_idx = (int*)(ws + w.keep_idx);
  int* keep_count = (int*)(ws + w.keep_count);

  mscnn::note_launch();
  box_decode_kernel<<<dim3((A + 255) / 256, N), 256, 0, stream>>>(p, N, keys, boxes);
  const size_t topk_smem = (size_t)Kpad * 8;
  cudaError_t e = cudaFuncSetAttribute(box_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)topk_smem);
  if (e != cudaSuccess) return MSCNN_ERR_CUDA;
  mscnn::note_launch();
  box_topk_kernel<<<N, kTopkThreads, topk_smem, stream>>>(keys, boxes, A, cfg->max_nms_num, Kpad, sboxes,
                                                         sscores, counts);
  const int words = Kpad / 64;
  mscnn::note_launch();
  nms_mask_kernel<<<dim3(words, words, N), 64, 0, stream>>>(sboxes, counts, Kpad, words,
                                                           BoxIouTest{cfg->iou_thr, cfg->nms_type}, mask);
  const size_t scan_smem = (size_t)2 * 64 * words * 8;
  e = cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scan_smem);
  if (e != cudaSuccess) return MSCNN_ERR_CUDA;
  mscnn::note_launch();
  nms_scan_kernel<<<N, kScanThreads, scan_smem, stream>>>(mask, counts, Kpad, words, cfg->max_post_nms_num,
                                                          keep_idx, keep_count);
  mscnn::note_launch();
  box_finalize_kernel<<<N, 256, 0, stream>>>(sboxes, sscores, keep_idx, keep_count, N, Kpad, proposals,
                                             proposals_score, num_out);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn_box_output_forward: %s\n", cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

// ------------------------------------------------------------------------- post-process
namespace mscnn {
struct DetWs {
  size_t dboxes, sboxes, sscores, counts, mask, keep_idx, keep_count, total;
};
static DetWs plan_det_ws(int N, int Kpad) {
  DetWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~(size_t)255; return r; };
  w.dboxes = take((size_t)N * Kpad * 16);
  w.sboxes = take((size_t)N * Kpad * 16);
  w.sscores = take((size_t)N * Kpad * 4);
  w.counts = take((size_t)N * 4);
  w.mask = take((size_t)N * Kpad * (Kpad / 64) * 8);
  w.keep_idx = take((size_t)N * Kpad * 4);
  w.keep_count = take((size_t)N * 4);
  w.total = o;
  return w;
}
}  // namespace mscnn

// The class set of the single-class entries: cfg->cls_id, no detection threshold.
static mscnn_detect_classes single_class(const mscnn_detect_cfg* c) {
  mscnn_detect_classes k;
  memset(&k, 0, sizeof(k));
  k.num_ids = 1;
  k.cls_ids[0] = c ? c->cls_id : 0;
  k.det_thr = -1.f;
  return k;
}

// cfg, N and the class set (cfg->cls_id is not read: the single-class entries pass it as the set's one id).
static int det_cfg_check(const mscnn_detect_cfg* c, const mscnn_detect_classes* k, int N, int* Kpad) {
  if (!c || !k || N <= 0 || N > 1024 || c->num_cls < 2) return MSCNN_ERR_INVALID;
  if (c->max_rois_per_image <= 0 || c->max_rois_per_image > 8192) return MSCNN_ERR_INVALID;
  if (k->num_ids < 1 || k->num_ids > MSCNN_MAX_DETECT_CLASSES || !isfinite(k->det_thr)) return MSCNN_ERR_INVALID;
  for (int i = 0; i < k->num_ids; ++i) {
    if (k->cls_ids[i] < 1 || k->cls_ids[i] > c->num_cls) return MSCNN_ERR_INVALID;
    for (int j = 0; j < i; ++j)
      if (k->cls_ids[j] == k->cls_ids[i]) return MSCNN_ERR_INVALID;
  }
  *Kpad = next_pow2(c->max_rois_per_image);
  return MSCNN_OK;
}

extern "C" int mscnn_detect_workspace_bytes(const mscnn_detect_cfg* cfg, int N, size_t* bytes) {
  const mscnn_detect_classes one = single_class(cfg);
  return mscnn_detect_classes_workspace_bytes(cfg, N, &one, bytes);
}

extern "C" int mscnn_detect_classes_workspace_bytes(const mscnn_detect_cfg* cfg, int N,
                                                    const mscnn_detect_classes* classes, size_t* bytes) {
  int Kpad;
  const int rc = det_cfg_check(cfg, classes, N, &Kpad);
  if (rc) return rc;
  if (!bytes) return MSCNN_ERR_INVALID;
  *bytes = plan_det_ws(N * classes->num_ids, Kpad).total;
  return MSCNN_OK;
}

int mscnn::detect_postprocess(bool cascade, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                              const float* proposals_score, const float* cls_pred, const float* bbox_pred,
                              const int* num_rois, void* workspace, size_t workspace_bytes, const float* geom,
                              const DetectOut& out, void* stream_v) {
  cudaStream_t stream = (cudaStream_t)stream_v;
  const mscnn_detect_classes one = single_class(cfg);
  if (!classes) classes = &one;
  int Kpad;
  const int rc = det_cfg_check(cfg, classes, N, &Kpad);
  if (rc) return rc;
  const int C = classes->num_ids, S = N * C;  // class slots, image-major
  if (!proposals_score || !cls_pred || !bbox_pred || !num_rois || !workspace) return MSCNN_ERR_INVALID;
  if (out.push) {
    if (out.push->count < 1 || out.push->count > kMaxPushRanks || !out.done_counter) return MSCNN_ERR_INVALID;
  } else if (!out.payload && (!out.dets || !out.det_counts)) {
    return MSCNN_ERR_INVALID;
  }
  if (geom)
    for (int k = 0; k < 4 * N; ++k)
      if (!(geom[k] > 0.f) || geom[k] == INFINITY) return MSCNN_ERR_INVALID;
  const DetWs w = plan_det_ws(S, Kpad);
  if (workspace_bytes < w.total) return MSCNN_ERR_NOMEM;
  char* ws = (char*)workspace;
  DetectParams p;
  memset(&p, 0, sizeof(p));
  p.num_cls = cfg->num_cls;
  p.num_ids = C;
  for (int c = 0; c < C; ++c) p.cls_ids[c] = classes->cls_ids[c];
  p.det_thr = classes->det_thr > 0.f ? classes->det_thr : -INFINITY;  // <= 0: off, as the drivers' -1
  for (int k = 0; k < 4; ++k) { p.mean[k] = cfg->bbox_mean[k]; p.stdv[k] = cfg->bbox_std[k]; }
  p.proposal_thr = cfg->proposal_thr;
  float4* dboxes = (float4*)(ws + w.dboxes);
  float4* sboxes = (float4*)(ws + w.sboxes);
  float* sscores = (float*)(ws + w.sscores);
  int* counts = (int*)(ws + w.counts);
  unsigned long long* mask = (unsigned long long*)(ws + w.mask);
  int* keep_idx = (int*)(ws + w.keep_idx);
  int* keep_count = (int*)(ws + w.keep_count);
  const size_t smem = (size_t)Kpad * 8;
  cudaError_t e = cudaFuncSetAttribute(detect_decode_sort_kernel<false>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(detect_decode_sort_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem);
  if (e != cudaSuccess) return MSCNN_ERR_CUDA;
  for (int s0 = 0; s0 < S; s0 += kGeomPerLaunch) {
    const int blocks = S - s0 < kGeomPerLaunch ? S - s0 : kGeomPerLaunch;
    DetectGeom g;
    g.s0 = s0;
    for (int i = 0; i < blocks; ++i) {
      const int n = (s0 + i) / C;
      g.g[i] = geom ? make_float4(geom[4 * n], geom[4 * n + 1], geom[4 * n + 2], geom[4 * n + 3])
                    : make_float4(cfg->ratio_h, cfg->ratio_w, cfg->org_h, cfg->org_w);
    }
    mscnn::note_launch();
    if (cascade)
      detect_decode_sort_kernel<true><<<blocks, kTopkThreads, smem, stream>>>(p, g, proposals_score, cls_pred, bbox_pred,
                                                                             num_rois, Kpad, dboxes, sboxes, sscores,
                                                                             counts);
    else
      detect_decode_sort_kernel<false><<<blocks, kTopkThreads, smem, stream>>>(p, g, proposals_score, cls_pred,
                                                                              bbox_pred, num_rois, Kpad, dboxes, sboxes,
                                                                              sscores, counts);
  }
  const int words = Kpad / 64;
  mscnn::note_launch();
  nms_mask_kernel<<<dim3(words, words, S), 64, 0, stream>>>(sboxes, counts, Kpad, words,
                                                           BbNmsTest{(double)cfg->nms_overlap}, mask);
  const size_t scan_smem = (size_t)2 * 64 * words * 8;
  e = cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scan_smem);
  if (e != cudaSuccess) return MSCNN_ERR_CUDA;
  mscnn::note_launch();
  nms_scan_kernel<<<S, kScanThreads, scan_smem, stream>>>(mask, counts, Kpad, words, 0, keep_idx, keep_count);
  mscnn::note_launch();
  if (out.push)
    detect_push_packed_kernel<<<S, 256, 0, stream>>>(sboxes, sscores, keep_idx, keep_count, Kpad,
                                                    cfg->max_rois_per_image, S, *out.push, out.seq, out.done_counter);
  else if (out.payload)
    detect_write_packed_kernel<<<S, 256, 0, stream>>>(sboxes, sscores, keep_idx, keep_count, Kpad,
                                                     cfg->max_rois_per_image, S, out.payload);
  else
    detect_write_kernel<<<S, 256, 0, stream>>>(sboxes, sscores, keep_idx, keep_count, Kpad,
                                              cfg->max_rois_per_image, out.dets, out.det_counts);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn_detect_postprocess: %s\n", cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

extern "C" int mscnn_detect_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                        const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                        void* workspace, size_t workspace_bytes, float* dets,
                                        int* det_counts, void* stream) {
  return detect_postprocess(false, cfg, nullptr, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace, workspace_bytes,
                            nullptr, DetectOut::padded(dets, det_counts), stream);
}

extern "C" int mscnn_detect_postprocess_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                              const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                              void* workspace, size_t workspace_bytes, float* dets, int* det_counts,
                                              const float* geom, void* stream) {
  if (!geom) return MSCNN_ERR_INVALID;
  return detect_postprocess(false, cfg, nullptr, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace, workspace_bytes,
                            geom, DetectOut::padded(dets, det_counts), stream);
}

extern "C" int mscnn_detect_image_geometry(int net_h, int net_w, int N, const int* org_hw, float* geom) {
  if (net_h < 1 || net_w < 1 || N < 1 || !org_hw || !geom) return MSCNN_ERR_INVALID;
  for (int n = 0; n < N; ++n)
    if (org_hw[2 * n] < 1 || org_hw[2 * n + 1] < 1) return MSCNN_ERR_INVALID;
  for (int n = 0; n < N; ++n) {
    const int oh = org_hw[2 * n], ow = org_hw[2 * n + 1];
    // ratios = [imgH imgW] ./ [orgH orgW] (run_mscnn_detection.m:65), in double, rounded once to the fp32 fields
    geom[4 * n + 0] = (float)((double)net_h / (double)oh);
    geom[4 * n + 1] = (float)((double)net_w / (double)ow);
    geom[4 * n + 2] = (float)oh;
    geom[4 * n + 3] = (float)ow;
  }
  return MSCNN_OK;
}

extern "C" size_t mscnn_detect_payload_floats(int N, int max_rois_per_image) {
  if (N <= 0 || max_rois_per_image <= 0) return 0;
  // header and rows, rounded up to 16 bytes so that consecutive slots of a gather buffer stay 16-byte aligned
  return ((size_t)((2 + N + 3) & ~3) + (size_t)N * max_rois_per_image * 5 + 3) & ~(size_t)3;
}

extern "C" int mscnn_detect_postprocess_packed(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                               const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                               void* workspace, size_t workspace_bytes, float* payload, void* stream) {
  if (!payload) return MSCNN_ERR_INVALID;
  return detect_postprocess(false, cfg, nullptr, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace, workspace_bytes,
                            nullptr, DetectOut::packed(payload), stream);
}

extern "C" int mscnn_detect_postprocess_packed_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                                     const float* cls_pred, const float* bbox_pred,
                                                     const int* num_rois, void* workspace, size_t workspace_bytes,
                                                     float* payload, const float* geom, void* stream) {
  if (!payload || !geom) return MSCNN_ERR_INVALID;
  return detect_postprocess(false, cfg, nullptr, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace, workspace_bytes,
                            geom, DetectOut::packed(payload), stream);
}

extern "C" int mscnn_cascade_detect_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals,
                                                const float* cls_prob, const float* output_bbox,
                                                const int* num_rois, void* workspace, size_t workspace_bytes,
                                                float* dets, int* det_counts, void* stream) {
  return detect_postprocess(true, cfg, nullptr, N, proposals, cls_prob, output_bbox, num_rois, workspace, workspace_bytes,
                            nullptr, DetectOut::padded(dets, det_counts), stream);
}

extern "C" int mscnn_cascade_detect_postprocess_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals,
                                                      const float* cls_prob, const float* output_bbox,
                                                      const int* num_rois, void* workspace, size_t workspace_bytes,
                                                      float* dets, int* det_counts, const float* geom, void* stream) {
  if (!geom) return MSCNN_ERR_INVALID;
  return detect_postprocess(true, cfg, nullptr, N, proposals, cls_prob, output_bbox, num_rois, workspace, workspace_bytes,
                            geom, DetectOut::padded(dets, det_counts), stream);
}

// Several classes in one post-process: N x num_ids slots, slot n * num_ids + c = image n, class cls_ids[c].
extern "C" int mscnn_detect_postprocess_classes(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                                                const float* proposals_score, const float* cls_pred,
                                                const float* bbox_pred, const int* num_rois, void* workspace,
                                                size_t workspace_bytes, float* dets, int* det_counts,
                                                const float* geom, void* stream) {
  if (!classes) return MSCNN_ERR_INVALID;
  return detect_postprocess(false, cfg, classes, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace,
                            workspace_bytes, geom, DetectOut::padded(dets, det_counts), stream);
}

extern "C" int mscnn_cascade_detect_postprocess_classes(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                                        int N, const float* proposals, const float* cls_prob,
                                                        const float* output_bbox, const int* num_rois, void* workspace,
                                                        size_t workspace_bytes, float* dets, int* det_counts,
                                                        const float* geom, void* stream) {
  if (!classes) return MSCNN_ERR_INVALID;
  return detect_postprocess(true, cfg, classes, N, proposals, cls_prob, output_bbox, num_rois, workspace,
                            workspace_bytes, geom, DetectOut::padded(dets, det_counts), stream);
}

extern "C" int mscnn_detect_postprocess_classes_packed(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                                       int N, const float* proposals_score, const float* cls_pred,
                                                       const float* bbox_pred, const int* num_rois, void* workspace,
                                                       size_t workspace_bytes, float* payload, const float* geom,
                                                       void* stream) {
  if (!classes || !payload) return MSCNN_ERR_INVALID;
  return detect_postprocess(false, cfg, classes, N, proposals_score, cls_pred, bbox_pred, num_rois, workspace,
                            workspace_bytes, geom, DetectOut::packed(payload), stream);
}

// ------------------------------------------------------------------------------------------------- proposal list
// The drivers' proposal list (examples/kitti_car/run_mscnn_detection.m:78-91, the same lines in kitti_ped_cyc, caltech
// :83-96, widerface :96-109): w = x2 - x1 and h = y2 - y1 of every proposals_score row in single (:78), the row kept iff
// score >= proposal_thr && w ~= 0 && h ~= 0 in single (:82, `find` keeps row order), then widened to double and divided
// by the double ratios net / original (:86-90), without clipping.  The detection path divides by the fp32 ratio_*
// instead, because there MATLAB divides singles; here the operands are doubles, and a single quotient rounded from the
// fp32 ratio can differ from the double one in the last place of the double.
namespace mscnn {
constexpr int kPropThreads = 256;
constexpr int kPropPerLaunch = 64;
struct ProposalRatios {
  int n0;
  double2 r[kPropPerLaunch];  // (ratio_h, ratio_w) of images n0, n0 + 1, ... (one CTA each)
};
}  // namespace mscnn

// One CTA per image: chunks of kPropThreads rows, each compacted in row order by a warp ballot and a prefix over the
// warps' counts, so the output order is the input order and does not depend on scheduling.
__global__ void __launch_bounds__(kPropThreads)
proposals_kernel(const ProposalRatios ratios, const float* __restrict__ prop, const int* __restrict__ num_rois,
                 float thr, int cap, double* __restrict__ out, int* __restrict__ counts) {
  __shared__ int s_warp[kPropThreads / 32];
  const int n = ratios.n0 + blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double rh = ratios.r[blockIdx.x].x, rw = ratios.r[blockIdx.x].y;
  int start = 0;
  for (int m = 0; m < n; ++m) start += num_rois[2 + m];
  const int cnt = num_rois[2 + n];
  double* o = out + (size_t)n * cap * 5;
  int base = 0;  // rows kept before this chunk
  for (int c0 = 0; c0 < cnt; c0 += kPropThreads) {
    const int i = c0 + tid;
    float x = 0.f, y = 0.f, w = 0.f, h = 0.f, sc = 0.f;
    bool keep = false;
    if (i < cnt) {
      const float* q = prop + (size_t)(start + i) * 6;
      x = q[1]; y = q[2]; w = q[3] - q[1]; h = q[4] - q[2]; sc = q[5];
      keep = sc >= thr && w != 0.f && h != 0.f;  // a NaN score fails the compare, as in MATLAB
    }
    const unsigned ballot = __ballot_sync(0xFFFFFFFFu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int rank = base, total = base;
    for (int k = 0; k < kPropThreads / 32; ++k) {
      if (k < warp) rank += s_warp[k];
      total += s_warp[k];
    }
    rank += __popc(ballot & ((1u << lane) - 1u));
    if (keep && rank < cap) {
      double* r = o + (size_t)rank * 5;
      r[0] = (double)x / rw; r[1] = (double)y / rh; r[2] = (double)w / rw; r[3] = (double)h / rh; r[4] = (double)sc;
    }
    base = total;
    __syncthreads();  // s_warp is rewritten by the next chunk
  }
  if (tid == 0) counts[n] = base <= cap ? base : -1;
}

extern "C" int mscnn_proposals_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                           const int* num_rois, int net_h, int net_w, const int* org_hw, double* props,
                                           int* counts, void* stream_v) {
  if (!cfg || N <= 0 || !proposals_score || !num_rois || !props || !counts || net_h < 1 || net_w < 1)
    return MSCNN_ERR_INVALID;
  if (cfg->max_rois_per_image <= 0) return MSCNN_ERR_INVALID;
  if (org_hw) {
    for (int n = 0; n < N; ++n)
      if (org_hw[2 * n] < 1 || org_hw[2 * n + 1] < 1) return MSCNN_ERR_INVALID;
  } else if (!(cfg->org_h > 0.f && cfg->org_w > 0.f) || cfg->org_h == INFINITY || cfg->org_w == INFINITY) {
    return MSCNN_ERR_INVALID;
  }
  cudaStream_t stream = (cudaStream_t)stream_v;
  for (int n0 = 0; n0 < N; n0 += kPropPerLaunch) {
    const int blocks = N - n0 < kPropPerLaunch ? N - n0 : kPropPerLaunch;
    ProposalRatios r;
    r.n0 = n0;
    for (int i = 0; i < blocks; ++i) {
      // ratios = [imgH imgW] ./ [orgH orgW] (run_mscnn_detection.m:65), in double as MATLAB keeps it
      const double oh = org_hw ? (double)org_hw[2 * (n0 + i)] : (double)cfg->org_h;
      const double ow = org_hw ? (double)org_hw[2 * (n0 + i) + 1] : (double)cfg->org_w;
      r.r[i] = make_double2((double)net_h / oh, (double)net_w / ow);
    }
    mscnn::note_launch();
    proposals_kernel<<<blocks, kPropThreads, 0, stream>>>(r, proposals_score, num_rois, cfg->proposal_thr,
                                                          cfg->max_rois_per_image, props, counts);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn_proposals_postprocess: %s\n", cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}
