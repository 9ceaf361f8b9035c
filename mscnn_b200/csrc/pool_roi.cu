// HBM-bound plane kernels: Pooling, ROIPooling (+ fused Concat), depthwise Deconvolution.
// All work on NHWC bf16 planes with 16-byte (8-channel) vector accesses, so a warp touches
// 512 contiguous bytes per pixel; values of split tensors are hi + lo evaluated in fp32.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "deconv_phase.h"
#include "mscnn_b200.h"
#include "launch_count.h"

namespace mscnn {

struct Vec8 {
  float v[8];
};

__device__ __forceinline__ Vec8 load8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t off) {
  Vec8 r;
  const uint4 a = *reinterpret_cast<const uint4*>(hi + off);
  const __nv_bfloat162* ap = reinterpret_cast<const __nv_bfloat162*>(&a);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.v[2 * i] = __bfloat162float(ap[i].x);
    r.v[2 * i + 1] = __bfloat162float(ap[i].y);
  }
  if (lo) {
    const uint4 b = *reinterpret_cast<const uint4*>(lo + off);
    const __nv_bfloat162* bp = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      r.v[2 * i] += __bfloat162float(bp[i].x);
      r.v[2 * i + 1] += __bfloat162float(bp[i].y);
    }
  }
  return r;
}

// STREAM: st.global.cs (evict-first).  ROI pooling writes 2.6 GB per batch while gathering from a 63 MB per-image
// feature map.  On an H100 (50 MB of L2) the map does not fit whole; evict-first stores keep the output stream from
// displacing the part of it that does, so that the bins of neighbouring ROIs still find their rows in L2.
template <bool STREAM = false>
__device__ __forceinline__ void store8(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t off, const Vec8& x) {
  uint4 a, b;
  __nv_bfloat162* ap = reinterpret_cast<__nv_bfloat162*>(&a);
  __nv_bfloat162* bp = reinterpret_cast<__nv_bfloat162*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(x.v[2 * i]), h1 = __float2bfloat16_rn(x.v[2 * i + 1]);
    ap[i] = __nv_bfloat162(h0, h1);
    bp[i] = __nv_bfloat162(__float2bfloat16_rn(x.v[2 * i] - __bfloat162float(h0)),
                           __float2bfloat16_rn(x.v[2 * i + 1] - __bfloat162float(h1)));
  }
  if (STREAM) {
    __stcs(reinterpret_cast<uint4*>(hi + off), a);
    if (lo) __stcs(reinterpret_cast<uint4*>(lo + off), b);
  } else {
    *reinterpret_cast<uint4*>(hi + off) = a;
    if (lo) *reinterpret_cast<uint4*>(lo + off) = b;
  }
}

// ------------------------------------------------------------------------------- Pooling
// PoolingLayer::Forward_cpu (src/caffe/layers/pooling_layer.cpp:128-220): windows start at o * stride - pad and are
// clipped to the image, so MAX never sees a padded position.  AVE divides by the window clipped to the PADDED extent
// (pool_size is taken with hend = min(hstart + kh, H + pad_h) before hstart / hend are clipped to [0, H], :196-204):
// padded positions count as zeros in the mean.  With pad 0 that is the clipped window itself.
struct PoolGeom {
  int kh, kw, sh, sw, ph, pw;
};
__global__ void pool_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                            __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int N, int H,
                            int W, int C, int Ho, int Wo, PoolGeom q, int mode, const int* __restrict__ dyn_n) {
  const int cg = C / 8;
  if (dyn_n) N = max(0, min(N, *dyn_n));  // data-dependent row count (mscnn_pool_forward_dyn)
  const size_t total = (size_t)N * Ho * Wo * cg;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int g = idx % cg;
    size_t r = idx / cg;
    const int ow = r % Wo; r /= Wo;
    const int oh = r % Ho;
    const int n = r / Ho;
    int hs = oh * q.sh - q.ph, ws = ow * q.sw - q.pw;
    int he = min(hs + q.kh, H + q.ph), we = min(ws + q.kw, W + q.pw);
    const float sz = (float)((he - hs) * (we - ws));
    hs = max(hs, 0); ws = max(ws, 0);
    he = min(he, H); we = min(we, W);
    Vec8 acc;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc.v[i] = (mode == MSCNN_POOL_MAX) ? -3.402823466e+38f : 0.f;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w) {
        const Vec8 v = load8(xh, xl, ((size_t)(n * H + h) * W + w) * C + g * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (mode == MSCNN_POOL_MAX) acc.v[i] = (v.v[i] > acc.v[i]) ? v.v[i] : acc.v[i];
          else acc.v[i] = acc.v[i] + v.v[i];
        }
      }
    if (mode == MSCNN_POOL_AVE) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc.v[i] = acc.v[i] / sz;
    }
    store8(yh, yl, ((size_t)(n * Ho + oh) * Wo + ow) * C + g * 8, acc);
  }
}

// Pooling whose one window is the whole image (global_pooling, or any kernel that covers the bottom): pool_kernel
// would walk a plane per thread.  Here a CTA owns one image and 8 consecutive 8-channel groups (128 contiguous bytes
// per pixel and plane); its 256 threads are 32 pixel slices x 8 groups, slice s taking pixels s, s + 32, ... with
// four loads in flight, and slice 0 then folds the 32 partial results in slice order.  MAX is exact in any order.
// AVE sums hi + lo in fp32 in that fixed order (deterministic), not the reference's row-major one: like the
// reference's, its mean lies within (H W - 1) 2^-24 mean|x| of the exact mean (plus the division's rounding), so the
// two differ by at most twice that (tests/test_faithful_planes_gpu.py holds the kernel to this order bit for bit and
// to the bound).
constexpr int kGlobalSlices = 32, kGlobalGroups = 8;
__global__ void __launch_bounds__(kGlobalSlices * kGlobalGroups)
global_pool_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                   __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int N, int HW, int C, int mode,
                   const int* __restrict__ dyn_n) {
  __shared__ Vec8 part[kGlobalSlices][kGlobalGroups];
  const int n = blockIdx.y;
  if (dyn_n && n >= *dyn_n) return;
  const int gl = threadIdx.x % kGlobalGroups, slice = threadIdx.x / kGlobalGroups;
  const int g = blockIdx.x * kGlobalGroups + gl;
  const bool live = g < C / 8;
  const bool is_max = mode == MSCNN_POOL_MAX;
  Vec8 acc;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc.v[i] = is_max ? -3.402823466e+38f : 0.f;
  auto fold = [&](const Vec8& v) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc.v[i] = is_max ? ((v.v[i] > acc.v[i]) ? v.v[i] : acc.v[i]) : acc.v[i] + v.v[i];
  };
  if (live) {
    const size_t base = (size_t)n * HW * C + g * 8;
    int px = slice;
    for (; px + 3 * kGlobalSlices < HW; px += 4 * kGlobalSlices) {
      Vec8 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = load8(xh, xl, base + (size_t)(px + u * kGlobalSlices) * C);
#pragma unroll
      for (int u = 0; u < 4; ++u) fold(v[u]);
    }
    for (; px < HW; px += kGlobalSlices) fold(load8(xh, xl, base + (size_t)px * C));
  }
  part[slice][gl] = acc;
  __syncthreads();
  if (slice != 0 || !live) return;
  const int used = min(HW, kGlobalSlices);  // slices beyond the pixel count hold the neutral element only
  for (int sl = 1; sl < used; ++sl) fold(part[sl][gl]);
  if (!is_max) {
    const float sz = (float)HW;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc.v[i] = acc.v[i] / sz;
  }
  store8(yh, yl, (size_t)n * C + g * 8, acc);
}

// --------------------------------------------------------------------------- ROIPooling
// ROIPoolingLayer::Forward_cpu (src/caffe/layers/roi_pooling_layer.cpp:49-139) including the
// MS-CNN pad_ratio context extension (:66-72).  Output rows are written at channel offset
// `c_off` of a [R][P][P][Cout_total] tensor, which fuses ConcatLayer (concat_layer.cpp:57-74).
// One warp per (ROI, output bin): the bin geometry is computed once per warp (uniform), lanes
// stride over the 8-channel groups so that every load / store is a 512-byte coalesced row segment.
// Up to four pad_ratio variants of the same ROI set are pooled by the same warp (MS-CNN pools every
// ROI twice, object and 1.5x context window, and concatenates): the context window contains the
// object window, so the second variant mostly hits lines the first one just touched.
// best[i] = max(best[i], hi[i] + lo[i]) for the 8 bf16 channels packed in `a` (+ `l` when has_lo)
__device__ __forceinline__ void max8(Vec8& best, const uint4& a, const uint4& l, bool has_lo) {
  const uint32_t ah[4] = {a.x, a.y, a.z, a.w}, al[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float v0 = __uint_as_float(ah[q] << 16), v1 = __uint_as_float(ah[q] & 0xFFFF0000u);
    if (has_lo) {
      v0 = v0 + __uint_as_float(al[q] << 16);
      v1 = v1 + __uint_as_float(al[q] & 0xFFFF0000u);
    }
    best.v[2 * q] = fmaxf(best.v[2 * q], v0);
    best.v[2 * q + 1] = fmaxf(best.v[2 * q + 1], v1);
  }
}

struct RoiVariants {
  int count;
  float pad_ratio[4];
  int c_off[4];
};

// Pools one (ROI, bin, variant) window for the channel groups g0 + lane (+ 32 when DUAL) and stores the result.
// The window is walked as one flattened pixel sequence in 16-byte units with 32-bit indices (the feature map has
// < 2^31 / 8 elements: checked by the launcher), two pixels per step, so up to eight 16-byte loads (hi, lo, second
// group) are in flight per lane: the kernel was bound by the latency of two.  fmaxf gives the
// reference's `if (x > max) max = x` result for every non-NaN input.  Stores are streaming (st.global.cs).
template <bool DUAL>
__device__ __forceinline__ void roi_pool_window(const uint4* __restrict__ xh4, const uint4* __restrict__ xl4, int base_idx,
                                                int npx, int bw, int row_skip, int cg, bool empty,
                                                __nv_bfloat16* yh, __nv_bfloat16* yl, size_t out_off) {
  const bool has_lo = xl4 != nullptr;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  Vec8 best0, best1;
#pragma unroll
  for (int i = 0; i < 8; ++i) best0.v[i] = best1.v[i] = empty ? 0.f : -3.402823466e+38f;
  int idx = base_idx;
  int wpos = 0;
  int k = 0;
  for (; k + 2 <= npx; k += 2) {
    int ix[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      ix[u] = idx;
      idx += cg;
      if (++wpos == bw) { wpos = 0; idx += row_skip; }
    }
    uint4 a[2], l[2], c[2], m[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      a[u] = __ldg(xh4 + ix[u]);
      l[u] = has_lo ? __ldg(xl4 + ix[u]) : z;
      if (DUAL) {
        c[u] = __ldg(xh4 + ix[u] + 32);
        m[u] = has_lo ? __ldg(xl4 + ix[u] + 32) : z;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      max8(best0, a[u], l[u], has_lo);
      if (DUAL) max8(best1, c[u], m[u], has_lo);
    }
  }
  if (k < npx) {
    max8(best0, __ldg(xh4 + idx), has_lo ? __ldg(xl4 + idx) : z, has_lo);
    if (DUAL) max8(best1, __ldg(xh4 + idx + 32), has_lo ? __ldg(xl4 + idx + 32) : z, has_lo);
  }
  store8<true>(yh, yl, out_off, best0);
  if (DUAL) store8<true>(yh, yl, out_off + 32 * 8, best1);
}

// One warp per (ROI, bin); a lane owns channel groups g and g + 32 (C = 512: all 64 groups in one visit).
// Other schedules tried: per-image half-channel passes (halve the L2 working set at the cost of a second walk over
// the ROIs), block-per-ROI (L1 sharing between the bins of one ROI), createpolicy evict_last loads / evict_first stores.
__global__ void roi_pool_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                                const float* __restrict__ rois, int R, int N, int H, int W, int C,
                                int PH, int PW, float scale, const RoiVariants var,
                                __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int Ctot,
                                const int* __restrict__ dyn_R) {
  const int cg = C / 8;
  const int lane = threadIdx.x & 31;
  const size_t warps_total = (size_t)gridDim.x * (blockDim.x >> 5);
  if (dyn_R) R = max(0, min(R, *dyn_R));  // data-dependent ROI count (mscnn_roi_pool_multi_forward_dyn)
  const size_t bins = (size_t)R * PH * PW;
  const uint4* xh4 = reinterpret_cast<const uint4*>(xh);
  const uint4* xl4 = reinterpret_cast<const uint4*>(xl);
  for (size_t bin = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); bin < bins; bin += warps_total) {
    const int pw = bin % PW;
    const int ph = (bin / PW) % PH;
    const int roi = bin / ((size_t)PW * PH);
    const float* q = rois + (size_t)roi * 5;
    int b = (int)q[0];
    b = min(max(b, 0), N - 1);  // the reference CHECKs the range (:63-64); never out of range here
    const float q1 = q[1], q2 = q[2], q3 = q[3], q4 = q[4];
    for (int vi = 0; vi < var.count; ++vi) {
      const float pad_w = (q3 - q1 + 1.f) * var.pad_ratio[vi];
      const float pad_h = (q4 - q2 + 1.f) * var.pad_ratio[vi];
      const int sw = (int)roundf((q1 - pad_w) * scale);
      const int sh = (int)roundf((q2 - pad_h) * scale);
      const int ew = (int)roundf((q3 + pad_w) * scale);
      const int eh = (int)roundf((q4 + pad_h) * scale);
      const int roi_h = max(eh - sh + 1, 1), roi_w = max(ew - sw + 1, 1);
      const float bin_h = (float)roi_h / (float)PH, bin_w = (float)roi_w / (float)PW;
      int hstart = (int)floorf((float)ph * bin_h);
      int wstart = (int)floorf((float)pw * bin_w);
      int hend = (int)ceilf((float)(ph + 1) * bin_h);
      int wend = (int)ceilf((float)(pw + 1) * bin_w);
      hstart = min(max(hstart + sh, 0), H);
      hend = min(max(hend + sh, 0), H);
      wstart = min(max(wstart + sw, 0), W);
      wend = min(max(wend + sw, 0), W);
      const bool empty = (hend <= hstart) || (wend <= wstart);
      const int bw = wend - wstart;
      const int npx = empty ? 0 : (hend - hstart) * bw;
      const int row_skip = (W - bw) * cg;
      const int base = ((b * H + hstart) * W + wstart) * cg;
      const size_t out = (size_t)bin * Ctot + var.c_off[vi];
      for (int g = lane; g < cg; g += 64) {
        if (g + 32 < cg) roi_pool_window<true>(xh4, xl4, base + g, npx, bw, row_skip, cg, empty, yh, yl, out + g * 8);
        else roi_pool_window<false>(xh4, xl4, base + g, npx, bw, row_skip, cg, empty, yh, yl, out + g * 8);
      }
    }
  }
}

// ------------------------------------------------------------------------------ ROIAlign
// ROIAlignLayer::Forward_cpu (src/caffe/layers/roi_align_layer.cpp:49-139; GPU twin
// roi_align_layer.cu:21-98): bilinear samples on the (PH+1) x (PW+1) GRID of bin corners of the
// (padded) ROI, in feature-map coordinates shifted by half a pixel.  Same work distribution as
// roi_pool_kernel: one warp per (ROI, grid point), lanes over 8-channel groups, so the four
// neighbour loads are coalesced 512-byte row segments.  fp32 arithmetic in the reference's order.
__global__ void roi_align_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                                 const float* __restrict__ rois, int R, int N, int H, int W, int C, int PH,
                                 int PW, float scale, float pad_ratio, __nv_bfloat16* __restrict__ yh,
                                 __nv_bfloat16* __restrict__ yl, int Ctot, int c_off, const int* __restrict__ dyn_R) {
  const int cg = C / 8;
  const int GH = PH + 1, GW = PW + 1;
  const int lane = threadIdx.x & 31;
  const size_t warps_total = (size_t)gridDim.x * (blockDim.x >> 5);
  if (dyn_R) R = max(0, min(R, *dyn_R));
  const size_t points = (size_t)R * GH * GW;
  for (size_t pt = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pt < points; pt += warps_total) {
    const int pw = pt % GW;
    const int ph = (pt / GW) % GH;
    const int roi = pt / ((size_t)GW * GH);
    const float* q = rois + (size_t)roi * 5;
    int b = (int)q[0];
    b = min(max(b, 0), N - 1);  // CHECKed by the reference (:63-64)
    // :67-81
    const float pad_w = (q[3] - q[1] + 1.f) * pad_ratio;
    const float pad_h = (q[4] - q[2] + 1.f) * pad_ratio;
    const float start_w = (q[1] - pad_w) * scale - 0.5f;
    const float start_h = (q[2] - pad_h) * scale - 0.5f;
    const float end_w = (q[3] + pad_w) * scale - 0.5f;
    const float end_h = (q[4] + pad_h) * scale - 0.5f;
    const float roi_h = end_h - start_h, roi_w = end_w - start_w;
    const float bin_h = roi_h / (float)PH, bin_w = roi_w / (float)PW;
    float hf = start_h + (float)ph * bin_h;
    float wf = start_w + (float)pw * bin_w;
    // malformed ROI (:94-97) or grid point outside the map (:104-108) -> 0
    const bool zero = (roi_h <= 0.f || roi_w <= 0.f) || hf < -0.5f || (double)hf > (double)H - 0.5 ||
                      wf < -0.5f || (double)wf > (double)W - 0.5;
    int h0 = (int)floorf(hf), w0 = (int)floorf(wf);
    int h1 = h0 + 1, w1 = w0 + 1;
    hf = fminf(fmaxf(hf, 0.f), (float)(H - 1));
    wf = fminf(fmaxf(wf, 0.f), (float)(W - 1));
    h0 = min(max(h0, 0), H - 1); w0 = min(max(w0, 0), W - 1);
    h1 = min(max(h1, 0), H - 1); w1 = min(max(w1, 0), W - 1);
    const float lh = hf - (float)h0, lw = wf - (float)w0;
    const float hh = 1.f - lh, hw = 1.f - lw;
    const float w00 = hw * hh, w10 = lw * hh, w01 = hw * lh, w11 = lw * lh;
    const size_t img = (size_t)b * H;
    for (int g = lane; g < cg; g += 32) {
      Vec8 r;
      if (zero) {
#pragma unroll
        for (int i = 0; i < 8; ++i) r.v[i] = 0.f;
      } else {
        const Vec8 v00 = load8(xh, xl, ((img + h0) * W + w0) * C + g * 8);
        const Vec8 v10 = load8(xh, xl, ((img + h0) * W + w1) * C + g * 8);
        const Vec8 v01 = load8(xh, xl, ((img + h1) * W + w0) * C + g * 8);
        const Vec8 v11 = load8(xh, xl, ((img + h1) * W + w1) * C + g * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i)  // :131 left-to-right
          r.v[i] = ((w00 * v00.v[i] + w10 * v10.v[i]) + w01 * v01.v[i]) + w11 * v11.v[i];
      }
      store8(yh, yl, pt * Ctot + c_off + g * 8, r);
    }
  }
}

// ------------------------------------------------------------ depthwise Deconvolution
// DeconvolutionLayer::Forward_cpu (src/caffe/layers/deconv_layer.cpp:25-40) with group == channels == num_output,
// e.g. the bilinear up-sampling of the MS-CNN "-2x" nets (kernel 4, stride 2, pad 1, no bias;
// examples/kitti_car/mscnn-7s-576-2x/mscnn_deploy.prototxt:452-466):
//   y[n, c, s_h iy - p_h + ky d_h, s_w ix - p_w + kx d_w] += x[n, c, iy, ix] * w[c, ky, kx],  then + bias[c]
// Gather form: output row oy is reached by the taps ky with (oy + p_h - ky d_h) mod s_h == 0, which start at
// ky0[(oy + p_h) mod s_h] and lie s_h / gcd(s_h, d_h) apart (likewise in x).  Weights are read from the layer blob
// (the bilinear filler is just the usual content, filler.hpp:248-258).
struct DwDeconvGeom {
  int KH, KW, sh, sw, ph, pw, dh, dw;
  int step_h, step_w;                          // s / gcd(s, d): distance between the taps of one output phase
  int ky0[8], kx0[8];                          // first tap of phase (o + p) mod s; KH / KW when none reaches it
};

// Every block stages the taps of its slice of channel groups [g0, g0 + cgs) (blockIdx.y) as
// w_s[(tap * 8 + i) * cgs + g - g0] (channel c = 8 g + i): a warp reads consecutive g, so the reads are
// conflict-free.  (Reading wt[c * taps + tap] from global memory cost scattered 4-byte loads per thread, many times
// the layer's HBM time.)  Wide kernels on many channels take several slices, so the staging fits shared memory.
// K > 0: the geometry is fixed at compile time to K x K, stride S, pad P, dilation 1 (the -2x nets' 4 / 2 / 1 layer):
// constant divisors and tap steps keep its index arithmetic as cheap as a kernel written for that shape alone.
template <int K, int S, int P>
__global__ void deconv_depthwise_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                                        const float* __restrict__ wt /*[Creal][KH][KW]*/,
                                        const float* __restrict__ bias /*[Creal] or NULL*/,
                                        __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, int N, int H,
                                        int W, int C, int Creal, int Ho, int Wo, int cgs, const DwDeconvGeom q) {
  constexpr bool kFixed = K > 0;
  const int KH = kFixed ? K : q.KH, KW = kFixed ? K : q.KW, sh = kFixed ? S : q.sh, sw = kFixed ? S : q.sw;
  const int ph = kFixed ? P : q.ph, pw = kFixed ? P : q.pw, dh = kFixed ? 1 : q.dh, dw = kFixed ? 1 : q.dw;
  const int step_h = kFixed ? S : q.step_h, step_w = kFixed ? S : q.step_w;
  extern __shared__ float w_s[];
  const int cg = C / 8, taps = KH * KW;
  const int g0 = blockIdx.y * cgs;
  for (int j = threadIdx.x; j < taps * 8 * cgs; j += blockDim.x) {
    const int g = g0 + j % cgs, i = (j / cgs) % 8, tap = j / (8 * cgs);
    const int c = g * 8 + i;
    w_s[j] = (g < cg && c < Creal) ? wt[c * taps + tap] : 0.f;
  }
  __syncthreads();
  const size_t total = (size_t)N * Ho * Wo * cgs;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int gl = idx % cgs, g = g0 + gl;
    size_t r = idx / cgs;
    const int ox = r % Wo; r /= Wo;
    const int oy = r % Ho;
    const int n = r / Ho;
    if (g >= cg) continue;
    Vec8 acc;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc.v[i] = 0.f;
    // The reference's col2im adds the kernel offsets in increasing (ky, kx) order (util/im2col.cpp:col2im_cpu), so
    // do we; taps that fall outside the input are skipped.  With dilation 1 the first tap of output row oy is
    // (oy + p) mod s.
    for (int ky = kFixed ? (int)((unsigned)(oy + P) % S) : q.ky0[(oy + ph) % sh]; ky < KH; ky += step_h) {
      const int ny = oy + ph - ky * dh;
      const int iy = ny / sh;
      if (ny < 0 || iy >= H) continue;
      for (int kx = kFixed ? (int)((unsigned)(ox + P) % S) : q.kx0[(ox + pw) % sw]; kx < KW; kx += step_w) {
        const int nx = ox + pw - kx * dw;
        const int ix = nx / sw;
        if (nx < 0 || ix >= W) continue;
        const Vec8 v = load8(xh, xl, ((size_t)(n * H + iy) * W + ix) * C + g * 8);
        const float* wp = w_s + (size_t)((ky * KW + kx) * 8) * cgs + gl;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc.v[i] = acc.v[i] + v.v[i] * wp[i * cgs];
      }
    }
    if (bias != nullptr) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (g * 8 + i < Creal) acc.v[i] = acc.v[i] + __ldg(bias + g * 8 + i);
    }
    store8(yh, yl, ((size_t)(n * Ho + oy) * Wo + ox) * C + g * 8, acc);
  }
}

// ------------------------------------------------------------------ stand-alone ReLU / Concat
// Used only when a ReLU / Concat layer is run unfused (outside mscnn_b200's Net, which folds
// ReLU into the producing convolution and Concat into ROIPooling).
// relu(hi + lo): |lo| <= ulp(hi)/2, so the sign of the sum is the sign of hi.
__global__ void relu_planes_kernel(__nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, size_t n8) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    uint4 a = reinterpret_cast<uint4*>(hi)[i];
    uint4 b = lo ? reinterpret_cast<uint4*>(lo)[i] : make_uint4(0, 0, 0, 0);
    uint32_t* ap = reinterpret_cast<uint32_t*>(&a);
    uint32_t* bp = reinterpret_cast<uint32_t*>(&b);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (ap[k] & 0x00008000u) { ap[k] &= 0xFFFF0000u; bp[k] &= 0xFFFF0000u; }   // low element negative
      if (ap[k] & 0x80000000u) { ap[k] &= 0x0000FFFFu; bp[k] &= 0x0000FFFFu; }   // high element negative
    }
    reinterpret_cast<uint4*>(hi)[i] = a;
    if (lo) reinterpret_cast<uint4*>(lo)[i] = b;
  }
}
__global__ void relu_f32_kernel(float* __restrict__ x, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    x[i] = fmaxf(x[i], 0.f);
}
// y[p][off .. off+C) = x[p][0 .. C) for every pixel p (channel concat of NHWC planes)
__global__ void concat_planes_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                     size_t pixels, int C, int Ctot, int off) {
  const int cg = C / 8;
  const size_t total = pixels * cg;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i / cg;
    const int g = i % cg;
    *reinterpret_cast<uint4*>(y + p * Ctot + off + g * 8) = *reinterpret_cast<const uint4*>(x + p * C + g * 8);
  }
}

static int launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn: %s launch failed: %s\n", what, cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

static int grid_for(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  const size_t cap = (size_t)mscnn_sm_count() * 16;  // 16 resident 256-thread CTAs per SM at most
  if (b > cap) b = cap;
  return (int)(b ? b : 1);
}

}  // namespace mscnn

using namespace mscnn;

extern "C" int mscnn_pool_output_size(int in, int kernel, int stride, int pad) {
  if (in <= 0 || kernel <= 0 || stride <= 0 || pad < 0 || pad >= kernel) return MSCNN_ERR_INVALID;
  int out = (in + 2 * pad - kernel + stride - 1) / stride + 1;
  if (pad > 0 && (out - 1) * stride >= in + pad) --out;  // the last window must start in the image or the left padding
  return out >= 1 ? out : MSCNN_ERR_INVALID;
}

extern "C" int mscnn_pool2d_forward_dyn(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H,
                                        int W, int C, int kernel_h, int kernel_w, int stride_h, int stride_w,
                                        int pad_h, int pad_w, int mode, const int* dyn_n, void* stream) {
  if (!x_hi || !y_hi || N <= 0 || C <= 0 || C % 8) return MSCNN_ERR_INVALID;
  if ((x_lo == nullptr) != (y_lo == nullptr)) return MSCNN_ERR_INVALID;
  if (mode != MSCNN_POOL_MAX && mode != MSCNN_POOL_AVE) return MSCNN_ERR_INVALID;
  const int Ho = mscnn_pool_output_size(H, kernel_h, stride_h, pad_h);
  const int Wo = mscnn_pool_output_size(W, kernel_w, stride_w, pad_w);
  if (Ho <= 0 || Wo <= 0) return MSCNN_ERR_INVALID;
  const __nv_bfloat16 *xh = (const __nv_bfloat16*)x_hi, *xl = (const __nv_bfloat16*)x_lo;
  __nv_bfloat16 *yh = (__nv_bfloat16*)y_hi, *yl = (__nv_bfloat16*)y_lo;
  mscnn::note_launch();
  // one unpadded window over a whole image of at least a pixel per slice: the CTA-wide reduction
  if (Ho == 1 && Wo == 1 && pad_h == 0 && pad_w == 0 && (long long)H * W >= kGlobalSlices && N <= 65535 &&
      (long long)H * W <= 2147483647ll) {
    const dim3 grid((C / 8 + kGlobalGroups - 1) / kGlobalGroups, N);
    global_pool_kernel<<<grid, kGlobalSlices * kGlobalGroups, 0, (cudaStream_t)stream>>>(xh, xl, yh, yl, N, H * W, C,
                                                                                         mode, dyn_n);
    return launch_check("global_pool");
  }
  const size_t total = (size_t)N * Ho * Wo * (C / 8);
  const PoolGeom q = {kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w};
  pool_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(xh, xl, yh, yl, N, H, W, C, Ho, Wo, q, mode,
                                                                     dyn_n);
  return launch_check("pool");
}

extern "C" int mscnn_pool_forward_dyn(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H,
                                      int W, int C, int kernel, int stride, int mode, const int* dyn_n, void* stream) {
  return mscnn_pool2d_forward_dyn(x_hi, x_lo, y_hi, y_lo, N, H, W, C, kernel, kernel, stride, stride, 0, 0, mode,
                                  dyn_n, stream);
}

extern "C" int mscnn_pool_forward(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H,
                                  int W, int C, int kernel, int stride, int mode, void* stream) {
  return mscnn_pool_forward_dyn(x_hi, x_lo, y_hi, y_lo, N, H, W, C, kernel, stride, mode, nullptr, stream);
}

extern "C" int mscnn_roi_pool_multi_forward_dyn(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                                const float* rois, int R, int pooled_h, int pooled_w,
                                                float spatial_scale, int num_variants, const float* pad_ratios,
                                                const int* out_channel_offsets, void* y_hi, void* y_lo,
                                                int out_channels_total, const int* dyn_R, void* stream) {
  if (!x_hi || !y_hi || !rois || !pad_ratios || !out_channel_offsets || N <= 0 || C % 8 || R < 0 ||
      pooled_h <= 0 || pooled_w <= 0 || out_channels_total % 8 || num_variants < 1 || num_variants > 4)
    return MSCNN_ERR_INVALID;
  // split input and split output go together, as in every other plane entry: the kernel would otherwise store the
  // rounded hi alone of an fp32-faithful input, or a lo plane of zeros
  if ((x_lo == nullptr) != (y_lo == nullptr)) return MSCNN_ERR_INVALID;
  RoiVariants var;
  var.count = num_variants;
  for (int i = 0; i < num_variants; ++i) {
    if (out_channel_offsets[i] % 8 || out_channel_offsets[i] + C > out_channels_total) return MSCNN_ERR_INVALID;
    var.pad_ratio[i] = pad_ratios[i];
    var.c_off[i] = out_channel_offsets[i];
  }
  if (R == 0) return MSCNN_OK;
  if ((size_t)N * H * W * (C / 8) >= (size_t)1 << 31) return MSCNN_ERR_INVALID;  // 32-bit 16-byte indices in the kernel
  const size_t total = (size_t)R * pooled_h * pooled_w * 32;  // one warp per (ROI, bin)
  mscnn::note_launch();
  roi_pool_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, rois, R, N, H, W, C, pooled_h, pooled_w,
      spatial_scale, var, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, out_channels_total, dyn_R);
  return launch_check("roi_pool");
}

extern "C" int mscnn_roi_pool_multi_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                            const float* rois, int R, int pooled_h, int pooled_w,
                                            float spatial_scale, int num_variants, const float* pad_ratios,
                                            const int* out_channel_offsets, void* y_hi, void* y_lo,
                                            int out_channels_total, void* stream) {
  return mscnn_roi_pool_multi_forward_dyn(x_hi, x_lo, N, H, W, C, rois, R, pooled_h, pooled_w, spatial_scale,
                                          num_variants, pad_ratios, out_channel_offsets, y_hi, y_lo, out_channels_total,
                                          nullptr, stream);
}

extern "C" int mscnn_roi_pool_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                      const float* rois, int R, int pooled_h, int pooled_w,
                                      float spatial_scale, float pad_ratio, void* y_hi, void* y_lo,
                                      int out_channels_total, int out_channel_offset, void* stream) {
  return mscnn_roi_pool_multi_forward(x_hi, x_lo, N, H, W, C, rois, R, pooled_h, pooled_w, spatial_scale, 1,
                                      &pad_ratio, &out_channel_offset, y_hi, y_lo, out_channels_total, stream);
}

extern "C" int mscnn_roi_align_forward_dyn(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                           const float* rois, int R, int pooled_h, int pooled_w,
                                           float spatial_scale, float pad_ratio, void* y_hi, void* y_lo,
                                           int out_channels_total, int out_channel_offset, const int* dyn_R,
                                           void* stream) {
  if (!x_hi || !y_hi || !rois || N <= 0 || H <= 0 || W <= 0 || C % 8 || R < 0 || pooled_h <= 0 || pooled_w <= 0 ||
      out_channels_total % 8 || out_channel_offset % 8 || out_channel_offset + C > out_channels_total)
    return MSCNN_ERR_INVALID;
  if ((x_lo == nullptr) != (y_lo == nullptr)) return MSCNN_ERR_INVALID;
  if (R == 0) return MSCNN_OK;
  const size_t total = (size_t)R * (pooled_h + 1) * (pooled_w + 1) * 32;  // one warp per (ROI, grid point)
  mscnn::note_launch();
  roi_align_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, rois, R, N, H, W, C, pooled_h, pooled_w,
      spatial_scale, pad_ratio, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, out_channels_total,
      out_channel_offset, dyn_R);
  return launch_check("roi_align");
}

extern "C" int mscnn_roi_align_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                       const float* rois, int R, int pooled_h, int pooled_w,
                                       float spatial_scale, float pad_ratio, void* y_hi, void* y_lo,
                                       int out_channels_total, int out_channel_offset, void* stream) {
  return mscnn_roi_align_forward_dyn(x_hi, x_lo, N, H, W, C, rois, R, pooled_h, pooled_w, spatial_scale, pad_ratio,
                                     y_hi, y_lo, out_channels_total, out_channel_offset, nullptr, stream);
}

extern "C" int mscnn_deconv_depthwise_forward(const void* x_hi, const void* x_lo, const float* w, const float* bias,
                                              void* y_hi, void* y_lo, int N, int H, int W, int C, int Creal, int KH,
                                              int KW, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                              int dil_w, void* stream) {
  if (!x_hi || !y_hi || !w || N <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || Creal <= 0 || Creal > C)
    return MSCNN_ERR_INVALID;
  if ((x_lo == nullptr) != (y_lo == nullptr)) return MSCNN_ERR_INVALID;
  if (!deconv_axis_ok(KH, stride_h, pad_h, dil_h) || !deconv_axis_ok(KW, stride_w, pad_w, dil_w)) {
    fprintf(stderr, "mscnn_deconv_depthwise_forward: kernel %dx%d, stride %dx%d, pad %dx%d, dilation %dx%d: strides "
            "1..8, pad >= 0 and dilation >= 1 with a reach up to 2^20 are served\n", KH, KW, stride_h, stride_w, pad_h,
            pad_w, dil_h, dil_w);
    return MSCNN_ERR_INVALID;
  }
  const int Ho = deconv_out_size(H, KH, stride_h, pad_h, dil_h), Wo = deconv_out_size(W, KW, stride_w, pad_w, dil_w);
  if (Ho <= 0 || Wo <= 0) return MSCNN_ERR_INVALID;
  DwDeconvGeom q = {KH, KW, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, 1, {}, {}};
  for (int r = 0; r < 8; ++r) {
    // phase r of (o + p) mod s: the axes' first taps (deconv_axis with p = 0 counts phases of o + p)
    const DeconvAxis ay = deconv_axis(KH, stride_h, 0, dil_h, 0, r % stride_h);
    const DeconvAxis ax = deconv_axis(KW, stride_w, 0, dil_w, 0, r % stride_w);
    q.ky0[r] = ay.taps ? ay.t0 : KH;
    q.kx0[r] = ax.taps ? ax.t0 : KW;
    q.step_h = ay.tstep;
    q.step_w = ax.tstep;
  }
  // channel-group slices whose staged taps fit 64 KB
  const int cg = C / 8, taps = KH * KW;
  const long long per_group = (long long)taps * 8 * sizeof(float);
  if (per_group > 64 * 1024) return MSCNN_ERR_INVALID;  // a kernel of more than 2048 taps
  const int max_groups = (int)((64 * 1024) / per_group);
  const int slices = (cg + max_groups - 1) / max_groups, cgs = (cg + slices - 1) / slices;
  if (slices > 65535) return MSCNN_ERR_INVALID;
  const size_t w_smem = (size_t)per_group * cgs;
  const bool shipped = KH == 4 && KW == 4 && stride_h == 2 && stride_w == 2 && pad_h == 1 && pad_w == 1 && dil_h == 1 &&
                       dil_w == 1;
  auto kern = shipped ? deconv_depthwise_kernel<4, 2, 1> : deconv_depthwise_kernel<0, 0, 0>;
  if (w_smem > 48 * 1024 &&
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024) != cudaSuccess)
    return MSCNN_ERR_CUDA;
  const size_t total = (size_t)N * Ho * Wo * cgs;
  mscnn::note_launch();
  kern<<<dim3(grid_for(total, 256), slices), 256, w_smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, w, bias, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, N,
      H, W, C, Creal, Ho, Wo, cgs, q);
  return launch_check("deconv_depthwise");
}

extern "C" int mscnn_deconv2x_forward(const void* x_hi, const void* x_lo, const float* w, void* y_hi,
                                      void* y_lo, int N, int H, int W, int C, int Creal, void* stream) {
  return mscnn_deconv_depthwise_forward(x_hi, x_lo, w, nullptr, y_hi, y_lo, N, H, W, C, Creal, 4, 4, 2, 2, 1, 1, 1, 1,
                                        stream);
}

extern "C" int mscnn_relu_planes(void* hi, void* lo, size_t count, void* stream) {
  if (!hi || count % 8) return MSCNN_ERR_INVALID;
  if (count == 0) return MSCNN_OK;
  mscnn::note_launch();
  relu_planes_kernel<<<grid_for(count / 8, 256), 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)hi,
                                                                                 (__nv_bfloat16*)lo, count / 8);
  return launch_check("relu_planes");
}

extern "C" int mscnn_relu_f32(float* x, size_t count, void* stream) {
  if (!x) return MSCNN_ERR_INVALID;
  if (count == 0) return MSCNN_OK;
  mscnn::note_launch();
  relu_f32_kernel<<<grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>(x, count);
  return launch_check("relu_f32");
}

extern "C" int mscnn_concat_planes(const void* x, void* y, size_t pixels, int C, int Ctot, int offset,
                                   void* stream) {
  if (!x || !y || C % 8 || Ctot % 8 || offset % 8 || offset + C > Ctot) return MSCNN_ERR_INVALID;
  if (pixels == 0) return MSCNN_OK;
  mscnn::note_launch();
  concat_planes_kernel<<<grid_for(pixels * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, (__nv_bfloat16*)y, pixels, C, Ctot, offset);
  return launch_check("concat_planes");
}
