// Layout converters and weight packers (HBM-bound, coalesced on both sides through a
// shared-memory transpose).  See include/mscnn_b200.h for the contracts.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "deconv_phase.h"
#include "mscnn_b200.h"
#include "launch_count.h"

namespace mscnn {

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// grid: ceil(W/32) * H * N * ceil(Cpad/64) blocks (linear); block 256 = 8 warps.
// read:  x[n][c][h][w0..w0+31]  (lanes along w, warps along c)       -> coalesced 128 B
// write: hi[n][h][w][c0..c0+63] (lanes along c pairs, warps along w) -> coalesced 128 B
__global__ void nchw_to_planes_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                      __nv_bfloat16* __restrict__ lo, int N, int C, int H, int W,
                                      int Cpad) {
  __shared__ float tile[64][33];
  // linear block index over (n, c block, h, w block): grid.x only (up to 2^31 - 1 blocks; the fc6 blob of a
  // full-size batch has R * 64 = 100k+ (n, c block) pairs, more than grid.z or grid.y can hold)
  const int cblocks = Cpad / 64, wblocks = (W + 31) / 32;
  unsigned bid = blockIdx.x;
  const int w0 = static_cast<int>(bid % wblocks) * 32;
  bid /= wblocks;
  const int h = static_cast<int>(bid % H);
  bid /= H;
  const int n = static_cast<int>(bid / cblocks), c0 = static_cast<int>(bid % cblocks) * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int cc = warp; cc < 64; cc += 8) {
    const int c = c0 + cc, w = w0 + lane;
    float v = 0.f;
    if (c < C && w < W) v = x[((size_t)(n * C + c) * H + h) * W + w];
    tile[cc][lane] = v;
  }
  __syncthreads();
  for (int ww = warp; ww < 32; ww += 8) {
    const int w = w0 + ww;
    if (w >= W) continue;
    const float v0 = tile[2 * lane][ww], v1 = tile[2 * lane + 1][ww];
    __nv_bfloat16 h0, l0, h1, l1;
    split_bf16(v0, h0, l0);
    split_bf16(v1, h1, l1);
    const size_t o = ((size_t)(n * H + h) * W + w) * Cpad + c0 + 2 * lane;
    *reinterpret_cast<__nv_bfloat162*>(hi + o) = __nv_bfloat162(h0, h1);
    if (lo) *reinterpret_cast<__nv_bfloat162*>(lo + o) = __nv_bfloat162(l0, l1);
  }
}

__global__ void planes_to_nchw_kernel(const __nv_bfloat16* __restrict__ hi,
                                      const __nv_bfloat16* __restrict__ lo, float* __restrict__ y,
                                      int N, int C, int H, int W, int Cpad) {
  __shared__ float tile[64][33];
  // linear block index over (n, c block, h, w block): grid.x only (up to 2^31 - 1 blocks; the fc6 blob of a
  // full-size batch has R * 64 = 100k+ (n, c block) pairs, more than grid.z or grid.y can hold)
  const int cblocks = Cpad / 64, wblocks = (W + 31) / 32;
  unsigned bid = blockIdx.x;
  const int w0 = static_cast<int>(bid % wblocks) * 32;
  bid /= wblocks;
  const int h = static_cast<int>(bid % H);
  bid /= H;
  const int n = static_cast<int>(bid / cblocks), c0 = static_cast<int>(bid % cblocks) * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int ww = warp; ww < 32; ww += 8) {
    const int w = w0 + ww;
    float v0 = 0.f, v1 = 0.f;
    if (w < W) {
      const size_t o = ((size_t)(n * H + h) * W + w) * Cpad + c0 + 2 * lane;
      const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(hi + o);
      v0 = __bfloat162float(a.x);
      v1 = __bfloat162float(a.y);
      if (lo) {
        const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(lo + o);
        v0 += __bfloat162float(b.x);
        v1 += __bfloat162float(b.y);
      }
    }
    tile[2 * lane][ww] = v0;
    tile[2 * lane + 1][ww] = v1;
  }
  __syncthreads();
  for (int cc = warp; cc < 64; cc += 8) {
    const int c = c0 + cc, w = w0 + lane;
    if (c < C && w < W) y[((size_t)(n * C + c) * H + h) * W + w] = tile[cc][lane];
  }
}

// One deconvolution output phase's sub-kernel (deconv_phase.h) from the Caffe blob [Cin][Cout / group][KH][KW]:
//   out[((co m_h + uh) m_w + uw) cin_gp + ci] = w[k cin_g + ci][co - k cout_g][t0_h + (m_h - 1 - uh) step_h]
//                                                [t0_w + (m_w - 1 - uw) step_w],   k = co / cout_g,
// input and output channels swapped and the taps reversed; zero for co >= Cout or ci >= cin_g.
__global__ void pack_deconv_w_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi,
                                     __nv_bfloat16* __restrict__ lo, int Cout, int cin_g, int cout_g, int KH, int KW,
                                     int Cout_pad, int cin_gp, DeconvAxis ah, DeconvAxis aw) {
  const size_t total = (size_t)Cout_pad * ah.taps * aw.taps * cin_gp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int ci = i % cin_gp;
    size_t r = i / cin_gp;
    const int uw = r % aw.taps;
    r /= aw.taps;
    const int uh = r % ah.taps;
    const int co = r / ah.taps;
    float v = 0.f;
    if (co < Cout && ci < cin_g) {
      const int k = co / cout_g;
      const int th = ah.t0 + (ah.taps - 1 - uh) * ah.tstep, tw = aw.t0 + (aw.taps - 1 - uw) * aw.tstep;
      v = w[(((size_t)(k * cin_g + ci) * cout_g + (co - k * cout_g)) * KH + th) * KW + tw];
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

// out[(co*KH*KW + tap)*Cin_pad + ci] = w[((co*Cin + ci)*KH*KW) + tap]
__global__ void pack_conv_w_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi,
                                   __nv_bfloat16* __restrict__ lo, int Cout, int Cin, int taps,
                                   int Cout_pad, int Cin_pad) {
  const size_t total = (size_t)Cout_pad * taps * Cin_pad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int ci = i % Cin_pad;
    const int tap = (i / Cin_pad) % taps;
    const int co = i / ((size_t)Cin_pad * taps);
    float v = 0.f;
    if (co < Cout && ci < Cin) v = w[((size_t)co * Cin + ci) * taps + tap];
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

// out[no][(hw)*Cpad + c] = w[no][c*HW + hw]
__global__ void pack_fc_w_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi,
                                 __nv_bfloat16* __restrict__ lo, int Nout, int C, int HW,
                                 int Nout_pad, int Cpad) {
  const size_t total = (size_t)Nout_pad * HW * Cpad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int c = i % Cpad;
    const int hw = (i / Cpad) % HW;
    const int no = i / ((size_t)Cpad * HW);
    float v = 0.f;
    if (no < Nout && c < C) v = w[(size_t)no * C * HW + (size_t)c * HW + hw];
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

// out[n = dx*Cout + co][dy][ci] = w[co][ci][dy][dx]  (rows beyond k*Cout and channels beyond Cin are zero)
__global__ void pack_head_w_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi,
                                   __nv_bfloat16* __restrict__ lo, int Cout, int Cin, int k, int N_pad,
                                   int Cin_pad) {
  const size_t total = (size_t)N_pad * k * Cin_pad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int ci = i % Cin_pad;
    const int dy = (i / Cin_pad) % k;
    const int n = i / ((size_t)Cin_pad * k);
    float v = 0.f;
    if (n < k * Cout && ci < Cin) {
      const int dx = n / Cout, co = n - dx * Cout;
      v = w[(((size_t)co * Cin + ci) * k + dy) * k + dx];
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

// y[n][co][h][w] = bias[co] + sum_dx P[(n, h, w + dx - pad)][dx*COUT + co]; one thread per output pixel,
// a warp covers 32 consecutive w so every P row is touched by k neighbouring lanes.
template <int COUT>
__global__ void head_gather_kernel(const float* __restrict__ P, int ld, const float* __restrict__ bias,
                                   float* __restrict__ y, int N, int H, int W, int k, int pad) {
  const size_t total = (size_t)N * H * W;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int w = idx % W;
  const size_t row0 = idx - w;  // pixel index of (n, h, 0)
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  for (int dx = 0; dx < k; ++dx) {
    const int ww = w + dx - pad;
    if (ww < 0 || ww >= W) continue;
    const float* src = P + (row0 + ww) * ld + dx * COUT;
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = acc[c] + src[c];
  }
  const size_t plane = (size_t)H * W;
  const size_t n = idx / plane, hw = idx - n * plane;
#pragma unroll
  for (int c = 0; c < COUT; ++c) y[(n * COUT + c) * plane + hw] = acc[c] + bias[c];
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn: %s launch failed: %s\n", what, cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

}  // namespace mscnn

using namespace mscnn;

extern "C" const char* mscnn_version(void) { return "mscnn_b200 0.1 (sm_90a)"; }

extern "C" int mscnn_nchw_f32_to_planes(const float* x, void* hi, void* lo, int N, int C, int H,
                                        int W, int Cpad, void* stream) {
  if (!x || !hi || N <= 0 || C <= 0 || H <= 0 || W <= 0 || Cpad % 64 || Cpad < C)
    return MSCNN_ERR_INVALID;
  const long long nblocks = (long long)((W + 31) / 32) * H * N * (Cpad / 64);
  if (nblocks > 2147483647ll) return MSCNN_ERR_INVALID;
  const unsigned grid = static_cast<unsigned>(nblocks);
  mscnn::note_launch();
  nchw_to_planes_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      x, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, N, C, H, W, Cpad);
  return check_launch("nchw_to_planes");
}

extern "C" int mscnn_planes_to_nchw_f32(const void* hi, const void* lo, float* y, int N, int C,
                                        int H, int W, int Cpad, void* stream) {
  if (!y || !hi || N <= 0 || C <= 0 || H <= 0 || W <= 0 || Cpad % 64 || Cpad < C)
    return MSCNN_ERR_INVALID;
  const long long nblocks = (long long)((W + 31) / 32) * H * N * (Cpad / 64);
  if (nblocks > 2147483647ll) return MSCNN_ERR_INVALID;
  const unsigned grid = static_cast<unsigned>(nblocks);
  mscnn::note_launch();
  planes_to_nchw_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)hi, (const __nv_bfloat16*)lo, y, N, C, H, W, Cpad);
  return check_launch("planes_to_nchw");
}

extern "C" int mscnn_pack_conv_weights(const float* w, void* hi, void* lo, int Cout, int Cin, int KH,
                                       int KW, int Cout_pad, int Cin_pad, void* stream) {
  if (!w || !hi || Cout <= 0 || Cin <= 0 || Cout_pad < Cout || Cin_pad < Cin || Cin_pad % 64)
    return MSCNN_ERR_INVALID;
  const size_t total = (size_t)Cout_pad * KH * KW * Cin_pad;
  const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  mscnn::note_launch();
  pack_conv_w_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      w, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, Cout, Cin, KH * KW, Cout_pad, Cin_pad);
  return check_launch("pack_conv_w");
}

extern "C" long long mscnn_deconv_packed_elems(int Cin, int Cout, int group, int KH, int KW, int stride_h, int stride_w,
                                               int pad_h, int pad_w, int dil_h, int dil_w, int Cout_pad) {
  if (Cout < 1 || group < 1 || Cout % group || Cout_pad < Cout) return -1;
  return mscnn::deconv_phase_offset(Cin, group, KH, KW, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, Cout_pad,
                                    stride_h * stride_w);
}

extern "C" int mscnn_pack_deconv_weights(const float* w, void* hi, void* lo, int Cin, int Cout, int group, int KH,
                                         int KW, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                         int dil_w, int Cout_pad, void* stream) {
  if (!w || !hi || mscnn_deconv_packed_elems(Cin, Cout, group, KH, KW, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                                             Cout_pad) < 0)
    return MSCNN_ERR_INVALID;
  const int cin_g = Cin / group, cin_gp = (cin_g + 63) / 64 * 64;
  for (int i = 0; i < stride_h * stride_w; ++i) {
    const DeconvAxis ah = deconv_axis(KH, stride_h, pad_h, dil_h, 0, i / stride_w);
    const DeconvAxis aw = deconv_axis(KW, stride_w, pad_w, dil_w, 0, i % stride_w);
    if (ah.taps == 0 || aw.taps == 0) continue;
    const long long off = deconv_phase_offset(Cin, group, KH, KW, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                                              Cout_pad, i);
    const size_t total = (size_t)Cout_pad * ah.taps * aw.taps * cin_gp;
    const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
    mscnn::note_launch();
    pack_deconv_w_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
        w, (__nv_bfloat16*)hi + off, lo ? (__nv_bfloat16*)lo + off : nullptr, Cout, cin_g, Cout / group, KH, KW,
        Cout_pad, cin_gp, ah, aw);
    const int rc = check_launch("pack_deconv_w");
    if (rc != MSCNN_OK) return rc;
  }
  return MSCNN_OK;
}

extern "C" int mscnn_pack_fc_weights(const float* w, void* hi, void* lo, int Nout, int C, int H,
                                     int W, int Nout_pad, int Cpad, void* stream) {
  if (!w || !hi || Nout <= 0 || C <= 0 || Nout_pad < Nout || Cpad < C || Cpad % 64)
    return MSCNN_ERR_INVALID;
  const size_t total = (size_t)Nout_pad * H * W * Cpad;
  const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  mscnn::note_launch();
  pack_fc_w_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      w, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, Nout, C, H * W, Nout_pad, Cpad);
  return check_launch("pack_fc_w");
}

extern "C" int mscnn_pack_head_weights(const float* w, void* hi, void* lo, int Cout, int Cin, int k, int N_pad,
                                       int Cin_pad, void* stream) {
  if (!w || !hi || Cout <= 0 || Cin <= 0 || k <= 0 || N_pad < k * Cout || Cin_pad < Cin || Cin_pad % 64)
    return MSCNN_ERR_INVALID;
  const size_t total = (size_t)N_pad * k * Cin_pad;
  const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  mscnn::note_launch();
  pack_head_w_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, Cout,
                                                              Cin, k, N_pad, Cin_pad);
  return check_launch("pack_head_w");
}

extern "C" int mscnn_head_gather(const float* P, int ld, const float* bias, float* y, int N, int H, int W,
                                 int Cout, int k, int pad, void* stream) {
  if (!P || !bias || !y || N <= 0 || H <= 0 || W <= 0 || k <= 0 || ld < k * Cout) return MSCNN_ERR_INVALID;
  const size_t total = (size_t)N * H * W;
  const unsigned blocks = (unsigned)((total + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  switch (Cout) {
    case 6: mscnn::note_launch(); head_gather_kernel<6><<<blocks, 128, 0, st>>>(P, ld, bias, y, N, H, W, k, pad); break;
    case 9: mscnn::note_launch(); head_gather_kernel<9><<<blocks, 128, 0, st>>>(P, ld, bias, y, N, H, W, k, pad); break;
    default: return MSCNN_ERR_INVALID;  // the MS-CNN heads have cls_num + 4 = 6 or 9 channels
  }
  return check_launch("head_gather");
}
