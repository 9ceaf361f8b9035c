// conv1_1 (3 -> 64 channels, 3x3, pad 1) as ONE kernel: fp32 NCHW image in, NHWC bf16 planes out.
//
// Replaces ConvolutionLayer::Forward_gpu + ReLULayer for the first layer of the trunk
// (src/caffe/layers/conv_layer.cpp:25-40, base_conv_layer.cpp:257-280; the reference builds a
// 27 x (H*W) im2col buffer per image and calls sgemm).  The layer is HBM-bound (K = 27): per pixel it
// must read 12 B and write 64 channels x 2 B (x2 for the (hi, lo) pair) = 256 B: 4.2 GB for 8 x 768 x 2560
// pixels, about 1.3 ms at the H100's 3.35 TB/s.  An im2col patch tensor feeding a GEMM (27 taps padded to
// 64 bf16 channels) would add 128 B per pixel and plane, 2 GB per plane at that size, written and read again.  Here:
//   * producer warps read the fp32 image rows themselves (coalesced along x, zero padding by predication),
//     split to bf16 (hi, lo) and write them to shared memory as PIXEL ROWS of 8 channels (3 real) = 16 B per
//     pixel.  Nothing else is staged: no im2col tensor, no padded copy of the image.
//   * the im2col is done by the wgmma shared-memory DESCRIPTOR: in the no-swizzle K-major layout a core
//     matrix is 8 rows x 16 B with rows 16 B apart, the next 8-row group is SBO bytes further and the next
//     K chunk LBO bytes further.  With SBO = 128 B and LBO = 16 B over a pixel row, A[row r][K chunk j] is
//     pixel (r + j): the three horizontal taps are three overlapping views of the same 2 KB row segment.
//     K = 16 per MMA = two taps; (dx = 0,1) and (dx = 2, zero weights) -> 2 MMAs per image row dy, 6 per tile
//     and term, accumulated in registers by two warpgroups (pixels [0, 64) and [64, 128) of the tile).
//     Weights (64 x 96, 12 KB per plane) stay resident in shared memory.
//   * the same two warpgroups convert to (hi, lo), stage the 128 pixel x 64 channel tile 128B-swizzled and
//     hand it to TMA stores, four staging buffers deep so that stores of earlier tiles drain while later
//     tiles are converted.
// fp32-faithful mode accumulates hi*lo + lo*hi + hi*hi like conv_igemm.cu; bf16 mode one term.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "mscnn_b200.h"
#include "ptx_sm90.cuh"
#include "tmap.h"
#include "launch_count.h"

namespace mscnn {
namespace c3 {

constexpr int kTileW = 128;                  // output pixels per tile = MMA rows
constexpr int kCout = 64;
constexpr int kRowPx = 132;                  // staged pixels per image row: 128 + 3 halo/overreach, padded
constexpr int kRowBytes = kRowPx * 16;       // 2112
constexpr int kPlaneBytes = 3 * kRowBytes;   // three image rows (dy)
constexpr int kStageBytes = 2 * kPlaneBytes; // hi + lo, 12672 B (multiple of 128)
constexpr int kStages = 4;
constexpr int kChunks = 12;                  // K chunks of 8 elements: (dy, dx = 0..3), dx = 3 is all-zero
constexpr int kWPlaneBytes = kChunks * 8 * 128;  // [chunk][n8][8 couts][8 k] = 12 KB
constexpr int kEpiBufs = 4;
constexpr int kEpiPlane = kTileW * 128;      // 16 KB: 128 pixels x 64 channels bf16
constexpr int kProducerWarps = 4;            // warpgroup 0
constexpr int kThreads = 32 * kProducerWarps + 256;  // + two MMA / epilogue warpgroups
constexpr int kEpiThreads = 256;
constexpr int kEpiBarId = 1;
// Shared memory, offsets from its 1024-aligned base: the output staging buffers (1024-aligned for the swizzled TMA
// stores), the resident weights, the pixel-row stages, the bias and the stage barriers; kSmemBytes adds the slack for
// aligning the base.
constexpr int kWOff = kEpiBufs * 2 * kEpiPlane;
constexpr int kAOff = kWOff + 2 * kWPlaneBytes;
constexpr int kBiasOff = kAOff + kStages * kStageBytes;
constexpr int kBarOff = kBiasOff + kCout * 4;
constexpr int kSmemBytes = kBarOff + 16 * kStages + 1024;

struct Params {
  const float* x;     // [N][3][H][W] fp32
  const uint8_t* w;   // packed weights: hi plane then lo plane, kWPlaneBytes each (smem image)
  const float* bias;  // [64]
  int N, H, W, tiles_w;
  int split, relu;
};

// SPLIT is a template parameter so that the MMA sequence has no runtime branch (see conv_igemm.cu).
template <bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
conv_c3_tc_kernel(const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
  const uint32_t sEpi = smem_base, sW = smem_base + kWOff, sA = smem_base + kAOff;
  const int epi_buf_bytes = kEpiPlane * (p.split ? 2 : 1);
  uint8_t* gW = gen + kWOff;
  uint8_t* gA = gen + kAOff;
  float* bias_s = reinterpret_cast<float*>(gen + kBiasOff);
  ptx::Ring ring(smem_base + kBarOff, kStages);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // resident weights + bias (generic-proxy writes, made visible to the tensor core's async proxy below)
  {
    const int n16 = (p.split ? 2 : 1) * kWPlaneBytes / 16;
    const uint4* src = reinterpret_cast<const uint4*>(p.w);
    uint4* dst = reinterpret_cast<uint4*>(gW);
    for (int i = threadIdx.x; i < n16; i += kThreads) dst[i] = src[i];
    if (threadIdx.x < kCout) bias_s[threadIdx.x] = p.bias[threadIdx.x];
  }
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmO_hi);
    if (p.split) ptx::prefetch_tmap(&tmO_lo);
    ring.init(32, 2);  // every lane of the filling producer warp, one arrival per MMA warpgroup
    ptx::fence_mbar_init();
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();

  const int total_tiles = p.N * p.H * p.tiles_w;
  const size_t plane = static_cast<size_t>(p.H) * p.W;

  if (warp < kProducerWarps) {
    // ---------------------------------------------------------------- producers: image rows -> pixel rows
    // Producer warp w fills stage w with every kStages-th tile of this CTA (kProducerWarps == kStages), so four
    // tiles' global loads are in flight per SM; the MMA warpgroups consume the stages in tile order.
    static_assert(kProducerWarps == kStages, "one stage per producer warp");
    constexpr int kItems = 3 * 131;                 // (dy, px) pixels a tile needs
    constexpr int kIters = (kItems + 31) / 32;      // 13
    ptx::Ring own(ring.bars + 16u * warp, 1);  // this warp's stage
    for (int tile = blockIdx.x + warp * gridDim.x; tile < total_tiles; tile += kStages * gridDim.x) {
      const int tw = tile % p.tiles_w;
      const int y = (tile / p.tiles_w) % p.H;
      const int n = tile / (p.tiles_w * p.H);
      const int x0 = tw * kTileW - 1;  // image x of staged pixel 0
      const float* img = p.x + static_cast<size_t>(n) * 3 * plane;
      // all global loads of the tile first ...
      float v[kIters][3];
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const int item = it * 32 + lane;
        const int dy = item / 131, px = item - dy * 131;
        const int yy = y + dy - 1, xx = x0 + px;
        const bool ok = item < kItems && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W;
        const float* q = img + static_cast<size_t>(ok ? yy : 0) * p.W + (ok ? xx : 0);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[it][c] = ok ? __ldg(q + c * plane) : 0.f;
      }
      // ... then wait for the slot and fill it
      own.wait_empty();
      uint8_t* a_hi = gA + warp * kStageBytes;
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const int item = it * 32 + lane;
        if (item < kItems) {
          const int dy = item / 131, px = item - dy * 131;
          uint32_t h[3], l[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const __nv_bfloat16 hb = __float2bfloat16_rn(v[it][c]);
            const __nv_bfloat16 lb = __float2bfloat16_rn(v[it][c] - __bfloat162float(hb));
            h[c] = __bfloat16_as_ushort(hb);
            l[c] = __bfloat16_as_ushort(lb);
          }
          uint8_t* dst = a_hi + dy * kRowBytes + px * 16;
          *reinterpret_cast<uint4*>(dst) = make_uint4(h[0] | (h[1] << 16), h[2], 0u, 0u);
          if (p.split) *reinterpret_cast<uint4*>(dst + kPlaneBytes) = make_uint4(l[0] | (l[1] << 16), l[2], 0u, 0u);
        }
      }
      ptx::fence_proxy_async_smem();  // generic-proxy stores -> visible to wgmma operand reads
      ptx::mbar_arrive(own.full_bar());
      own.advance();
    }
    return;
  }

  // ------------------------------------------------------------------ MMA warpgroups + epilogue
  const int et = threadIdx.x - kProducerWarps * 32;  // 0..255
  const int wg = et >> 7;                            // pixels [64 wg, 64 wg + 64) of the tile
  const int wl = et & 127;
  const bool issuer = (et == 0);
  const int r0 = wg * 64 + (wl >> 5) * 16 + (lane >> 2);  // accumulator rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);
  float bias_r[16];  // this thread's 16 output channels: constant over tiles
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    bias_r[2 * j] = bias_s[8 * j + cq];
    bias_r[2 * j + 1] = bias_s[8 * j + cq + 1];
  }
  int ebuf = 0;
  float acc[kCout / 2];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int tw = tile % p.tiles_w;
    const int y = (tile / p.tiles_w) % p.H;
    const int n = tile / (p.tiles_w * p.H);
    ring.wait_full();
    ptx::wgmma_fence();
    {
      const uint32_t a_hi = sA + ring.slot * kStageBytes + static_cast<uint32_t>(wg) * 64u * 16u, a_lo = a_hi + kPlaneBytes;
      const uint32_t w_hi = sW, w_lo = sW + kWPlaneBytes;
      uint32_t accum = 0;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
        for (int m = 0; m < 2; ++m) {  // K chunks (2m, 2m+1) = pixels r + 2m, r + 2m + 1
          const uint32_t aoff = dy * kRowBytes + m * 32;
          const uint32_t boff = (dy * 4 + 2 * m) * 1024;
          const uint64_t ah = ptx::gmma_desc_nosw(a_hi + aoff, 16, 128), al = ptx::gmma_desc_nosw(a_lo + aoff, 16, 128);
          const uint64_t bh = ptx::gmma_desc_nosw(w_hi + boff, 1024, 128), bl = ptx::gmma_desc_nosw(w_lo + boff, 1024, 128);
          if constexpr (SPLIT) {
            ptx::wgmma_bf16<kCout>(acc, ah, bl, accum);
            ptx::wgmma_bf16<kCout>(acc, al, bh, 1u);
            ptx::wgmma_bf16<kCout>(acc, ah, bh, 1u);
          } else {
            ptx::wgmma_bf16<kCout>(acc, ah, bh, accum);
          }
          accum = 1u;
        }
      }
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    if (wl == 0) ptx::mbar_arrive(ring.empty_bar(ring.slot));  // the stage's operands have been read
    ring.advance();
    if (issuer) ptx::tma_store_wait_read<kEpiBufs - 1>();  // the buffer we are about to overwrite has been read
    ptx::named_bar_sync(kEpiBarId, kEpiThreads);
    const uint32_t buf = sEpi + ebuf * epi_buf_bytes;
#pragma unroll
    for (int j = 0; j < 8; ++j)  // 8-channel groups
#pragma unroll
      for (int h = 0; h < 2; ++h)
        ptx::stage_pair(buf, r0 + 8 * h, j, cq, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], bias_r[2 * j],
                        bias_r[2 * j + 1], p.relu, p.split, kEpiPlane);
    ptx::fence_proxy_async_smem();
    ptx::named_bar_sync(kEpiBarId, kEpiThreads);
    if (issuer) {
      ptx::tma_store_hi_lo(&tmO_hi, &tmO_lo, buf, p.split, kEpiPlane, 0, tw * kTileW, y, n);
      ptx::tma_store_commit();
    }
    if (++ebuf == kEpiBufs) ebuf = 0;
  }
  if (issuer) ptx::tma_store_wait_all<0>();
}

// fp32 [64][3][3][3] -> the kernel's shared-memory weight image, hi plane then lo plane:
// [chunk = dy*4 + dx][n8][8 couts][8 k = input channel], zero for dx = 3 and channels 3..7.
__global__ void pack_c3_weights_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int split) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // element of the hi plane
  if (i >= kWPlaneBytes / 2) return;
  const int k = i & 7, r = (i >> 3) & 7, n8 = (i >> 6) & 7, chunk = i >> 9;
  const int dy = chunk >> 2, dx = chunk & 3, co = n8 * 8 + r;
  float v = 0.f;
  if (dx < 3 && k < 3) v = w[((co * 3 + k) * 3 + dy) * 3 + dx];
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  out[i] = h;
  if (split) out[kWPlaneBytes / 2 + i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

}  // namespace c3
}  // namespace mscnn

using namespace mscnn;

extern "C" int mscnn_conv1_tc_packed_bytes(void) { return 2 * c3::kWPlaneBytes; }

extern "C" int mscnn_pack_conv1_tc_weights(const float* w_f32, void* packed, int split, void* stream) {
  if (!w_f32 || !packed) return MSCNN_ERR_INVALID;
  note_launch();
  c3::pack_c3_weights_kernel<<<(c3::kWPlaneBytes / 2 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      w_f32, (__nv_bfloat16*)packed, split ? 1 : 0);
  return cudaPeekAtLastError() == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}

extern "C" int mscnn_conv1_tc_forward(const float* x, const void* packed_w, const float* bias64, void* y_hi, void* y_lo,
                                      int N, int H, int W, int relu, void* stream) {
  if (!x || !packed_w || !bias64 || !y_hi || N < 1 || H < 1 || W < 1) return MSCNN_ERR_INVALID;
  c3::Params p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.w = static_cast<const uint8_t*>(packed_w);
  p.bias = bias64;
  p.N = N;
  p.H = H;
  p.W = W;
  p.tiles_w = (W + c3::kTileW - 1) / c3::kTileW;
  p.split = y_lo ? 1 : 0;
  p.relu = relu ? 1 : 0;
  CUtensorMap maps[2];
  memset(maps, 0, sizeof(maps));
  const uint64_t odim[4] = {64u, (uint64_t)W, (uint64_t)H, (uint64_t)N};
  const uint32_t obox[4] = {64u, (uint32_t)(W < c3::kTileW ? W : c3::kTileW), 1u, 1u};
  int rc = tmap_nhwc_bf16(&maps[0], y_hi, odim, obox);
  if (rc) return rc;
  if (y_lo) {
    rc = tmap_nhwc_bf16(&maps[1], y_lo, odim, obox);
    if (rc) return rc;
  } else {
    maps[1] = maps[0];
  }
  const size_t smem = c3::kSmemBytes;
  auto kern = p.split ? c3::conv_c3_tc_kernel<true> : c3::conv_c3_tc_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return MSCNN_ERR_CUDA;
  const long total = (long)N * H * p.tiles_w;
  int grid = mscnn_sm_count();
  if (grid > total) grid = (int)total;
  note_launch();
  kern<<<grid, c3::kThreads, smem, (cudaStream_t)stream>>>(maps[0], maps[1], p);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "mscnn_conv1_tc_forward: launch failed: %s\n", cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}
