// Implicit-GEMM convolution / inner product on the sm_90a tensor cores (wgmma).
//
// Replaces, for the MS-CNN forward path, the reference's
//   ConvolutionLayer::Forward_{cpu,gpu}   (src/caffe/layers/conv_layer.cpp:25-40,
//                                          base_conv_layer.cpp:257-280: im2col + sgemm + bias gemm)
//   InnerProductLayer::Forward_{cpu,gpu}  (src/caffe/layers/inner_product_layer.cpp:84-97)
//   ReLULayer::Forward_*                  (src/caffe/layers/relu_layer.cpp:9-19, fused here)
//
// Design (not a translation of im2col+sgemm):
//   * activations live in HBM as NHWC bf16 ("planes"); an fp32-faithful tensor is the pair
//     (hi, lo) with x ~= hi + lo, |lo| <= ulp_bf16(hi)/2;
//   * GEMM view: M = output pixels, N = output channels, K = taps x input channels.
//     An M tile is a TMA box {64 ch, bw, bh, bn} with bw*bh*bn <= 128 pixels; the tap
//     (dy,dx) operand is the same box shifted by (dx-pad, dy-pad): TMA zero-fills out-of-
//     bounds pixels, which *is* the convolution's zero padding.  No im2col buffer exists.
//   * stride / dilation: the same box traversed with the tensor map's element strides {1, stride_w, stride_h, 1}
//     (bw x bh pixels land in shared memory, bw stride_w x bh stride_h are spanned in the image), starting at
//     (w0 stride_w + dx dil_w - pad_w, h0 stride_h + dy dil_h - pad_h).  Nothing else in the kernel knows about them.
//   * groups: BLOCK_N divides Cout / group, so an n tile lies in one group k = n_base / (Cout / group); its
//     activation chunks start at channel k Cin / group, its weight rows and output channels are n_base as always.
//   * warp specialisation: warpgroup 0 = TMA producer (one warp issues, the others idle and hand
//     their registers to the MMA warpgroups), warpgroups 1 and 2 = wgmma (m64 x BLOCK_N x k16,
//     bf16 -> fp32) over rows [0, 64) and [64, 128) of the M tile, accumulators in registers, then
//     the epilogue from those registers (bias/ReLU -> bf16 split -> swizzled smem -> TMA store, or
//     direct fp32 stores for the narrow proposal / prediction heads).
//   * fp32-faithful mode = three bf16 GEMM terms accumulated in the same registers:
//     hi*hi + hi*lo + lo*hi (the dropped lo*lo term is < 2^-16 relative).
//       - "fat" stages (BLOCK_N <= 128): A_hi, A_lo, B_hi, B_lo of one (tap, channel chunk) in one stage,
//         the three products per K step in the order hi*lo, lo*hi, hi*hi;
//       - BLOCK_N = 256 (or MSCNN_NO_FAT): term-major, every (tap, chunk) k-block once per term
//         (all of hi*hi, then hi*lo, then lo*hi) -- four weight tiles per stage would leave room for one stage.
//   * row-share (3x3, BLOCK_N <= 128, 64x2 or 128x1 boxes): the taps dx = 0..2 of a (term, dy, chunk) read ONE
//     haloed activation tile ({64, bw + 2, bh, 1}) from a separate A ring, each MMA warpgroup's descriptor starting
//     dx rows further in; only the weights are fetched per tap.  Same MMAs in the same order: bit-identical results.
//   * optional fused 2x2 / stride-2 MAX pooling of the staged output tile (box_w, box_h even): bit-identical
//     to conv -> store -> pool_kernel, since it pools the stored (hi, lo) values.
//   * persistent CTAs (one per SM), static round-robin tile schedule, n-tile fastest so
//     CTAs working on the same pixels share the activation tile through L2.
//   All paths accumulate K in the order (dy, channel chunk, dx).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>
#include <vector>

#include "config.h"
#include "deconv_phase.h"
#include "mscnn_b200.h"
#include "ptx_sm90.cuh"
#include "tmap.h"
#include "launch_count.h"

namespace mscnn {

struct IgemmParams {
  int num_terms;   // 1: bf16; 3: split-bf16 (hi*hi, hi*lo, lo*hi)
  int taps_h, taps_w, pad_h, pad_w;
  int stride_h, stride_w, dil_h, dil_w;
  int cin_chunks;  // channels of one group / 64
  int cin_g, cout_g;  // input / output channels of one group (the whole padded extents when group == 1)
  int tiles_w, tiles_h, tiles_n, n_tiles;
  int box_w, box_h, box_n;
  int relu;
  int out_mode;    // MSCNN_OUT_NHWC_BF16, MSCNN_OUT_NCHW_F32 or MSCNN_OUT_NHWC_F32
  int has_lo_out;
  int pool;           // fused 2x2 / stride-2 MAX pooling of the output tile (box_w, box_h even)
  int store_full;     // also store the un-pooled tile (0 when only the pooling layer reads it)
  int stages, epi_bufs;  // stages: depth of the ring that carries B (and, without row-share, A with it)
  int fat;            // split mode with all four operand tiles (A_hi, A_lo, B_hi, B_lo) in one stage
  int rowshare;       // 3 horizontal taps read one haloed activation tile, delivered on its own ring of a_stages slots
  int a_stages;       // row-share: A-ring depth (0 otherwise)
  int a_slot;         // bytes of one A slot ([A_hi] or [A_hi][A_lo]); without row-share the A part of a stage
  int a_plane;        // bytes from A_hi to A_lo inside a slot
  int a_wg_row;       // activation-tile row where MMA warpgroup 1's 64 pixels start (tap dx = 0)
  const float* bias;  // [Cout_pad]
  const int* dyn_n;   // optional device count: process min(*dyn_n, out_n) images only (mscnn_conv_desc.dyn_n)
  float* out_f32;     // NCHW fp32 (out_mode 1)
  int out_n, out_c, out_h, out_w;
  int out_ld;         // row length of the pixel-major fp32 output (MSCNN_OUT_NHWC_F32)
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                       // bf16 elements = 128 B = one swizzle row
constexpr int kABytes = kBlockM * kBlockK * 2;    // 16 KB
constexpr int kPoolBytes = kABytes / 4;           // pooled tile: 32 rows x 128 B
constexpr int kThreads = 384;                     // producer warpgroup + two MMA warpgroups
constexpr int kEpiThreads = 256;
constexpr int kEpiBarId = 1;
constexpr int kMaxStages = 8, kMaxAStages = 4;    // deepest B ring and row-share A ring a plan builds

// Shared memory of conv_igemm_kernel<block_n, p.fat>, offsets from its 1024-aligned base: the A slots (their own ring
// with row-share, else one per stage), the B stages, the epilogue staging buffers and a barrier block sized for the
// deepest rings.  `total` is what a launch reserves, the slack for aligning the base included.  a_slot and the B tiles
// are multiples of 1024 B, so every region starts 1024-aligned (128B-swizzled tiles need it).
struct IgemmLayout {
  int b, epi, epi_buf, bar, total;
};
__host__ __device__ inline IgemmLayout igemm_layout(const IgemmParams& p, int block_n) {
  IgemmLayout l;
  l.b = (p.rowshare ? p.a_stages : p.stages) * p.a_slot;
  l.epi = l.b + p.stages * (p.fat ? 2 : 1) * block_n * kBlockK * 2;
  l.epi_buf = (kABytes + (p.pool ? kPoolBytes : 0)) * (p.has_lo_out ? 2 : 1);
  l.bar = l.epi + p.epi_bufs * l.epi_buf;
  l.total = l.bar + 16 * (kMaxStages + (p.rowshare ? kMaxAStages : 0)) + 1024;
  return l;
}

// Tile `tile` of the static schedule: n tile fastest, so CTAs working on the same pixels share the activation tile
// through L2; the M tile is the pixel box (tw, th, tn).
struct TileCoord {
  int n_tile, tw, th, tn;
};
__device__ __forceinline__ TileCoord tile_coord(const IgemmParams& p, int tile) {
  TileCoord t;
  t.n_tile = tile % p.n_tiles;
  int m = tile / p.n_tiles;
  t.tw = m % p.tiles_w;
  m /= p.tiles_w;
  t.th = m % p.tiles_h;
  t.tn = m / p.tiles_h;
  return t;
}

// Producer warp: the TMA loads of every tile of this CTA, k-blocks in the order (term, dy, chunk, dx), each k-block into
// the next stage of `ring` (A slot s at sA + s a_stride, B stage s at sB + s b_stride).  The whole warp
// walks the loops (warp-uniform control flow); one elected lane issues.  Row-share fetches the activation rows of one
// (term, dy, channel chunk) ONCE, with a one-pixel halo on each side ({64, box_w + 2, box_h, 1} from column w0 - pad:
// TMA zero fill is still the padding), for the taps dx = 0, 1, 2; each stage then carries only the weight tiles.
// Without row-share each stage carries the tap's shifted activation tile as well.
template <int BLOCK_N, bool FAT>
__device__ __forceinline__ void produce_tiles(const IgemmParams& p, const CUtensorMap* tmA_hi, const CUtensorMap* tmA_lo,
                                              const CUtensorMap* tmB_hi, const CUtensorMap* tmB_lo, uint32_t sA,
                                              uint32_t a_stride, uint32_t sB, uint32_t b_stride, ptx::Ring& ring,
                                              ptx::Ring& a_ring, int terms, int total_tiles) {
  constexpr uint32_t kPlanes = FAT ? 2u : 1u;
  constexpr uint32_t kBBytes = BLOCK_N * kBlockK * 2;
  const uint32_t a_tx = kPlanes * static_cast<uint32_t>((p.box_w + (p.rowshare ? 2 : 0)) * p.box_h * p.box_n) * kBlockK * 2;
  const uint32_t stage_tx = kPlanes * kBBytes + (p.rowshare ? 0u : a_tx);
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const TileCoord t = tile_coord(p, tile);
    const int w0 = t.tw * p.box_w * p.stride_w - p.pad_w, h0 = t.th * p.box_h * p.stride_h - p.pad_h, n0 = t.tn * p.box_n;
    const int c_base = t.n_tile * BLOCK_N / p.cout_g * p.cin_g;  // first input channel of the tile's group
    for (int term = 0; term < terms; ++term) {
      const CUtensorMap* mapA = (term == 2) ? tmA_lo : tmA_hi;
      const CUtensorMap* mapB = (term == 1) ? tmB_lo : tmB_hi;
      for (int dy = 0; dy < p.taps_h; ++dy) {
        for (int cc = 0; cc < p.cin_chunks; ++cc) {
          if (p.rowshare) {
            a_ring.wait_empty();
            if (ptx::elect_one()) {
              const uint32_t a0 = sA + a_ring.slot * a_stride;
              ptx::mbar_expect_tx(a_ring.full_bar(), a_tx);
              const int c0 = c_base + cc * kBlockK, h = h0 + dy * p.dil_h;
              ptx::tma_load_4d(a0, mapA, a_ring.full_bar(), c0, w0, h, n0);
              if (FAT) ptx::tma_load_4d(a0 + p.a_plane, tmA_lo, a_ring.full_bar(), c0, w0, h, n0);
            }
            __syncwarp();
            a_ring.advance();
          }
          for (int dx = 0; dx < p.taps_w; ++dx) {
            const int kcol = ((dy * p.taps_w + dx) * p.cin_chunks + cc) * kBlockK;
            ring.wait_empty();
            if (ptx::elect_one()) {
              const uint32_t a0 = sA + ring.slot * a_stride, b0 = sB + ring.slot * b_stride;
              ptx::mbar_expect_tx(ring.full_bar(), stage_tx);
              ptx::tma_load_2d(b0, mapB, ring.full_bar(), kcol, t.n_tile * BLOCK_N);
              if (FAT) ptx::tma_load_2d(b0 + kBBytes, tmB_lo, ring.full_bar(), kcol, t.n_tile * BLOCK_N);
              if (!p.rowshare) {
                const int c0 = c_base + cc * kBlockK, w = w0 + dx * p.dil_w, h = h0 + dy * p.dil_h;
                ptx::tma_load_4d(a0, mapA, ring.full_bar(), c0, w, h, n0);
                if (FAT) ptx::tma_load_4d(a0 + p.a_plane, tmA_lo, ring.full_bar(), c0, w, h, n0);
              }
            }
            __syncwarp();
            ring.advance();
          }
        }
      }
    }
  }
}

// The num_kb k-blocks of one tile on one MMA warpgroup, from the rings in the producer's order; the tile's first K step
// overwrites `acc`.  The warpgroup's rows start a_row_off bytes into the A tile, and tap dx a further dx a_dx_step bytes.
// On return every MMA has completed and every stage is handed back (the warpgroup's leader arrives).
template <int BLOCK_N, bool FAT>
__device__ __forceinline__ void mma_tile(const IgemmParams& p, uint32_t sA, uint32_t a_stride, uint32_t sB,
                                         uint32_t b_stride, ptx::Ring& ring, ptx::Ring& a_ring, int num_kb,
                                         uint32_t a_row_off, uint32_t a_dx_step, bool wg_leader,
                                         float (&acc)[BLOCK_N / 2]) {
  constexpr uint32_t kBBytes = BLOCK_N * kBlockK * 2;
  // the MMAs of a k-block may still read its stage (and A slot) until the next k-block's wgmma_wait<1>
  auto release_held = [&] {
    ring.release_held(wg_leader);
    a_ring.release_held(wg_leader);
  };
  int dx = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    // operands first, then the fence: between wgmma.fence and the MMAs nothing but the MMAs is issued
    const uint32_t a0 = sA + (p.rowshare ? a_ring.slot : ring.slot) * a_stride + a_row_off + dx * a_dx_step;
    const uint32_t b0 = sB + ring.slot * b_stride;
    const uint64_t ah = ptx::gmma_desc_sw128(a0), bh = ptx::gmma_desc_sw128(b0);
    const uint64_t al = ptx::gmma_desc_sw128(a0 + p.a_plane), bl = ptx::gmma_desc_sw128(b0 + kBBytes);
    const uint32_t accumulate = kb != 0 ? 1u : 0u;  // the tile's first K step overwrites the accumulators
    if (p.rowshare && dx == 0) a_ring.wait_full();
    ring.wait_full();
    ptx::fence_regs(acc);  // keep the accumulators in place across the asynchronous MMAs
    ptx::wgmma_fence();
    if constexpr (FAT) {
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        ptx::wgmma_bf16<BLOCK_N>(acc, ah + 2u * k, bl + 2u * k, k != 0 ? 1u : accumulate);
        ptx::wgmma_bf16<BLOCK_N>(acc, al + 2u * k, bh + 2u * k, 1u);
        ptx::wgmma_bf16<BLOCK_N>(acc, ah + 2u * k, bh + 2u * k, 1u);
      }
    } else {
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)
        // +32 B per K step inside the 128 B swizzle atom -> +2 in the address field
        ptx::wgmma_bf16<BLOCK_N>(acc, ah + 2u * k, bh + 2u * k, k != 0 ? 1u : accumulate);
    }
    ptx::wgmma_commit();
    ptx::fence_regs(acc);
    // the previous k-block's MMAs have finished reading their stage: hand it back to the producer
    ptx::wgmma_wait<1>();
    release_held();
    ring.hold_and_advance();
    // k-blocks run (term, dy, chunk, dx) with dx innermost: after the last dx the A slot is done with
    if (++dx == p.taps_w) {
      dx = 0;
      if (p.rowshare) a_ring.hold_and_advance();
    }
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  release_held();
}

// Fused PoolingLayer (MAX, 2x2, stride 2; pooling_layer.cpp:128-187) of the staged 64-channel chunk at `buf` into the
// pooled staging tile at `pbuf` ([hi][lo], kPoolBytes apart): exactly what pool_kernel would compute from the stored
// planes (value = hi + lo).  et: the thread's index among the kEpiThreads epilogue threads; hw_box = box_w box_h.
__device__ __forceinline__ void pool_staged_chunk(const IgemmParams& p, uint32_t buf, uint32_t pbuf, int et,
                                                  int hw_box) {
  const uint32_t lo_plane = kABytes;
  const int pw_box = p.box_w >> 1, phw_box = pw_box * (p.box_h >> 1);
  const int prows = phw_box * p.box_n;  // <= 32
  for (int item = et; item < prows * 8; item += kEpiThreads) {
    const int pr = item >> 3, j = item & 7;
    const int dn = pr / phw_box, rem = pr - dn * phw_box;
    const int ph = rem / pw_box, pwi = rem - ph * pw_box;
    const int r00 = dn * hw_box + (2 * ph) * p.box_w + 2 * pwi;
    float best[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) best[e] = -3.402823466e+38f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int r = r00 + (c >> 1) * p.box_w + (c & 1);
      const uint32_t a = buf + r * 128 + static_cast<uint32_t>((j ^ (r & 7)) << 4);
      uint32_t xh[4], xl[4] = {0u, 0u, 0u, 0u};
      ptx::ld_shared_v4(a, xh);
      if (p.has_lo_out) ptx::ld_shared_v4(a + lo_plane, xl);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v0 = __uint_as_float(xh[q] << 16) + __uint_as_float(xl[q] << 16);
        const float v1 = __uint_as_float(xh[q] & 0xFFFF0000u) + __uint_as_float(xl[q] & 0xFFFF0000u);
        best[2 * q] = (v0 > best[2 * q]) ? v0 : best[2 * q];
        best[2 * q + 1] = (v1 > best[2 * q + 1]) ? v1 : best[2 * q + 1];
      }
    }
    uint32_t oh[4], ol[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      oh[q] = ptx::pack_bf16x2(best[2 * q], best[2 * q + 1]);
      ol[q] = ptx::pack_bf16x2(best[2 * q] - __uint_as_float(oh[q] << 16),
                               best[2 * q + 1] - __uint_as_float(oh[q] & 0xFFFF0000u));
    }
    const uint32_t pa = pbuf + pr * 128 + static_cast<uint32_t>((j ^ (pr & 7)) << 4);
    ptx::st_shared_v4(pa, oh);
    if (p.has_lo_out) ptx::st_shared_v4(pa + kPoolBytes, ol);
  }
}

// FAT is a template parameter, not a runtime branch: with both MMA sequences in one body the accumulator registers
// cross a divergent region and ptxas has to insert extra warpgroup.arrive synchronisation before the MMAs.
template <int BLOCK_N, bool FAT>
__global__ void __launch_bounds__(kThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA_hi,
                  const __grid_constant__ CUtensorMap tmA_lo,
                  const __grid_constant__ CUtensorMap tmB_hi,
                  const __grid_constant__ CUtensorMap tmB_lo,
                  const __grid_constant__ CUtensorMap tmO_hi,
                  const __grid_constant__ CUtensorMap tmO_lo,
                  const __grid_constant__ CUtensorMap tmP_hi,
                  const __grid_constant__ CUtensorMap tmP_lo, const IgemmParams p) {
  constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  constexpr int kAcc = BLOCK_N / 2;  // fp32 accumulators per thread of an MMA warpgroup
  constexpr uint32_t kPlanes = FAT ? 2u : 1u;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const IgemmLayout lay = igemm_layout(p, BLOCK_N);
  const uint32_t a_stride = p.a_slot;                // [A_hi] or [A_hi][A_lo]
  const uint32_t b_stride = kPlanes * kBBytes;       // [B_hi] or [B_hi][B_lo]
  const uint32_t sA = smem_base, sB = smem_base + lay.b, sEpi = smem_base + lay.epi;
  // the B ring (stages; without row-share its slots carry the A tiles too), then the row-share A ring
  ptx::Ring ring(smem_base + lay.bar, p.stages);
  ptx::Ring a_ring(smem_base + lay.bar + 16u * p.stages, p.a_stages);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmA_hi);
    ptx::prefetch_tmap(&tmB_hi);
    if (p.num_terms > 1) {
      ptx::prefetch_tmap(&tmA_lo);
      ptx::prefetch_tmap(&tmB_lo);
    }
    if (p.out_mode == MSCNN_OUT_NHWC_BF16) {
      ptx::prefetch_tmap(&tmO_hi);
      if (p.has_lo_out) ptx::prefetch_tmap(&tmO_lo);
      if (p.pool) {
        ptx::prefetch_tmap(&tmP_hi);
        if (p.has_lo_out) ptx::prefetch_tmap(&tmP_lo);
      }
    }
    ring.init(1, 2);  // one producer arrival (+ TMA bytes), one arrival per MMA warpgroup
    if (p.rowshare) a_ring.init(1, 2);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // data-dependent batch size: every role derives the same tile count from the device-side count
  int tiles_n = p.tiles_n;
  if (p.dyn_n != nullptr) {
    int n_eff = *p.dyn_n;
    n_eff = n_eff < 0 ? 0 : (n_eff > p.out_n ? p.out_n : n_eff);
    tiles_n = (n_eff + p.box_n - 1) / p.box_n;
  }
  const int m_tiles = p.tiles_w * p.tiles_h * tiles_n;
  const int total_tiles = m_tiles * p.n_tiles;
  const int terms = FAT ? 1 : p.num_terms;  // a fat stage carries all three products of its k-block
  const int num_kb = terms * p.taps_h * p.taps_w * p.cin_chunks;

  if (warp < 4) {
    // TMA producer: one warp issues, the others hand their registers to the MMA warpgroups
    ptx::setmaxnreg_dec<40>();
    if (warp == 0)
      produce_tiles<BLOCK_N, FAT>(p, &tmA_hi, &tmA_lo, &tmB_hi, &tmB_lo, sA, a_stride, sB, b_stride, ring, a_ring, terms,
                                  total_tiles);
    return;
  }

  // MMA warpgroups + epilogue
  ptx::setmaxnreg_inc<232>();
  const int et = threadIdx.x - 128;          // 0..255
  const int wg = et >> 7;                    // rows [64 wg, 64 wg + 64) of the M tile
  const int wl = et & 127;
  const bool wg_leader = (wl == 0);
  const bool issuer = (et == 0);
  const int r0 = wg * 64 + (wl >> 5) * 16 + (lane >> 2);  // accumulator rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);                          // column offset within an 8-column group
  const uint32_t a_row_off = static_cast<uint32_t>(wg * p.a_wg_row) * 128u;
  // row-share: tap dx starts dx rows further into the haloed tile
  const uint32_t a_dx_step = p.rowshare ? 128u : 0u;
  const int hw_box = p.box_w * p.box_h;
  const int box_rows = hw_box * p.box_n;
  int ebuf = 0;
  float acc[kAcc];

  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    // The first output channel before the k-block loop, the pixel box after it: the instruction schedule depends on
    // where these divisions are issued.
    const int n_base = tile % p.n_tiles * BLOCK_N;
    mma_tile<BLOCK_N, FAT>(p, sA, a_stride, sB, b_stride, ring, a_ring, num_kb, a_row_off, a_dx_step, wg_leader, acc);
    const TileCoord t = tile_coord(p, tile);
    if (p.out_mode == MSCNN_OUT_NHWC_BF16) {
      if constexpr (BLOCK_N >= 64) {
        const uint32_t lo_plane = kABytes;
#pragma unroll
        for (int chunk = 0; chunk < BLOCK_N / 64; ++chunk) {
          // the staging buffer we are about to overwrite must have been read by its TMA store
          if (issuer) {
            if (p.epi_bufs == 1) ptx::tma_store_wait_read<0>();
            else ptx::tma_store_wait_read<1>();
          }
          ptx::named_bar_sync(kEpiBarId, kEpiThreads);
          const uint32_t buf = sEpi + ebuf * lay.epi_buf;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {  // 8-column groups of this 64-channel chunk
            const int j = chunk * 8 + jj;
            const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * j + cq));
#pragma unroll
            for (int h = 0; h < 2; ++h)
              ptx::stage_pair(buf, r0 + 8 * h, jj, cq, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], bb.x, bb.y, p.relu,
                              p.has_lo_out, lo_plane);
          }
          const uint32_t pbuf = buf + kABytes * (p.has_lo_out ? 2 : 1);  // pooled staging [hi][lo]
          if (p.pool) {
            ptx::named_bar_sync(kEpiBarId, kEpiThreads);
            pool_staged_chunk(p, buf, pbuf, et, hw_box);
          }
          ptx::fence_proxy_async_smem();
          ptx::named_bar_sync(kEpiBarId, kEpiThreads);
          if (issuer) {
            // one bulk group per staging buffer, pooled tile included
            const int c0 = n_base + chunk * 64;
            if (!p.pool || p.store_full)
              ptx::tma_store_hi_lo(&tmO_hi, &tmO_lo, buf, p.has_lo_out, lo_plane, c0, t.tw * p.box_w,
                                   t.th * p.box_h, t.tn * p.box_n);
            if (p.pool)
              ptx::tma_store_hi_lo(&tmP_hi, &tmP_lo, pbuf, p.has_lo_out, kPoolBytes, c0, t.tw * (p.box_w >> 1),
                                   t.th * (p.box_h >> 1), t.tn * p.box_n);
            ptx::tma_store_commit();
          }
          if (++ebuf == p.epi_bufs) ebuf = 0;
        }
      }
    } else {
      // fp32 outputs, direct stores
      const size_t plane = static_cast<size_t>(p.out_h) * p.out_w;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        const int dn = row / hw_box, rem = row - dn * hw_box;
        const int dh = rem / p.box_w, dw = rem - dh * p.box_w;
        const int n = t.tn * p.box_n + dn, y = t.th * p.box_h + dh, x = t.tw * p.box_w + dw;
        const bool ok = row < box_rows && n < p.out_n && y < p.out_h && x < p.out_w;
        if (!ok) continue;
        // NCHW: lanes of one quad are consecutive channels of one pixel
        float* obase = p.out_f32 + (static_cast<size_t>(n) * p.out_c) * plane + static_cast<size_t>(y) * p.out_w + x;
        // pixel-major fp32 rows [pixel][ld]
        float* rbase = p.out_f32 + ((static_cast<size_t>(n) * p.out_h + y) * p.out_w + x) * p.out_ld + n_base;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int c = 8 * j + cq;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + c));
          const float2 f = ptx::bias_relu(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], bb.x, bb.y, p.relu);
          if (p.out_mode == MSCNN_OUT_NHWC_F32) {
            *reinterpret_cast<float2*>(rbase + c) = f;
          } else {
            const int ch = n_base + c;
            if (ch < p.out_c) obase[static_cast<size_t>(ch) * plane] = f.x;
            if (ch + 1 < p.out_c) obase[static_cast<size_t>(ch + 1) * plane] = f.y;
          }
        }
      }
    }
  }
  if (issuer) ptx::tma_store_wait_all<0>();
}

// ------------------------------------------------------------------ host side

static int pick_block_n(int cout_pad) {
  if (cout_pad % 256 == 0) return 256;
  if (cout_pad % 128 == 0) return 128;
  if (cout_pad % 64 == 0) return 64;
  return 32;
}

// Choose the pixel box (bw, bh, bn), bw*bh*bn <= 128, that wastes the fewest MMA rows.  The activation box spans
// bw stride_w x bh stride_h image pixels, and a tensor map's box dimension is at most 256 elements.
static void pick_box(int N, int Ho, int Wo, bool even, int stride_h, int stride_w, int* bw_o, int* bh_o, int* bn_o) {
  double best = -1.0;
  int b_w = 1, b_h = 1, b_n = 1;
  for (int bw = 1; bw <= 128 && bw <= Wo && bw * stride_w <= 256; ++bw) {
    for (int bh = 1; bh * bw <= 128 && bh <= Ho && bh * stride_h <= 256; ++bh) {
      if (even && ((bw & 1) || (bh & 1))) continue;  // 2x2 pooling windows must not straddle tiles
      int bn = 128 / (bw * bh);
      if (bn > N) bn = N;
      // rows of a K-major SW128 tile come in groups of 8: any row count works for TMA, the
      // MMA simply computes (and the epilogue drops) the tail rows.
      const long tiles = (long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * ((N + bn - 1) / bn);
      const double eff = (double)N * Ho * Wo / (tiles * 128.0);
      // prefer wider boxes on ties: longer contiguous runs for TMA
      const double score = eff + 1e-6 * bw + 1e-9 * bh;
      if (score > best) {
        best = score;
        b_w = bw;
        b_h = bh;
        b_n = bn;
      }
    }
  }
  *bw_o = b_w;
  *bh_o = b_h;
  *bn_o = b_n;
}

constexpr int kSmemBudget = 227 * 1024;
constexpr int kMaxDevices = 64;

// The kernel's tensor-map arguments, in order (P: the fused pooling output).
enum MapSlot { kMapAHi, kMapALo, kMapBHi, kMapBLo, kMapOHi, kMapOLo, kMapPHi, kMapPLo, kNumMaps };

// A launch plan: everything mscnn_conv_forward derives from a descriptor (tile shapes, ring sizes, the eight tensor
// maps).  Plans are cached per (descriptor, device, config epoch): a steady-state forward does one hash lookup per
// convolution instead of a few getenv() and up to 8 cuTensorMapEncodeTiled calls (27 convolutions per step).
struct ConvPlan {
  IgemmParams p;
  CUtensorMap maps[kNumMaps];
  int grid;
  int BN;
  size_t smem;
};

// The output a launch writes instead of the dense planes [N][Ho][Wo][Cout_pad]: pixels (q_h step_h + r_h,
// q_w step_w + r_w), q in [0, ho) x [0, wo), of planes [N][full_h][full_w][Cout_pad] -- one output phase of a
// deconvolution (mscnn_deconv_forward), whose stride-1 sub-convolution may also have a negative pad.
struct OutView {
  int ho, wo, step_h, step_w, r_h, r_w, full_h, full_w;
};

// The deepest B ring, up to kMaxStages, whose layout fits the shared-memory budget (0 if none does).
static int deepest_ring(IgemmParams p, int block_n) {
  for (p.stages = kMaxStages; p.stages > 0 && igemm_layout(p, block_n).total > kSmemBudget; --p.stages) {
  }
  return p.stages;
}

// Ring depths of a candidate plan (per-tap or row-share, staging buffers preset): the B ring as deep as fits, one
// staging buffer instead of two where two would leave it shallower than 4 stages; with row-share, room left once the B
// ring is at its cap deepens the A ring from 2 up to kMaxAStages slots: with short k-blocks (plain bf16) two slots leave
// only one group of three taps to cover the L2 latency of the next activation tile.
static void fit_rings(IgemmParams& p, int block_n) {
  p.stages = deepest_ring(p, block_n);
  if (p.stages < 4 && p.epi_bufs == 2) {
    p.epi_bufs = 1;
    p.stages = deepest_ring(p, block_n);
  }
  while (p.rowshare && p.a_stages < kMaxAStages) {
    IgemmParams deeper = p;
    ++deeper.a_stages;
    if (deepest_ring(deeper, block_n) < kMaxStages) break;
    p.a_stages = deeper.a_stages;
  }
  p.stages = deepest_ring(p, block_n);
}

// A geometry field of mscnn_conv_desc: 0 means 1.
static inline int or1(int v) { return v == 0 ? 1 : v; }

static int unsupported(const mscnn_conv_desc* d, const char* rule) {
  fprintf(stderr, "mscnn_conv_forward: stride %dx%d, dilation %dx%d, group %d, C=%d Cout=%d Cout_pad=%d: %s\n",
          or1(d->stride_h), or1(d->stride_w), or1(d->dil_h), or1(d->dil_w), or1(d->group), d->C, d->Cout, d->Cout_pad,
          rule);
  return MSCNN_ERR_INVALID;
}

// What a served descriptor implies before any plan choice: strides, dilations and group (0 read as 1), the output
// extents, the channels of one group, the instantiation's BLOCK_N, and which operands and outputs the launch has.
struct ConvShape {
  int sh, sw, dh, dw, g, Ho, Wo, cin_g, cout_g, BN;
  bool split;   // fp32-faithful operands (x_lo, w_lo)
  bool pool;    // fused 2x2 pooling output
  bool staged;  // NHWC bf16 planes, written through shared-memory staging
};

// Plan step 1: check the descriptor and derive its shape.  view != NULL (a deconvolution phase): the output extents are
// the view's, the pad may be negative (the extents are not derived from it), and only NHWC_BF16 planes without pooling
// or dyn_n are written.
static int conv_shape(const mscnn_conv_desc* d, const OutView* view, ConvShape* s) {
  if (!d->x_hi || !d->w_hi || !d->bias) return MSCNN_ERR_INVALID;
  if (d->C % 64 != 0) return MSCNN_ERR_INVALID;
  const bool split = (d->x_lo != nullptr);
  if (split && !d->w_lo) return MSCNN_ERR_INVALID;
  const int sh = or1(d->stride_h), sw = or1(d->stride_w), dh = or1(d->dil_h), dw = or1(d->dil_w), g = or1(d->group);
  if (d->KH <= 0 || d->KW <= 0 || (!view && (d->pad_h < 0 || d->pad_w < 0))) return MSCNN_ERR_INVALID;
  if (view && (view->ho <= 0 || view->wo <= 0 || d->out_mode != MSCNN_OUT_NHWC_BF16 || d->pool_hi || d->dyn_n))
    return MSCNN_ERR_INVALID;
  if (sh < 1 || sh > 4 || sw < 1 || sw > 4) return unsupported(d, "strides 1..4 are served");
  // the furthest tap coordinate, pad + extent + reach, has to stay far inside a tensor map's int32 coordinates
  if (dh < 1 || dw < 1 || dh > (1 << 20) / d->KH || dw > (1 << 20) / d->KW)
    return unsupported(d, "the dilated kernel reach must be in 1..2^20");
  if (g < 1) return unsupported(d, "group must be positive");
  if (g > 1 && (d->C % g || d->Cout % g || d->C / g % 64 || d->Cout / g % 64 || d->Cout_pad != d->Cout))
    return unsupported(d, "a grouped convolution needs C / group and Cout / group to be multiples of 64");
  const int ext_h = dh * (d->KH - 1) + 1, ext_w = dw * (d->KW - 1) + 1;  // conv_layer.cpp:8-22
  if (d->N <= 0 || (!view && (d->H + 2 * d->pad_h < ext_h || d->W + 2 * d->pad_w < ext_w))) return MSCNN_ERR_INVALID;
  const int Ho = view ? view->ho : (d->H + 2 * d->pad_h - ext_h) / sh + 1;
  const int Wo = view ? view->wo : (d->W + 2 * d->pad_w - ext_w) / sw + 1;
  const int cin_g = d->C / g, cout_g = d->Cout_pad / g;
  const int BN = pick_block_n(cout_g);
  if (d->Cout_pad % BN != 0 || d->Cout > d->Cout_pad) return MSCNN_ERR_INVALID;
  const bool staged = d->out_mode == MSCNN_OUT_NHWC_BF16;
  const bool pool = (staged && d->pool_hi != nullptr);
  if (staged && (BN < 64 || (!d->y_hi && !pool))) return MSCNN_ERR_INVALID;
  if (pool && ((Ho & 1) || (Wo & 1))) return MSCNN_ERR_INVALID;  // fused pooling: even output extents only
  if ((d->out_mode == MSCNN_OUT_NCHW_F32 || d->out_mode == MSCNN_OUT_NHWC_F32) && !d->y_f32) return MSCNN_ERR_INVALID;
  // a lo plane is written for every staged output or none
  const bool lo_out = staged && (d->y_lo != nullptr || (pool && d->pool_lo != nullptr));
  if (pool && d->y_hi && lo_out && !d->y_lo) return MSCNN_ERR_INVALID;
  if (pool && lo_out && !d->pool_lo) return MSCNN_ERR_INVALID;
  *s = {sh, sw, dh, dw, g, Ho, Wo, cin_g, cout_g, BN, split, pool, staged};
  return MSCNN_OK;
}

// Plan step 2: the kernel parameters of the geometry, tiles and outputs; staging is left to stage_operands.
static IgemmParams igemm_params(const mscnn_conv_desc* d, const ConvShape& s) {
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.num_terms = s.split ? 3 : 1;
  p.taps_h = d->KH;
  p.taps_w = d->KW;
  p.pad_h = d->pad_h;
  p.pad_w = d->pad_w;
  p.stride_h = s.sh;
  p.stride_w = s.sw;
  p.dil_h = s.dh;
  p.dil_w = s.dw;
  p.cin_g = s.cin_g;
  p.cout_g = s.cout_g;
  p.cin_chunks = s.cin_g / 64;
  pick_box(d->N, s.Ho, s.Wo, s.pool, s.sh, s.sw, &p.box_w, &p.box_h, &p.box_n);
  p.tiles_w = (s.Wo + p.box_w - 1) / p.box_w;
  p.tiles_h = (s.Ho + p.box_h - 1) / p.box_h;
  p.tiles_n = (d->N + p.box_n - 1) / p.box_n;
  p.n_tiles = d->Cout_pad / s.BN;
  p.relu = d->relu;
  p.out_mode = d->out_mode;
  p.has_lo_out = (s.staged && (d->y_lo != nullptr || (s.pool && d->pool_lo != nullptr))) ? 1 : 0;
  p.pool = s.pool ? 1 : 0;
  p.store_full = (d->y_hi != nullptr) ? 1 : 0;
  p.bias = d->bias;
  p.dyn_n = d->dyn_n;
  p.out_f32 = d->y_f32;
  p.out_n = d->N;
  p.out_c = d->Cout;
  p.out_h = s.Ho;
  p.out_w = s.Wo;
  p.out_ld = d->Cout_pad;
  return p;
}

// Plan step 3: operand staging and ring depths.
static int stage_operands(const mscnn_conv_desc* d, const ConvShape& s, IgemmParams& p) {
  const Config& cfg = config();
  // Fat stages (A_hi, A_lo, B_hi, B_lo of a k-block in one stage, three MMAs per K step) for the narrow-N layers of
  // the fp32-faithful path: A_hi / B_hi are fetched once instead of twice and a barrier round trip covers 3x the MMAs.
  // BLOCK_N = 256 keeps single tiles: a fat stage would be 96 KB.  The choice depends on the layer alone (not on
  // pooling), so that fused and unfused launches of a layer sum in the same order.
  const int planes = (s.split && s.BN <= 128 && !cfg.no_fat) ? 2 : 1;
  p.fat = planes == 2;
  p.a_slot = kABytes * planes;
  p.a_plane = kABytes;
  p.a_wg_row = 64;
  p.epi_bufs = s.staged ? 2 : 0;  // fp32 outputs carve no staging region
  fit_rings(p, s.BN);
  if (p.stages < 2) return MSCNN_ERR_INVALID;

  // Row-share (3 horizontal taps, one image row per MMA warpgroup: 64x2 and 128x1 boxes, BLOCK_N <= 128).  The three
  // taps dx of a (term, dy, chunk) are the same activation rows shifted by one pixel: fetch them once with a one-pixel
  // halo per side into an A ring, and deliver only the weight tiles per tap on the B ring.  The MMAs, their order and
  // hence the results are those of the per-tap plan; L2->SM bytes per k-block drop from A + B to A / 3 + B.  The B ring
  // has to be at least as deep (in taps) as the per-tap ring it replaces, else the per-tap plan stays.  The haloed
  // row serves neighbouring taps only when they are neighbouring columns: stride and dilation 1 in W.
  const bool rs_box = p.box_n == 1 && ((p.box_w == 64 && p.box_h == 2) || (p.box_w == 128 && p.box_h == 1));
  if (!cfg.no_rowshare && d->KW == 3 && s.sw == 1 && s.dw == 1 && s.BN <= 128 && rs_box) {
    IgemmParams rs = p;
    rs.rowshare = 1;
    rs.a_stages = 2;
    rs.a_plane = ((p.box_w + 2) * p.box_h * 128 + 1023) / 1024 * 1024;  // each plane 1024-aligned (swizzle)
    rs.a_slot = rs.a_plane * planes;
    rs.a_wg_row = 64 / p.box_w * (p.box_w + 2) + 64 % p.box_w;  // halo-tile row of output pixel 64
    // a second epilogue buffer only overlaps the two 64-channel chunks of a BLOCK_N = 128 tile
    rs.epi_bufs = s.staged ? (s.BN > 64 ? 2 : 1) : 0;
    fit_rings(rs, s.BN);
    if (rs.stages >= p.stages) p = rs;
  }
  return MSCNN_OK;
}

// Plan step 4: the eight tensor maps.  A map the launch does not use is a copy of its primary (a lo plane of its hi
// plane, a hi plane of A_hi), so every kernel argument is a valid map.
static int encode_maps(const mscnn_conv_desc* d, const OutView* view, const ConvShape& s, const IgemmParams& p,
                       CUtensorMap (&maps)[kNumMaps]) {
  const uint64_t N = (uint64_t)d->N, Ho = (uint64_t)s.Ho, Wo = (uint64_t)s.Wo, cout_pad = (uint64_t)d->Cout_pad;
  // activation: with element strides TMA loads ceil(box / stride) = box_w (+ the row-share halo) x box_h pixels of a
  // box given in image pixels
  const uint64_t act_dims[4] = {(uint64_t)d->C, (uint64_t)d->W, (uint64_t)d->H, N};
  const uint32_t act_box[4] = {64u, (uint32_t)((p.box_w + (p.rowshare ? 2 : 0)) * s.sw), (uint32_t)(p.box_h * s.sh),
                               (uint32_t)p.box_n};
  const uint32_t act_strides[4] = {1u, (uint32_t)s.sw, (uint32_t)s.sh, 1u};
  auto activation = [&](CUtensorMap* m, const void* x) { return tmap_nhwc_bf16(m, x, act_dims, act_box, act_strides); };
  // weights: K-major [Cout_pad][taps x channels of one group]
  auto weights = [&](CUtensorMap* m, const void* w) {
    return tmap_2d_bf16(m, w, (uint64_t)d->KH * d->KW * s.cin_g, cout_pad, 64u, (uint32_t)s.BN);
  };
  // output: a view starts at pixel (r_h, r_w) of the full planes and steps (step_h, step_w) pixels: every byte stride
  // is a multiple of Cout_pad * 2 = 128 B
  const size_t pix = (size_t)d->Cout_pad * 2;
  const size_t view_off = view ? ((size_t)view->r_h * view->full_w + view->r_w) * pix : 0;
  const uint64_t view_strides[3] = {view ? view->step_w * pix : 0, view ? (size_t)view->step_h * view->full_w * pix : 0,
                                    view ? (size_t)view->full_h * view->full_w * pix : 0};
  const uint64_t out_dims[4] = {cout_pad, Wo, Ho, N};
  const uint32_t out_box[4] = {64u, (uint32_t)p.box_w, (uint32_t)p.box_h, (uint32_t)p.box_n};
  auto output = [&](CUtensorMap* m, const void* y) {
    return tmap_nhwc_bf16(m, static_cast<const uint8_t*>(y) + view_off, out_dims, out_box, nullptr,
                          view ? view_strides : nullptr);
  };
  const uint64_t pool_dims[4] = {cout_pad, Wo / 2, Ho / 2, N};
  const uint32_t pool_box[4] = {64u, (uint32_t)(p.box_w / 2), (uint32_t)(p.box_h / 2), (uint32_t)p.box_n};
  auto pooled = [&](CUtensorMap* m, const void* y) { return tmap_nhwc_bf16(m, y, pool_dims, pool_box); };

  // slot i encoded from `base`, or a copy of slot `primary` where the launch has no such operand (base NULL)
  auto put = [&](MapSlot i, const void* base, MapSlot primary, auto encode) -> int {
    if (!base) {
      maps[i] = maps[primary];
      return MSCNN_OK;
    }
    return encode(&maps[i], base);
  };
  const bool lo = p.has_lo_out;
  int rc = put(kMapAHi, d->x_hi, kMapAHi, activation);
  if (!rc) rc = put(kMapALo, s.split ? d->x_lo : nullptr, kMapAHi, activation);
  if (!rc) rc = put(kMapBHi, d->w_hi, kMapAHi, weights);
  if (!rc) rc = put(kMapBLo, s.split ? d->w_lo : nullptr, kMapBHi, weights);
  if (!rc) rc = put(kMapOHi, s.staged ? d->y_hi : nullptr, kMapAHi, output);
  if (!rc) rc = put(kMapOLo, lo ? d->y_lo : nullptr, kMapOHi, output);
  if (!rc) rc = put(kMapPHi, p.pool ? d->pool_hi : nullptr, kMapAHi, pooled);
  if (!rc) rc = put(kMapPLo, p.pool && lo ? d->pool_lo : nullptr, kMapPHi, pooled);
  return rc;
}

// The launch plan of (d, view).  encode = false (mscnn_*_plan_describe): the shape decisions only, no driver call.
static int build_plan(const mscnn_conv_desc* d, const OutView* view, bool encode, ConvPlan* plan) {
  ConvShape s;
  int rc = conv_shape(d, view, &s);
  if (rc != MSCNN_OK) return rc;
  IgemmParams& p = plan->p;
  p = igemm_params(d, s);
  if ((rc = stage_operands(d, s, p)) != MSCNN_OK) return rc;
  plan->BN = s.BN;
  plan->smem = igemm_layout(p, s.BN).total;
  const int total_tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_tiles;
  if (config().verbose_conv)
    fprintf(stderr, "conv plan: N=%d H=%d W=%d C=%d Cout_pad=%d k=%dx%d BN=%d box=%dx%dx%d fat=%d terms=%d rowshare=%d a_stages=%d stages=%d epi_bufs=%d smem=%zu tiles=%d\n",
            d->N, d->H, d->W, d->C, d->Cout_pad, d->KH, d->KW, s.BN, p.box_w, p.box_h, p.box_n, p.fat, p.num_terms,
            p.rowshare, p.a_stages, p.stages, p.epi_bufs, plan->smem, total_tiles);
  memset(plan->maps, 0, sizeof(plan->maps));
  plan->grid = 0;
  if (!encode) return MSCNN_OK;
  if ((rc = encode_maps(d, view, s, p, plan->maps)) != MSCNN_OK) return rc;
  plan->grid = mscnn_sm_count();
  if (plan->grid > total_tiles) plan->grid = total_tiles;
  return MSCNN_OK;
}

// The plan as text: which instantiation, pixel box, operand staging and pipeline depth (`stages` = depth of the ring
// carrying the weights; with rowshare=1 the activation tiles have their own ring of a_stages slots).
static int format_plan(const ConvPlan& plan, const mscnn_conv_desc* d, char* buf, int cap) {
  const IgemmParams& p = plan.p;
  int n = snprintf(buf, (size_t)cap,
                         "kernel=conv_igemm_kernel<%d, %s> box=%dx%dx%d terms=%d fat=%d pool=%d stages=%d epi_bufs=%d "
                         "smem=%zu dyn=%d rowshare=%d a_stages=%d",
                         plan.BN, p.fat ? "true" : "false", p.box_w, p.box_h, p.box_n, p.num_terms, p.fat, p.pool, p.stages, p.epi_bufs,
                         plan.smem, p.dyn_n ? 1 : 0, p.rowshare, p.a_stages);
  // stride / dilation / groups only where a layer has them: the plain convolution's line stays as it was
  const int group = d->Cout_pad / p.cout_g;
  if (n > 0 && n < cap && (p.stride_h != 1 || p.stride_w != 1 || p.dil_h != 1 || p.dil_w != 1 || group != 1)) {
    const int m = snprintf(buf + n, (size_t)(cap - n), " stride=%dx%d dil=%dx%d group=%d", p.stride_h, p.stride_w,
                           p.dil_h, p.dil_w, group);
    n = m > 0 ? n + m : -1;
  }
  return (n > 0 && n < cap) ? MSCNN_OK : MSCNN_ERR_INVALID;
}

// ------------------------------------------------------------------ plan cache

struct PlanKey {
  const void* ptr[11];
  int v[28];
  bool operator==(const PlanKey& o) const { return memcmp(this, &o, sizeof(PlanKey)) == 0; }
};
struct PlanKeyHash {
  size_t operator()(const PlanKey& k) const {
    const unsigned char* b = reinterpret_cast<const unsigned char*>(&k);
    uint64_t h = 1469598103934665603ull;  // FNV-1a
    for (size_t i = 0; i < sizeof(PlanKey); ++i) h = (h ^ b[i]) * 1099511628211ull;
    return static_cast<size_t>(h);
  }
};
static std::mutex g_plan_mu;
static std::unordered_map<PlanKey, ConvPlan, PlanKeyHash> g_plans;

void conv_plan_cache_clear() {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  g_plans.clear();
}

// The cached launch plan of (d, view), built and cached on a miss.
static int resolve_plan(const mscnn_conv_desc* d, const OutView* view, int device, ConvPlan* plan) {
  PlanKey key;
  memset(&key, 0, sizeof(key));
  const void* ptrs[11] = {d->x_hi, d->x_lo, d->w_hi, d->w_lo, d->bias, d->y_hi, d->y_lo, d->y_f32, d->pool_hi, d->pool_lo, d->dyn_n};
  memcpy(key.ptr, ptrs, sizeof(ptrs));
  const OutView dense = {0, 0, 0, 0, 0, 0, 0, 0};
  const OutView& v = view ? *view : dense;
  const int vals[28] = {d->N, d->H, d->W, d->C, d->Cout, d->Cout_pad, d->KH, d->KW, d->pad_h, d->pad_w, d->relu,
                        d->out_mode, device, static_cast<int>(config().epoch), 0,
                        d->stride_h, d->stride_w, d->dil_h, d->dil_w, d->group,
                        v.ho, v.wo, v.step_h, v.step_w, v.r_h, v.r_w, v.full_h, v.full_w};
  memcpy(key.v, vals, sizeof(vals));
  {
    std::lock_guard<std::mutex> lk(g_plan_mu);
    auto it = g_plans.find(key);
    if (it != g_plans.end()) {
      *plan = it->second;
      return MSCNN_OK;
    }
  }
  const int rc = build_plan(d, view, true, plan);
  if (rc != MSCNN_OK) return rc;
  std::lock_guard<std::mutex> lk(g_plan_mu);
  if (g_plans.size() >= 4096) g_plans.clear();  // blobs that keep moving (re-allocation): bound the table
  g_plans.emplace(key, *plan);
  return MSCNN_OK;
}

// ------------------------------------------------------------------ launch

// cudaFuncAttributeMaxDynamicSharedMemorySize is per device and function: raised once to the whole budget.
template <typename K>
static cudaError_t raise_smem_once(K kern, bool (&done)[kMaxDevices], int device) {
  if (device >= 0 && device < kMaxDevices && done[device]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget);
  if (e == cudaSuccess && device >= 0 && device < kMaxDevices) done[device] = true;
  return e;
}

template <int BLOCK_N, bool FAT>
static cudaError_t launch_igemm(const CUtensorMap (&maps)[kNumMaps], const IgemmParams& p, int grid, size_t smem,
                                int device, cudaStream_t stream) {
  auto kern = conv_igemm_kernel<BLOCK_N, FAT>;
  static bool done[kMaxDevices];
  cudaError_t e = raise_smem_once(kern, done, device);
  if (e != cudaSuccess) return e;
  mscnn::note_launch();
  kern<<<grid, kThreads, smem, stream>>>(maps[kMapAHi], maps[kMapALo], maps[kMapBHi], maps[kMapBLo], maps[kMapOHi],
                                         maps[kMapOLo], maps[kMapPHi], maps[kMapPLo], p);
  return cudaGetLastError();
}

static int launch_plan(const ConvPlan& plan, int device, cudaStream_t stream, const char* who) {
  // [BLOCK_N = 32 << i][fat]; fat stages only below BLOCK_N = 256 (stage_operands): no <256, true> instantiation
  static const decltype(&launch_igemm<32, false>) launch[4][2] = {
      {launch_igemm<32, false>, launch_igemm<32, true>}, {launch_igemm<64, false>, launch_igemm<64, true>},
      {launch_igemm<128, false>, launch_igemm<128, true>}, {launch_igemm<256, false>, nullptr}};
  const cudaError_t e =
      launch[__builtin_ctz(plan.BN) - 5][plan.p.fat](plan.maps, plan.p, plan.grid, plan.smem, device, stream);
  if (e != cudaSuccess) {
    fprintf(stderr, "%s: launch failed: %s\n", who, cudaGetErrorString(e));
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

}  // namespace mscnn

using namespace mscnn;

// ------------------------------------------------------------------ C entries

extern "C" int mscnn_conv_forward(const mscnn_conv_desc* d, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!d) return MSCNN_ERR_INVALID;
  int device = 0;
  if (cudaGetDevice(&device) != cudaSuccess) return MSCNN_ERR_CUDA;
  ConvPlan plan;
  const int rc = resolve_plan(d, nullptr, device, &plan);
  if (rc != MSCNN_OK) return rc;
  return launch_plan(plan, device, stream, "mscnn_conv_forward");
}

// The launch plan mscnn_conv_forward would use for `d`, as text, WITHOUT touching the device (no tensor map is encoded,
// the pointers in `d` only have to be non-NULL where the call would require them).  Host-side tests pin the variant
// every full-size layer takes.
extern "C" int mscnn_conv_plan_describe(const mscnn_conv_desc* d, char* buf, int cap) {
  if (!d || !buf || cap <= 0) return MSCNN_ERR_INVALID;
  ConvPlan plan;
  const int rc = build_plan(d, nullptr, false, &plan);
  if (rc != MSCNN_OK) return rc;
  return format_plan(plan, d, buf, cap);
}

// Entries in the launch-plan cache.  A net adds one per convolution for every new combination of input shape and blob
// addresses it runs with; the table is emptied when it reaches 4096 entries, so it stays bounded however many input
// sizes a process goes through.
extern "C" int mscnn_conv_plan_count(void) {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  return (int)g_plans.size();
}

// ------------------------------------------------------------------ deconvolution by output phase
// DeconvolutionLayer::Forward_gpu (deconv_layer.cu) for dense and 64-aligned grouped layers: the output is split by
// phase (deconv_phase.h) and each phase is a stride-1 convolution of the input with its own sub-kernel, signed pad and
// extent, run by conv_igemm_kernel with the phase's pixels of the full output planes as its output tensor map.

namespace mscnn {

// A phase no tap reaches holds the bias alone (col2im leaves it zero, the bias is added after): one channel pair of
// one pixel of the view per thread, bias + ReLU split into (hi, lo) as the GEMM epilogue does with a zero sum.
__global__ void deconv_bias_fill_kernel(const float* __restrict__ bias, __nv_bfloat16* __restrict__ yh,
                                        __nv_bfloat16* __restrict__ yl, int N, int Ho, int Wo, int cpad, int r_h,
                                        int r_w, int s_h, int s_w, int q_h, int q_w, int relu) {
  const int pairs = cpad / 2;
  const size_t total = (size_t)N * q_h * q_w * pairs;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = 2 * (int)(i % pairs);
    size_t r = i / pairs;
    const int qw = (int)(r % q_w);
    r /= q_w;
    const int qh = (int)(r % q_h);
    const size_t n = r / q_h;
    const float2 f = ptx::bias_relu(0.f, 0.f, bias[c], bias[c + 1], relu);
    const uint32_t h = ptx::pack_bf16x2(f.x, f.y);
    const uint32_t l = ptx::pack_bf16x2(f.x - __uint_as_float(h << 16), f.y - __uint_as_float(h & 0xFFFF0000u));
    const size_t o = ((n * Ho + (size_t)qh * s_h + r_h) * Wo + (size_t)qw * s_w + r_w) * cpad + c;
    *reinterpret_cast<uint32_t*>(yh + o) = h;
    if (yl) *reinterpret_cast<uint32_t*>(yl + o) = l;
  }
}

struct DeconvGeom {
  int sh, sw, dh, dw, g, Ho, Wo;
};

static int deconv_unsupported(const mscnn_conv_desc* d, const char* rule) {
  fprintf(stderr,
          "mscnn_deconv_forward: kernel %dx%d, stride %dx%d, pad %dx%d, dilation %dx%d, group %d, C=%d Cout=%d "
          "Cout_pad=%d, input %dx%d: %s\n",
          d->KH, d->KW, or1(d->stride_h), or1(d->stride_w), d->pad_h, d->pad_w, or1(d->dil_h), or1(d->dil_w),
          or1(d->group), d->C, d->Cout, d->Cout_pad, d->H, d->W, rule);
  return MSCNN_ERR_INVALID;
}

// The geometry of a deconvolution descriptor; MSCNN_ERR_INVALID, with a message for a geometry not served.
static int deconv_geometry(const mscnn_conv_desc* d, DeconvGeom* q) {
  if (!d->x_hi || !d->w_hi || !d->bias || !d->y_hi || d->N <= 0 || d->H <= 0 || d->W <= 0) return MSCNN_ERR_INVALID;
  if (d->x_lo && !d->w_lo) return MSCNN_ERR_INVALID;
  if (d->out_mode != MSCNN_OUT_NHWC_BF16) return deconv_unsupported(d, "the output is served as NHWC_BF16 planes only");
  if (d->pool_hi || d->pool_lo) return deconv_unsupported(d, "no fused pooling is served");
  if (d->dyn_n) return deconv_unsupported(d, "dyn_n must be NULL");
  q->sh = or1(d->stride_h);
  q->sw = or1(d->stride_w);
  q->dh = or1(d->dil_h);
  q->dw = or1(d->dil_w);
  q->g = or1(d->group);
  if (q->sh < 1 || q->sh > kDeconvMaxStride || q->sw < 1 || q->sw > kDeconvMaxStride)
    return deconv_unsupported(d, "strides 1..8 are served");
  if (!deconv_axis_ok(d->KH, q->sh, d->pad_h, q->dh) || !deconv_axis_ok(d->KW, q->sw, d->pad_w, q->dw))
    return deconv_unsupported(d, "kernel >= 1, pad in 0..2^20 and dilation >= 1 with a kernel reach up to 2^20 are served");
  if (q->g < 1 || d->C % 64 || d->Cout < 1 || d->Cout_pad % 64 || d->Cout > d->Cout_pad)
    return deconv_unsupported(d, "C and Cout_pad must be multiples of 64 and Cout_pad >= Cout >= 1");
  if (q->g > 1 && (d->C % q->g || d->Cout % q->g || d->C / q->g % 64 || d->Cout / q->g % 64 || d->Cout_pad != d->Cout))
    return deconv_unsupported(d, "a grouped deconvolution needs C / group and Cout / group to be multiples of 64 "
                                 "(group == channels: mscnn_deconv_depthwise_forward)");
  q->Ho = deconv_out_size(d->H, d->KH, q->sh, d->pad_h, q->dh);
  q->Wo = deconv_out_size(d->W, d->KW, q->sw, d->pad_w, q->dw);
  if (q->Ho <= 0 || q->Wo <= 0) return deconv_unsupported(d, "the output extent must be positive");
  return MSCNN_OK;
}

// Phase i = r_h s_w + r_w: its axes, its stride-1 sub-convolution and the view of the output it writes.
struct DeconvPhase {
  DeconvAxis h, w;
  mscnn_conv_desc sub;
  OutView view;
  bool launches() const { return h.taps > 0 && w.taps > 0 && view.ho > 0 && view.wo > 0; }
  bool fills() const { return (h.taps == 0 || w.taps == 0) && view.ho > 0 && view.wo > 0; }
};

static DeconvPhase deconv_phase(const mscnn_conv_desc* d, const DeconvGeom& q, int i) {
  DeconvPhase ph;
  ph.h = deconv_axis(d->KH, q.sh, d->pad_h, q.dh, q.Ho, i / q.sw);
  ph.w = deconv_axis(d->KW, q.sw, d->pad_w, q.dw, q.Wo, i % q.sw);
  const long long off =
      deconv_phase_offset(d->C, q.g, d->KH, d->KW, q.sh, q.sw, d->pad_h, d->pad_w, q.dh, q.dw, d->Cout_pad, i);
  ph.sub = *d;
  ph.sub.w_hi = static_cast<const __nv_bfloat16*>(d->w_hi) + off;
  ph.sub.w_lo = d->w_lo ? static_cast<const __nv_bfloat16*>(d->w_lo) + off : nullptr;
  ph.sub.KH = ph.h.taps;
  ph.sub.KW = ph.w.taps;
  ph.sub.pad_h = ph.h.pad;
  ph.sub.pad_w = ph.w.pad;
  ph.sub.stride_h = ph.sub.stride_w = 1;
  ph.sub.dil_h = ph.h.dil;
  ph.sub.dil_w = ph.w.dil;
  ph.sub.group = q.g;
  ph.view = {ph.h.ext, ph.w.ext, q.sh, q.sw, i / q.sw, i % q.sw, q.Ho, q.Wo};
  return ph;
}

}  // namespace mscnn

extern "C" int mscnn_deconv_forward(const mscnn_conv_desc* d, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!d) return MSCNN_ERR_INVALID;
  DeconvGeom q;
  int rc = deconv_geometry(d, &q);
  if (rc != MSCNN_OK) return rc;
  int device = 0;
  if (cudaGetDevice(&device) != cudaSuccess) return MSCNN_ERR_CUDA;
  // every phase's plan before the first launch: a descriptor that any phase refuses writes nothing
  const int phases = q.sh * q.sw;
  std::vector<DeconvPhase> ph(phases);
  std::vector<ConvPlan> plans(phases);
  for (int i = 0; i < phases; ++i) {
    ph[i] = deconv_phase(d, q, i);
    if (ph[i].launches() && (rc = resolve_plan(&ph[i].sub, &ph[i].view, device, &plans[i])) != MSCNN_OK) return rc;
  }
  for (int i = 0; i < phases; ++i) {
    if (ph[i].launches()) {
      if ((rc = launch_plan(plans[i], device, stream, "mscnn_deconv_forward")) != MSCNN_OK) return rc;
    } else if (ph[i].fills()) {
      const OutView& v = ph[i].view;
      const size_t total = (size_t)d->N * v.ho * v.wo * (d->Cout_pad / 2);
      const size_t cap = (size_t)mscnn_sm_count() * 16;
      const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
      mscnn::note_launch();
      deconv_bias_fill_kernel<<<grid, 256, 0, stream>>>(d->bias, static_cast<__nv_bfloat16*>(d->y_hi),
                                                         static_cast<__nv_bfloat16*>(d->y_lo), d->N, q.Ho, q.Wo,
                                                         d->Cout_pad, v.r_h, v.r_w, v.step_h, v.step_w, v.ho, v.wo,
                                                         d->relu);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) {
        fprintf(stderr, "mscnn_deconv_forward: bias fill launch failed: %s\n", cudaGetErrorString(e));
        return MSCNN_ERR_CUDA;
      }
    }
  }
  return MSCNN_OK;
}

// One line per output phase: its taps, sub-dilation, signed pad and extent, and the launch plan it runs
// (mscnn_conv_plan_describe's text), "bias_fill" where no tap reaches it, "none" where it holds no output pixel.
extern "C" int mscnn_deconv_plan_describe(const mscnn_conv_desc* d, char* buf, int cap) {
  if (!d || !buf || cap <= 0) return MSCNN_ERR_INVALID;
  DeconvGeom q;
  int rc = deconv_geometry(d, &q);
  if (rc != MSCNN_OK) return rc;
  int n = 0;
  buf[0] = '\0';
  for (int i = 0; i < q.sh * q.sw; ++i) {
    const DeconvPhase ph = deconv_phase(d, q, i);
    int m = snprintf(buf + n, (size_t)(cap - n), "phase=%dx%d taps=%dx%d dil=%dx%d pad=%dx%d out=%dx%d plan=",
                     ph.view.r_h, ph.view.r_w, ph.h.taps, ph.w.taps, ph.h.dil, ph.w.dil, ph.h.pad, ph.w.pad, ph.view.ho,
                     ph.view.wo);
    if (m < 0 || m >= cap - n) return MSCNN_ERR_INVALID;
    n += m;
    if (ph.launches()) {
      ConvPlan plan;
      if ((rc = build_plan(&ph.sub, &ph.view, false, &plan)) != MSCNN_OK) return rc;
      if ((rc = format_plan(plan, &ph.sub, buf + n, cap - n)) != MSCNN_OK) return rc;
      m = (int)strlen(buf + n);
    } else {
      m = snprintf(buf + n, (size_t)(cap - n), "%s", ph.fills() ? "bias_fill" : "none");
    }
    if (m < 0 || m + 1 >= cap - n) return MSCNN_ERR_INVALID;
    n += m;
    buf[n++] = '\n';
    buf[n] = '\0';
  }
  return MSCNN_OK;
}
