// Thin inline-PTX wrappers for the sm_90a features the MS-CNN kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors)
// and the proxy fences between them, plus the mbarrier ring and the (hi, lo) epilogue staging both kernels share.
// Nothing here is generic: it is the minimal set needed by conv_igemm.cu and conv_c3_tc.cu.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mscnn {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// A ring of `depth` shared-memory slots, each guarded by a "full" and an "empty" mbarrier (16 B per slot from `bars`).
// Producer and consumer walk the slots in order; the parity they wait for flips each time the ring wraps.  A consumer
// whose asynchronous reads of a slot outlive its wait holds the slot and releases it later (release_held).
struct Ring {
  uint32_t bars;
  int depth, slot = 0, held = -1;
  uint32_t phase = 0;
  __device__ Ring(uint32_t bars_, int depth_) : bars(bars_), depth(depth_) {}
  __device__ uint32_t full_bar() const { return bars + 16u * slot; }
  __device__ uint32_t empty_bar(int s) const { return bars + 16u * s + 8u; }
  __device__ void init(uint32_t fill_arrivals, uint32_t drain_arrivals) const {
    for (int s = 0; s < depth; ++s) {
      mbar_init(bars + 16u * s, fill_arrivals);
      mbar_init(empty_bar(s), drain_arrivals);
    }
  }
  __device__ void wait_full() const { mbar_wait(full_bar(), phase); }
  __device__ void wait_empty() const { mbar_wait(empty_bar(slot), phase ^ 1u); }
  __device__ void advance() {
    if (++slot == depth) {
      slot = 0;
      phase ^= 1u;
    }
  }
  __device__ void hold_and_advance() {
    held = slot;
    advance();
  }
  __device__ void release_held(bool arrive) {
    if (held >= 0 && arrive) mbar_arrive(empty_bar(held));
    held = -1;
  }
};

// ---------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1,
                                             int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::
          "l"(reinterpret_cast<uint64_t>(m)),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA store source, wgmma operands)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------- epilogue
// packed conversion (cvt.rn.bf16x2.f32): rounds like two scalar ones in half the issue slots
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h2);
}
__device__ __forceinline__ float2 bias_relu(float a0, float a1, float b0, float b1, bool relu) {
  float f0 = a0 + b0, f1 = a1 + b1;
  if (relu) {
    f0 = fmaxf(f0, 0.f);
    f1 = fmaxf(f1, 0.f);
  }
  return make_float2(f0, f1);
}
// One accumulator pair (two adjacent channels of one pixel) + bias, ReLU, split into bf16 (hi, lo) and stored into an
// output staging tile of 128 B rows laid out for a SWIZZLE_128B TMA store: row r, 16 B chunk j, bytes [2 c, 2 c + 4)
// of it; the lo plane lies `lo_plane` bytes after the hi plane and is written only when `lo` is set.
__device__ __forceinline__ void stage_pair(uint32_t buf, int r, int j, int c, float a0, float a1, float b0, float b1,
                                           bool relu, bool lo, uint32_t lo_plane) {
  const float2 f = bias_relu(a0, a1, b0, b1, relu);
  const uint32_t h = pack_bf16x2(f.x, f.y);
  const uint32_t l = pack_bf16x2(f.x - __uint_as_float(h << 16), f.y - __uint_as_float(h & 0xFFFF0000u));
  const uint32_t a = buf + r * 128 + static_cast<uint32_t>((j ^ (r & 7)) << 4) + 2u * c;
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(h) : "memory");
  if (lo) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + lo_plane), "r"(l) : "memory");
}
// 16 B of a staged tile as four 32-bit words (the fused pooling of conv_igemm.cu reads and writes its tiles this way)
__device__ __forceinline__ void ld_shared_v4(uint32_t addr, uint32_t (&v)[4]) {
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr));
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint32_t (&v)[4]) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3])
               : "memory");
}
// TMA store of a staged (hi, lo) tile pair at NHWC coordinates (c0, c1, c2, c3); the caller commits the bulk group.
__device__ __forceinline__ void tma_store_hi_lo(const CUtensorMap* hi, const CUtensorMap* lo, uint32_t src, bool has_lo,
                                                uint32_t lo_plane, int c0, int c1, int c2, int c3) {
  tma_store_4d(hi, src, c0, c1, c2, c3);
  if (has_lo) tma_store_4d(lo, src + lo_plane, c0, c1, c2, c3);
}

// One lane of a CONVERGED warp (the lowest): lets single-thread instructions (TMA) be issued from
// warp-uniform code, so that their operands live in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Register budget of a warpgroup role (producer warps give registers to the MMA warpgroups).
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// -------------------------------------------------------------------- wgmma
// wgmma shared-memory matrix descriptor (sm_90):
//   bits [0,14)  start address >> 4
//   bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4
//   bits [49,52) base offset (0: the tiles here are written by TMA from 1024-aligned bases, see below)
//   bits [62,64) layout: 0 = no swizzle (core matrices of 8 rows x 16 B), 1 = SWIZZLE_128B
// K-major bf16 tile whose rows are 128 B (64 bf16) written by TMA with CU_TENSOR_MAP_SWIZZLE_128B:
// LBO unused (1), SBO = 8 rows * 128 B = 1024 B.  Advancing by one K step (16 bf16 = 32 B) inside
// the 128 B swizzle atom adds 2 to the start-address field.
// The operand may also start at any 128 B row of such a tile, with the base offset left at 0 (the row-share halo of
// conv_igemm.cu: tap dx reads the tile dx rows further in).  wgmma takes the swizzle phase from the address bits
// [7,10) as TMA wrote them; measured on H100 for starts 0..15 rows in, where a base offset of (addr >> 7) & 7 instead
// reads the rows with the wrong phase.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// no-swizzle K-major descriptor: LBO = byte distance of K-adjacent core matrices, SBO = byte distance
// of the 8-row groups.
__device__ __forceinline__ uint64_t gmma_desc_nosw(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
  return d;
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Accumulator registers must not be touched between issue and wait: keep the compiler from moving
// their uses across the asynchronous MMA.
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 inputs, fp32 accumulate, both operands K-major in
// shared memory.  Per thread of the warpgroup: N / 2 accumulators; d[4 j + {0, 1}] = row
// 16 warp + lane / 4, columns 8 j + 2 (lane % 4) + {0, 1}; d[4 j + {2, 3}] = the same eight rows further.
__device__ __forceinline__ void wgmma_m64n32k16_bf16(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (N == 256) wgmma_m64n256k16_bf16(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 128) wgmma_m64n128k16_bf16(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 64) wgmma_m64n64k16_bf16(d, a_desc, b_desc, scale_d);
  else wgmma_m64n32k16_bf16(d, a_desc, b_desc, scale_d);
}

}  // namespace ptx
}  // namespace mscnn
