// Host helpers: TMA tensor-map construction (driver entry point resolved at run time so the
// library has no link-time dependency on libcuda) and a cached SM count.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mscnn {

// 4-D NHWC bf16 tensor, dims = {C, W, H, N} (fastest first), box = {64, bw, bh, bn},
// 128-byte swizzle (the box's inner extent is exactly 128 B).  elem_strides (NULL = all 1): the box is traversed
// with these steps, so ceil(box[i] / elem_strides[i]) elements per dimension reach shared memory.
// byte_strides (NULL = the dense tensor): the global strides of dims 1..3 in bytes, multiples of 16; a strided view
// of a larger tensor (one output phase of a deconvolution) sets them.
int tmap_nhwc_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4],
                   const uint32_t box[4], const uint32_t elem_strides[4] = nullptr,
                   const uint64_t byte_strides[3] = nullptr);
// 2-D row-major bf16 matrix [rows][cols], box = {box_cols(=64), box_rows}, 128-byte swizzle.
int tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows,
                 uint32_t box_cols, uint32_t box_rows);

}  // namespace mscnn

#include "mscnn_b200.h"  // mscnn_sm_count
