#include "tmap.h"
#include "launch_count.h"

#include <cudaTypedefs.h>
#include <stdio.h>

#include <mutex>

#include "mscnn_b200.h"

namespace mscnn {

static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    } else {
      fprintf(stderr, "mscnn: cuTensorMapEncodeTiled entry point unavailable (%s)\n",
              cudaGetErrorString(e));
    }
  });
  return fn;
}

int tmap_nhwc_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4],
                   const uint32_t box[4], const uint32_t elem_strides[4], const uint64_t byte_strides[3]) {
  auto enc = get_encode();
  if (!enc) return MSCNN_ERR_CUDA;
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstride[3] = {dims[0] * 2, dims[0] * dims[1] * 2, dims[0] * dims[1] * dims[2] * 2};
  for (int i = 0; byte_strides && i < 3; ++i) gstride[i] = byte_strides[i];
  cuuint32_t b[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int i = 0; elem_strides && i < 4; ++i) estr[i] = elem_strides[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstride,
                   b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr,
            "mscnn: cuTensorMapEncodeTiled(4d) failed rc=%d dims={%llu,%llu,%llu,%llu} "
            "box={%u,%u,%u,%u} strides={%u,%u,%u,%u} byte strides={%llu,%llu,%llu} base=%p\n",
            (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1],
            (unsigned long long)dims[2], (unsigned long long)dims[3], box[0], box[1], box[2],
            box[3], estr[0], estr[1], estr[2], estr[3], (unsigned long long)gstride[0],
            (unsigned long long)gstride[1], (unsigned long long)gstride[2], base);
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

int tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows,
                 uint32_t box_cols, uint32_t box_rows) {
  auto enc = get_encode();
  if (!enc) return MSCNN_ERR_CUDA;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * 2};
  cuuint32_t b[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride,
                   b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "mscnn: cuTensorMapEncodeTiled(2d) failed rc=%d cols=%llu rows=%llu box={%u,%u}\n",
            (int)r, (unsigned long long)cols, (unsigned long long)rows, box_cols, box_rows);
    return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}

std::atomic<unsigned long long> g_kernel_launches{0};
std::atomic<unsigned long long> g_weight_packs{0};

}  // namespace mscnn

extern "C" unsigned long long mscnn_kernel_launch_count(void) {
  return mscnn::g_kernel_launches.load(std::memory_order_relaxed);
}

extern "C" unsigned long long mscnn_weight_pack_count(void) {
  return mscnn::g_weight_packs.load(std::memory_order_relaxed);
}

extern "C" int mscnn_sm_count(void) {
  static int cached = 0;
  if (cached > 0) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;
  cached = n;
  return n;
}
