// caffe::Caffe context and common macros -- source-compatible subset of
// /root/reference/include/caffe/common.hpp:1-183 for the MS-CNN forward path.
//
// Differences that matter:
//   * Brew::CPU exists so that existing code compiles, but every mscnn_b200 layer's
//     Forward_cpu is a LOG(FATAL): there is no CPU fallback (see layer.hpp).  The default
//     mode is GPU.
//   * shared_ptr is std::shared_ptr (the reference aliases boost::shared_ptr, common.hpp:74).
//   * One extension: Caffe::precision() selects the convolution arithmetic,
//     FP32_SPLIT (3-term bf16 split, fp32-faithful; default) or BF16 (single term).
//     Env MSCNN_PRECISION=bf16|fp32 sets the initial value.
#pragma once
#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <fstream>
#include <iostream>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <string>
#include <utility>
#include <vector>

#include "caffe/logging.hpp"
#include "mscnn_b200.h"

// libmscnn_b200.so is built with hidden visibility; the Caffe-API mirror is its exported C++ surface, so that a C++
// host that includes these headers links against the library like it would against libcaffe.so.
#if defined(__GNUC__)
#define CAFFE_API __attribute__((visibility("default")))
#else
#define CAFFE_API
#endif

#define DISABLE_COPY_AND_ASSIGN(classname) \
 private:                                  \
  classname(const classname&);             \
  classname& operator=(const classname&)

// mscnn_b200 instantiates float only (the reference also instantiates double,
// common.hpp:41-44; no shipped MS-CNN net is a Net<double>).
#define INSTANTIATE_CLASS(classname) template class classname<float>

#define NOT_IMPLEMENTED LOG(FATAL) << "Not Implemented Yet"

#define CUDA_CHECK(condition)                                            \
  do {                                                                   \
    cudaError_t error = condition;                                       \
    CHECK_EQ(error, cudaSuccess) << " " << cudaGetErrorString(error);    \
  } while (0)

// C-ABI status -> Caffe's abort-on-error convention
#define MSCNN_CHECK(call)                                           \
  do {                                                              \
    const int mscnn_rc_ = (call);                                   \
    CHECK_EQ(mscnn_rc_, MSCNN_OK) << " " #call " failed";           \
  } while (0)

namespace caffe {

using std::shared_ptr;
using std::make_pair;
using std::map;
using std::pair;
using std::set;
using std::string;
using std::vector;

class CAFFE_API Caffe {
 public:
  enum Brew { CPU, GPU };
  enum Precision { FP32_SPLIT, BF16 };
  static Caffe& Get();  // thread-local, like common.cpp:13-22; freed when its thread ends
  ~Caffe();
  inline static Brew mode() { return Get().mode_; }
  inline static void set_mode(Brew mode) { Get().mode_ = mode; }
  inline static Precision precision() { return Get().precision_; }
  inline static void set_precision(Precision p) { Get().precision_ = p; }
  inline static bool split() { return Get().precision_ == FP32_SPLIT; }
  static void SetDevice(const int device_id);
  static void DeviceQuery();
  // the stream every layer launches on (the reference uses the legacy default stream)
  inline static cudaStream_t stream() { return Get().stream_; }
  inline static void set_stream(cudaStream_t s) { Get().stream_ = s; }
  // Transient device scratch (grow-only, per thread context); valid until the next scratch() call
  // on the same context.  Work using it is stream-ordered, so layers may reuse it back to back.
  static void* scratch(size_t bytes);
  inline static int solver_count() { return 1; }
  inline static bool root_solver() { return true; }

 private:
  Caffe();
  Brew mode_;
  Precision precision_;
  cudaStream_t stream_;
  void* scratch_;
  size_t scratch_bytes_;
  DISABLE_COPY_AND_ASSIGN(Caffe);
};

}  // namespace caffe
