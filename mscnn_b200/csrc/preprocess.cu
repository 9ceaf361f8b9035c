// Image pre-processing on the device (SURVEY.md section 8(f) rank 3): the step in front of the path.
//   examples/kitti_car/run_mscnn_detection.m:64-69, examples/widerface/run_mscnn_detection.m:70-86:
//     test_image = imresize(test_image,[imgH imgW]);        uint8 in, uint8 out, bicubic + antialiasing
//     test_image = single(test_image(:,:,[3 2 1]));          RGB -> BGR, to fp32
//     test_image = bsxfun(@minus,test_image,mu);             mu = [104 117 123] per BGR channel
//     test_image = permute(test_image, [2 1 3]);             MATLAB [W H C] column-major = Caffe C x H x W
// The reference does this on the host in MATLAB and uploads 4 bytes per value of the RESIZED image
// (23.6 MB for 3x768x2560); here the ORIGINAL uint8 image (1.4 MB for a 375x1242 KITTI frame) is
// uploaded and both resize passes, the channel swap, the mean subtraction and the layout change run on
// the device, writing straight into the net's `data` blob.
//
// imresize itself is MathWorks code that is not part of /root/reference; its published algorithm
// (imresize.m `contributions`, cubic kernel a = -0.5, Keys 1981) is restated here:
//   scale = out / in per dimension;   antialiasing widens the kernel by 1/scale when scale < 1;
//   u = x/scale + 0.5 (1 - 1/scale), left = floor(u - kw/2), P = ceil(kw) + 2 taps, weights normalised per
//   output sample, out-of-range taps mirrored (symmetric padding), all-zero tap columns dropped;
//   dimensions are resized in ascending order of scale; each pass accumulates in fp64 and, for uint8
//   images, rounds (half away from zero) and saturates back to uint8.
// Tap tables are built on the host in fp64 (mscnn_imresize_contributions, testable without a GPU); the
// kernels multiply and add in the table's tap order without FMA contraction (-fmad=false), so the result
// is bit-identical to the numpy restatement in oracle/port.py.
//
// Grayscale frames ([h][w] or [h][w][1], as imread returns them): the cascade drivers turn them into RGB first
// (`if (size(img,3)==1), img = repmat(img,[1 1 3]); end`, examples/kitti_car/run_cascademscnn.m:76,
// examples/citypersons/run_cascademscnn.m:82).  imresize works per channel, so the three copies would resize to the
// same bytes: here the one channel is resized once, and the second pass writes its value into all three planes,
// each minus its own mean.  The result is bit for bit that of the repmat'ed frame.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>

#include <vector>

#include "mscnn_b200.h"
#include "launch_count.h"

namespace mscnn {

namespace {

// Keys cubic convolution kernel, a = -0.5 (imresize.m `cubic`).
double cubic(double x) {
  const double a = fabs(x), a2 = a * a, a3 = a2 * a;
  if (a <= 1.0) return (1.5 * a3 - 2.5 * a2) + 1.0;
  if (a <= 2.0) return ((-0.5 * a3 + 2.5 * a2) - 4.0 * a) + 2.0;
  return 0.0;
}

struct Contrib {
  int taps = 0;
  std::vector<double> w;  // [out_len][taps]
  std::vector<int> idx;   // [out_len][taps], 0-based
};

Contrib contributions(int in_len, int out_len) {
  const double scale = (double)out_len / (double)in_len;
  const bool aa = scale < 1.0;
  const double kw = aa ? 4.0 / scale : 4.0;
  const int P = (int)ceil(kw) + 2;
  std::vector<double> w((size_t)out_len * P);
  std::vector<int> idx((size_t)out_len * P);
  std::vector<char> used(P, 0);
  const int period = 2 * in_len;
  for (int o = 0; o < out_len; ++o) {
    const double x = (double)(o + 1);
    const double u = x / scale + 0.5 * (1.0 - 1.0 / scale);
    const double left = floor(u - kw / 2.0);
    double sum = 0.0;
    for (int k = 0; k < P; ++k) {
      const double ind = left + (double)k;  // 1-based sample position
      const double d = u - ind;
      const double v = aa ? scale * cubic(scale * d) : cubic(d);
      w[(size_t)o * P + k] = v;
      sum += v;
      long m = ((long)ind - 1) % period;
      if (m < 0) m += period;
      idx[(size_t)o * P + k] = (int)(m < in_len ? m : period - 1 - m);
    }
    for (int k = 0; k < P; ++k) {
      w[(size_t)o * P + k] /= sum;
      if (w[(size_t)o * P + k] != 0.0) used[k] = 1;
    }
  }
  Contrib c;
  for (int k = 0; k < P; ++k) c.taps += used[k];
  c.w.resize((size_t)out_len * c.taps);
  c.idx.resize((size_t)out_len * c.taps);
  for (int o = 0; o < out_len; ++o) {
    int t = 0;
    for (int k = 0; k < P; ++k) {
      if (!used[k]) continue;
      c.w[(size_t)o * c.taps + t] = w[(size_t)o * P + k];
      c.idx[(size_t)o * c.taps + t] = idx[(size_t)o * P + k];
      ++t;
    }
  }
  return c;
}

struct DevTable {
  int taps = 0;
  double* w = nullptr;
  int* idx = nullptr;
};

// The tap tables of one input size (the output size is the plan's), uploaded once.
struct SizeTables {
  int in_h, in_w;
  int first_dim;  // 0: height pass first, 1: width pass first (ascending scale, ties -> height)
  DevTable th, tw;
};

}  // namespace

struct PreprocessPlan {
  mscnn_preprocess_desc d;         // in_h / in_w = sizes[0], the size the plan was created for
  std::vector<SizeTables> sizes;   // one entry per distinct input size seen so far
  unsigned char* mid = nullptr;    // intermediate images after the first pass
  size_t mid_cap = 0;
  unsigned char* stage = nullptr;  // device copy of host images (mscnn_preprocess_forward*_host)
  size_t stage_cap = 0;
  // `stage` and `mid` are rewritten by every call.  A call issued on another stream than the previous one first makes
  // its stream wait, on the device, for this event, recorded behind the previous call's last launch.
  cudaEvent_t used = nullptr;
  cudaStream_t used_on = nullptr;
  bool used_valid = false;
};

// One image of a batch as both passes see it.  The descriptors of a launch travel by value in the kernel parameter
// block, so a later call can never overwrite them before the kernels have read them.
struct ImageDesc {
  size_t src, mid;  // byte offsets of the image in the input batch and of its intermediate image
  int in_h, in_w;   // original size
  int channels;     // 3 (interleaved RGB) or 1 (gray: the one channel stands for all three)
  int mid_h, mid_w; // size after the first pass
  int first_dim;    // the first pass resizes along this dimension (0: height), the second along the other
  DevTable t1, t2;  // tap tables of the first and the second pass
};

// 32 descriptors = 2.8 KB of parameters; larger batches take several launches of both kernels.
constexpr int kImagesPerLaunch = 32;
struct ImageBatch {
  int n0;  // batch index of d[0]
  ImageDesc d[kImagesPerLaunch];
};

// uint8 conversion of an fp64 accumulator: saturate, round half away from zero.
__device__ __forceinline__ double round_u8(double v) {
  v = fmin(fmax(v, 0.0), 255.0);
  return round(v);
}

// First pass: resize image d[blockIdx.y] of the launch along one dimension, uint8 [h][w][C] -> uint8 [mid_h][mid_w][C].
// One thread per output byte (the C channels of a pixel are adjacent bytes, so a warp writes 32 consecutive bytes
// and reads `taps` rows or pixel neighbourhoods that its lanes share).
//   along = 0: out[y][x][c] = sum_k w[y][k] * in[idx[y][k]][x][c]   (out_h x in_w)
//   along = 1: out[y][x][c] = sum_k w[x][k] * in[y][idx[x][k]][c]   (in_h x out_w)
template <int C>
__device__ __forceinline__ void imresize_pass_u8(const ImageDesc& D, const unsigned char* __restrict__ images,
                                                 unsigned char* __restrict__ mid) {
  const int in_w = D.in_w, out_w = D.mid_w, along = D.first_dim, taps = D.t1.taps;
  const double* __restrict__ w = D.t1.w;
  const int* __restrict__ idx = D.t1.idx;
  const unsigned char* img = images + D.src;
  unsigned char* out = mid + D.mid;
  const size_t total = (size_t)D.mid_h * out_w * C;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const size_t p = e / C;
    const int x = (int)(p % out_w);
    const int y = (int)(p / out_w);
    const int o = along == 0 ? y : x;
    const double* wr = w + (size_t)o * taps;
    const int* ir = idx + (size_t)o * taps;
    double acc = 0.0;
    for (int k = 0; k < taps; ++k) {
      const int s = ir[k];
      const size_t off = along == 0 ? ((size_t)s * in_w + x) * C + c : ((size_t)y * in_w + s) * C + c;
      acc = __dadd_rn(acc, __dmul_rn(wr[k], (double)img[off]));
    }
    out[e] = (unsigned char)round_u8(acc);
  }
}

__global__ void imresize_pass_u8_kernel(const unsigned char* __restrict__ images, unsigned char* __restrict__ mid,
                                        const ImageBatch b) {
  const ImageDesc& D = b.d[blockIdx.y];
  if (D.channels == 3)
    imresize_pass_u8<3>(D, images, mid);
  else
    imresize_pass_u8<1>(D, images, mid);
}

// Second pass + channel swap + mean subtraction + HWC -> CHW, into slot b.n0 + blockIdx.y of the blob.  One thread
// per output pixel; a warp writes 32 consecutive floats of each of the three output planes.
template <int C>
__device__ __forceinline__ void imresize_pass_to_blob(const ImageDesc& D, const unsigned char* __restrict__ mid,
                                                      float* __restrict__ data, int out_h, int out_w, int n,
                                                      float mean0, float mean1, float mean2, int swap_rb) {
  const int in_w = D.mid_w, along = 1 - D.first_dim, taps = D.t2.taps;
  const double* __restrict__ w = D.t2.w;
  const int* __restrict__ idx = D.t2.idx;
  const unsigned char* img = mid + D.mid;
  const size_t plane = (size_t)out_h * out_w;
  float* out = data + (size_t)n * 3 * plane;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < plane; e += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(e % out_w);
    const int y = (int)(e / out_w);
    const int o = along == 0 ? y : x;
    const double* wr = w + (size_t)o * taps;
    const int* ir = idx + (size_t)o * taps;
    float* dst = out + (size_t)y * out_w + x;
    if (C == 1) {
      // gray: the three channels of the repmat'ed frame are equal, whatever the swap
      double a = 0.0;
#pragma unroll 1
      for (int k = 0; k < taps; ++k) {
        const int s = ir[k];
        const unsigned char* q = img + (along == 0 ? (size_t)s * in_w + x : (size_t)y * in_w + s);
        a = __dadd_rn(a, __dmul_rn(wr[k], (double)q[0]));
      }
      const float v = (float)round_u8(a);
      dst[0] = v - mean0;
      dst[plane] = v - mean1;
      dst[2 * plane] = v - mean2;
      continue;
    }
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (int k = 0; k < taps; ++k) {
      const int s = ir[k];
      const unsigned char* q = img + (along == 0 ? ((size_t)s * in_w + x) * 3 : ((size_t)y * in_w + s) * 3);
      const double wk = wr[k];
      a0 = __dadd_rn(a0, __dmul_rn(wk, (double)q[0]));
      a1 = __dadd_rn(a1, __dmul_rn(wk, (double)q[1]));
      a2 = __dadd_rn(a2, __dmul_rn(wk, (double)q[2]));
    }
    const float v0 = (float)round_u8(a0), v1 = (float)round_u8(a1), v2 = (float)round_u8(a2);
    // output channel order after test_image(:,:,[3 2 1]): plane 0 = input channel 2 when swapping
    dst[0] = (swap_rb ? v2 : v0) - mean0;
    dst[plane] = v1 - mean1;
    dst[2 * plane] = (swap_rb ? v0 : v2) - mean2;
  }
}

__global__ void imresize_pass_to_blob_kernel(const unsigned char* __restrict__ mid, float* __restrict__ data,
                                             int out_h, int out_w, const ImageBatch b, float mean0, float mean1,
                                             float mean2, int swap_rb) {
  const ImageDesc& D = b.d[blockIdx.y];
  if (D.channels == 3)
    imresize_pass_to_blob<3>(D, mid, data, out_h, out_w, b.n0 + blockIdx.y, mean0, mean1, mean2, swap_rb);
  else
    imresize_pass_to_blob<1>(D, mid, data, out_h, out_w, b.n0 + blockIdx.y, mean0, mean1, mean2, swap_rb);
}

// No resize needed in a dimension (out == in): imresize still runs the pass, and the cubic kernel at
// integer offsets is exactly the identity, so the general kernels are used unchanged.

static int upload(const Contrib& c, DevTable* t) {
  t->taps = c.taps;
  if (cudaMalloc(&t->w, c.w.size() * sizeof(double)) != cudaSuccess) return MSCNN_ERR_NOMEM;
  if (cudaMalloc(&t->idx, c.idx.size() * sizeof(int)) != cudaSuccess) return MSCNN_ERR_NOMEM;
  if (cudaMemcpy(t->w, c.w.data(), c.w.size() * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(t->idx, c.idx.data(), c.idx.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess)
    return MSCNN_ERR_CUDA;
  return MSCNN_OK;
}

static int grow(unsigned char** buf, size_t* cap, size_t need) {
  if (need <= *cap) return MSCNN_OK;
  if (*buf) cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  if (cudaMalloc(buf, need) != cudaSuccess) return MSCNN_ERR_NOMEM;
  *cap = need;
  return MSCNN_OK;
}

static void free_tables(SizeTables* s) {
  cudaFree(s->th.w);
  cudaFree(s->th.idx);
  cudaFree(s->tw.w);
  cudaFree(s->tw.idx);
}

// Index of the tap tables of input size (in_h, in_w) in the plan's cache; built in fp64 and uploaded on first use.
static int tables_for(PreprocessPlan* p, int in_h, int in_w, int* index) {
  for (size_t i = 0; i < p->sizes.size(); ++i)
    if (p->sizes[i].in_h == in_h && p->sizes[i].in_w == in_w) {
      *index = (int)i;
      return MSCNN_OK;
    }
  SizeTables s;
  s.in_h = in_h;
  s.in_w = in_w;
  const double sh = (double)p->d.out_h / in_h, sw = (double)p->d.out_w / in_w;
  s.first_dim = sw < sh ? 1 : 0;  // ascending scale, stable: height first on ties (imresize.m sort(scale))
  int rc = upload(contributions(in_h, p->d.out_h), &s.th);
  if (rc == MSCNN_OK) rc = upload(contributions(in_w, p->d.out_w), &s.tw);
  if (rc != MSCNN_OK) {
    free_tables(&s);
    return rc;
  }
  p->sizes.push_back(s);
  *index = (int)p->sizes.size() - 1;
  return MSCNN_OK;
}

// Sizes >= 1; channel counts 1 or 3 (in_c NULL: every image is colour).
static bool sizes_valid(int N, const int* in_hw, const int* in_c = nullptr) {
  if (N < 1 || !in_hw) return false;
  for (int n = 0; n < N; ++n)
    if (in_hw[2 * n] < 1 || in_hw[2 * n + 1] < 1 || (in_c && in_c[n] != 1 && in_c[n] != 3)) return false;
  return true;
}

static std::vector<int> uniform_sizes(const PreprocessPlan* p, int N) {
  std::vector<int> hw((size_t)2 * N);
  for (int n = 0; n < N; ++n) {
    hw[2 * n] = p->d.in_h;
    hw[2 * n + 1] = p->d.in_w;
  }
  return hw;
}

static unsigned grid_x(size_t work, unsigned cap) {
  const size_t blocks = (work + 255) / 256;
  return (unsigned)(blocks > cap ? cap : blocks);
}

// Images packed back to back in batch order (image n starts at byte sum_{m<n} h_m w_m c_m) -> data
// [N][3][out_h][out_w].  `host` images are first copied into the plan's staging buffer on `st`.  Both passes cover up to
// kImagesPerLaunch images per launch, image = blockIdx.y.
static int forward_sized(PreprocessPlan* p, int N, const int* in_hw, const int* in_c, const unsigned char* images,
                         bool host, float* data, cudaStream_t st) {
  const mscnn_preprocess_desc& d = p->d;
  std::vector<ImageDesc> desc(N);
  size_t src = 0, mid = 0;
  for (int n = 0; n < N; ++n) {
    int t;
    const int rc = tables_for(p, in_hw[2 * n], in_hw[2 * n + 1], &t);
    if (rc != MSCNN_OK) return rc;
    const SizeTables& s = p->sizes[t];
    ImageDesc& D = desc[n];
    D.src = src;
    D.mid = mid;
    D.in_h = s.in_h;
    D.in_w = s.in_w;
    D.channels = in_c ? in_c[n] : 3;
    D.first_dim = s.first_dim;
    D.mid_h = s.first_dim == 0 ? d.out_h : s.in_h;
    D.mid_w = s.first_dim == 0 ? s.in_w : d.out_w;
    D.t1 = s.first_dim == 0 ? s.th : s.tw;
    D.t2 = s.first_dim == 0 ? s.tw : s.th;
    src += (size_t)s.in_h * s.in_w * D.channels;
    mid += (size_t)D.mid_h * D.mid_w * D.channels;
  }
  int rc = grow(&p->mid, &p->mid_cap, mid);
  if (rc == MSCNN_OK && host) rc = grow(&p->stage, &p->stage_cap, src);
  if (rc != MSCNN_OK) return rc;
  if (!p->used && cudaEventCreateWithFlags(&p->used, cudaEventDisableTiming) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (p->used_valid && p->used_on != st && cudaStreamWaitEvent(st, p->used, 0) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (host) {
    if (cudaMemcpyAsync(p->stage, images, src, cudaMemcpyHostToDevice, st) != cudaSuccess) return MSCNN_ERR_CUDA;
    images = p->stage;
  }
  const size_t px = (size_t)d.out_h * d.out_w;
  for (int n0 = 0; n0 < N; n0 += kImagesPerLaunch) {
    const int count = N - n0 < kImagesPerLaunch ? N - n0 : kImagesPerLaunch;
    ImageBatch b;
    b.n0 = n0;
    size_t mid_max = 0;
    for (int i = 0; i < count; ++i) {
      b.d[i] = desc[n0 + i];
      const size_t m = (size_t)b.d[i].mid_h * b.d[i].mid_w * b.d[i].channels;
      if (m > mid_max) mid_max = m;
    }
    const unsigned cap = 132u * 64 / count;  // at most 132 x 64 blocks per launch, as before
    imresize_pass_u8_kernel<<<dim3(grid_x(mid_max, cap), count), 256, 0, st>>>(images, p->mid, b);
    note_launch();
    imresize_pass_to_blob_kernel<<<dim3(grid_x(px, cap), count), 256, 0, st>>>(p->mid, data, d.out_h, d.out_w, b,
                                                                               d.mean[0], d.mean[1], d.mean[2],
                                                                               d.swap_rb);
    note_launch();
  }
  if (cudaEventRecord(p->used, st) != cudaSuccess) return MSCNN_ERR_CUDA;
  p->used_on = st;
  p->used_valid = true;
  return cudaPeekAtLastError() == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}

}  // namespace mscnn

using namespace mscnn;

extern "C" {

int mscnn_imresize_taps(int in_len, int out_len) {
  if (in_len < 1 || out_len < 1) return MSCNN_ERR_INVALID;
  return contributions(in_len, out_len).taps;
}

int mscnn_imresize_contributions(int in_len, int out_len, double* host_weights, int* host_indices, int cap_taps) {
  if (in_len < 1 || out_len < 1 || !host_weights || !host_indices) return MSCNN_ERR_INVALID;
  const Contrib c = contributions(in_len, out_len);
  if (c.taps > cap_taps) return MSCNN_ERR_INVALID;
  for (int o = 0; o < out_len; ++o)
    for (int k = 0; k < c.taps; ++k) {
      host_weights[(size_t)o * cap_taps + k] = c.w[(size_t)o * c.taps + k];
      host_indices[(size_t)o * cap_taps + k] = c.idx[(size_t)o * c.taps + k];
    }
  return c.taps;
}

int mscnn_widerface_net_size(int org_h, int org_w, int img_h, int img_w, int max_size, int* rz_h, int* rz_w) {
  if (org_h < 1 || org_w < 1 || !rz_h || !rz_w || max_size < 32) return MSCNN_ERR_INVALID;
  // examples/widerface/run_mscnn_detection.m:72-80 (MATLAB round = half away from zero)
  double w = img_w == 0 ? org_w : img_w, h = img_h == 0 ? org_h : img_h;
  w = round(w / 32.0) * 32.0;
  h = round(h / 32.0) * 32.0;
  if (h > max_size || w > max_size) {
    const double r = (double)max_size / fmax(h, w);
    h = round(h * r / 32.0) * 32.0;
    w = round(w * r / 32.0) * 32.0;
  }
  *rz_h = (int)h;
  *rz_w = (int)w;
  return MSCNN_OK;
}

int mscnn_preprocess_create(const mscnn_preprocess_desc* d, void** plan) {
  if (!d || !plan || d->in_h < 1 || d->in_w < 1 || d->out_h < 1 || d->out_w < 1) return MSCNN_ERR_INVALID;
  PreprocessPlan* p = new PreprocessPlan();
  p->d = *d;
  int first;
  const int rc = tables_for(p, d->in_h, d->in_w, &first);
  if (rc != MSCNN_OK) {
    mscnn_preprocess_destroy(p);
    return rc;
  }
  *plan = p;
  return MSCNN_OK;
}

int mscnn_preprocess_get_desc(void* plan, mscnn_preprocess_desc* d) {
  if (!plan || !d) return MSCNN_ERR_INVALID;
  *d = static_cast<PreprocessPlan*>(plan)->d;
  return MSCNN_OK;
}

int mscnn_preprocess_destroy(void* plan) {
  PreprocessPlan* p = static_cast<PreprocessPlan*>(plan);
  if (!p) return MSCNN_OK;
  for (SizeTables& s : p->sizes) free_tables(&s);
  cudaFree(p->mid);
  cudaFree(p->stage);
  if (p->used) cudaEventDestroy(p->used);
  delete p;
  return MSCNN_OK;
}

int mscnn_preprocess_forward_sized_c(void* plan, int N, const int* in_hw, const int* in_c,
                                     const unsigned char* images, float* data, void* stream) {
  PreprocessPlan* p = static_cast<PreprocessPlan*>(plan);
  if (!p || !sizes_valid(N, in_hw, in_c) || !images || !data) return MSCNN_ERR_INVALID;
  return forward_sized(p, N, in_hw, in_c, images, false, data, (cudaStream_t)stream);
}

int mscnn_preprocess_forward_sized_c_host(void* plan, int N, const int* in_hw, const int* in_c,
                                          const unsigned char* host_images, float* data, void* stream) {
  PreprocessPlan* p = static_cast<PreprocessPlan*>(plan);
  if (!p || !sizes_valid(N, in_hw, in_c) || !host_images || !data) return MSCNN_ERR_INVALID;
  return forward_sized(p, N, in_hw, in_c, host_images, true, data, (cudaStream_t)stream);
}

int mscnn_preprocess_forward_sized(void* plan, int N, const int* in_hw, const unsigned char* images, float* data,
                                   void* stream) {
  return mscnn_preprocess_forward_sized_c(plan, N, in_hw, nullptr, images, data, stream);
}

int mscnn_preprocess_forward_sized_host(void* plan, int N, const int* in_hw, const unsigned char* host_images,
                                        float* data, void* stream) {
  return mscnn_preprocess_forward_sized_c_host(plan, N, in_hw, nullptr, host_images, data, stream);
}

// The uniform batch: every image has the plan's own input size.
int mscnn_preprocess_forward(void* plan, int N, const unsigned char* images, float* data, void* stream) {
  PreprocessPlan* p = static_cast<PreprocessPlan*>(plan);
  if (!p || N < 1 || !images || !data) return MSCNN_ERR_INVALID;
  return mscnn_preprocess_forward_sized(plan, N, uniform_sizes(p, N).data(), images, data, stream);
}

int mscnn_preprocess_forward_host(void* plan, int N, const unsigned char* host_images, float* data, void* stream) {
  PreprocessPlan* p = static_cast<PreprocessPlan*>(plan);
  if (!p || N < 1 || !host_images || !data) return MSCNN_ERR_INVALID;
  return mscnn_preprocess_forward_sized_host(plan, N, uniform_sizes(p, N).data(), host_images, data, stream);
}

}  // extern "C"
