// Layer implementations of the Caffe-API mirror: parameter parsing and shapes follow the
// reference layer sources (cited per method); the arithmetic is delegated to the C ABI.
#include <cstring>
#include <random>
#include <string>

#include "caffe/layers/mscnn_layers.hpp"
#include "config.h"
#include "deconv_phase.h"
#include "launch_count.h"

namespace caffe {

static inline int pad64(int c) { return (c + 63) / 64 * 64; }
static inline int out_pad(int c) { return c > 32 ? pad64(c) : 32; }

PackedBias::~PackedBias() {
  if (data) cudaFree(data);
}
void PackedBias::update(Blob<float>* b, int n, int n_pad) {
  const unsigned long ver = b ? b->version() : 0;
  if (data && len == n_pad && src == b && version == ver) return;
  if (data && len != n_pad) { CUDA_CHECK(cudaFree(data)); data = nullptr; }
  if (!data) CUDA_CHECK(cudaMalloc(&data, sizeof(float) * n_pad));
  CUDA_CHECK(cudaMemsetAsync(data, 0, sizeof(float) * n_pad, Caffe::stream()));
  if (b)
    CUDA_CHECK(cudaMemcpyAsync(data, b->gpu_data(), sizeof(float) * n, cudaMemcpyDeviceToDevice, Caffe::stream()));
  len = n_pad;
  src = b;
  version = ver;
}
template <typename Pack>
void PackedParam::update_weights(Blob<float>* wb, const Layout& l, size_t bytes, Pack pack) {
  const unsigned long ver = wb->version();
  if (img && w_version == ver && memcmp(&layout, &l, sizeof(l)) == 0) return;
  shared_ptr<PackedImage> im = wb->packed_image(std::string(reinterpret_cast<const char*>(&l), sizeof(l)));
  const cudaStream_t s = Caffe::stream();
  {
    std::lock_guard<std::mutex> lk(im->mu);  // one thread packs a given version
    if (im->version != ver) {
      im->w.reserve(bytes, l.split);
      pack(wb->gpu_data(), im->w.hi, l.split ? im->w.lo : nullptr);
      if (!im->ready) CUDA_CHECK(cudaEventCreateWithFlags(&im->ready, cudaEventDisableTiming));
      CUDA_CHECK(cudaEventRecord(im->ready, s));
      im->version = ver;
      mscnn::g_weight_packs.fetch_add(1, std::memory_order_relaxed);
    } else {
      // packed by a layer that shares the storage, maybe on another thread's stream
      CUDA_CHECK(cudaStreamWaitEvent(s, im->ready, 0));
    }
  }
  img = im;
  layout = l;
  w_version = ver;
}

// The mscnn_conv_desc fields every route through mscnn_conv_forward shares; the caller sets out_mode, the outputs,
// pooling and relu.
static mscnn_conv_desc conv_desc(const Blob<float>::Planes& x, const PackedParam& pk, int N, int H, int W, int C,
                                 int cout, int kh, int kw, int pad_h, int pad_w, const int* dyn_n) {
  mscnn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.x_hi = x.hi; d.x_lo = x.lo;
  d.N = N; d.H = H; d.W = W; d.C = C;
  d.w_hi = pk.hi(); d.w_lo = pk.lo();
  d.bias = pk.bias.data;
  d.Cout = cout; d.Cout_pad = pk.layout.out_pad;
  d.KH = kh; d.KW = kw;
  d.pad_h = pad_h; d.pad_w = pad_w;
  d.dyn_n = dyn_n;
  return d;
}

// Defines T::Accesses (Layer::Accesses), whose parameters are bottom, top and out.
#define LAYER_ACCESSES(T)                                                                                              \
  template <typename Dtype>                                                                                           \
  bool T<Dtype>::Accesses(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top,                       \
                          BlobAccesses<Dtype>* out) const

// every blob of `blobs` in representation a
template <typename Dtype>
static bool access_all(BlobAccesses<Dtype>* out, const vector<Blob<Dtype>*>& blobs, Access a) {
  for (size_t k = 0; k < blobs.size(); ++k) out->push_back(make_pair(blobs[k], a));
  return true;
}

void FillBlob(const FillerParameter& filler, Blob<float>* blob) {
  const std::string& type = filler.type();
  float* data = blob->mutable_cpu_data();
  const int n = blob->count();
  if (type == "constant") {  // filler.hpp:36-51
    for (int i = 0; i < n; ++i) data[i] = filler.value();
  } else if (type == "gaussian") {  // filler.hpp:70-107 (without sparsity)
    CHECK_EQ(filler.sparse(), -1) << "sparse gaussian filler is not supported";
    std::mt19937 gen(1706);
    std::normal_distribution<float> dist(filler.mean(), filler.std());
    for (int i = 0; i < n; ++i) data[i] = dist(gen);
  } else if (type == "bilinear") {  // filler.hpp:244-262
    CHECK_EQ(blob->num_axes(), 4) << "Blob must be 4 dim.";
    CHECK_EQ(blob->width(), blob->height()) << "Filter must be square";
    const int f = (int)std::ceil(blob->width() / 2.);
    const float c = (2 * f - 1 - f % 2) / (2. * f);
    for (int i = 0; i < n; ++i) {
      const float x = i % blob->width();
      const float y = (i / blob->width()) % blob->height();
      data[i] = (1 - std::fabs(x / f - c)) * (1 - std::fabs(y / f - c));
    }
  } else {
    LOG(FATAL) << "Unknown or unsupported filler name: " << type;
  }
}

// ---------------------------------------------------------------------------------- Input
template <typename Dtype>
void InputLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const int num_top = (int)top.size();
  const InputParameter& param = this->layer_param_.input_param();
  const int num_shape = param.shape_size();
  CHECK(num_shape == 0 || num_shape == 1 || num_shape == num_top)
      << "Must specify 'shape' once, once per top blob, or not at all: " << num_top << " tops vs. "
      << num_shape << " shapes.";
  if (num_shape > 0) {
    for (int i = 0; i < num_top; ++i) top[i]->Reshape(param.shape(num_shape == 1 ? 0 : i));
  }
}
LAYER_ACCESSES(InputLayer) { return access_all(out, top, NCHW); }

// Kernel, pad, stride and dilation of a 2-D ConvolutionParameter (base_conv_layer.cpp:27-108), shared by Convolution
// and Deconvolution.
static void ParseConvGeometry(const ConvolutionParameter& p, int* kh, int* kw, int* ph, int* pw, int* sh, int* sw,
                              int* dh, int* dw) {
  if (p.has_kernel_h() || p.has_kernel_w()) {
    CHECK_EQ(0, p.kernel_size_size()) << "Either kernel_size or kernel_h/w should be specified; not both.";
    *kh = p.kernel_h();
    *kw = p.kernel_w();
  } else {
    CHECK(p.kernel_size_size() == 1 || p.kernel_size_size() == 2) << "kernel_size must be specified once or twice";
    *kh = p.kernel_size(0);
    *kw = p.kernel_size(p.kernel_size_size() == 1 ? 0 : 1);
  }
  CHECK_GT(*kh, 0) << "Filter dimensions must be nonzero.";
  CHECK_GT(*kw, 0) << "Filter dimensions must be nonzero.";
  if (p.has_pad_h() || p.has_pad_w()) {
    *ph = p.pad_h();
    *pw = p.pad_w();
  } else {
    *ph = p.pad_size() > 0 ? p.pad(0) : 0;
    *pw = p.pad_size() > 1 ? p.pad(1) : *ph;
  }
  *sh = 1;
  *sw = 1;
  if (p.has_stride_h() || p.has_stride_w()) {
    *sh = p.stride_h();
    *sw = p.stride_w();
  } else if (p.stride_size() > 0) {
    *sh = p.stride(0);
    *sw = p.stride_size() > 1 ? p.stride(1) : *sh;
  }
  CHECK_GT(*sh, 0) << "Stride dimensions must be nonzero.";
  CHECK_GT(*sw, 0) << "Stride dimensions must be nonzero.";
  CHECK_LE(p.dilation_size(), 2) << "dilation must be specified once, or once per spatial dimension";
  *dh = p.dilation_size() > 0 ? p.dilation(0) : 1;  // base_conv_layer.cpp:95-108
  *dw = p.dilation_size() > 1 ? p.dilation(1) : *dh;
  CHECK_GT(*dh, 0) << "dilation must be nonzero.";
  CHECK_GT(*dw, 0) << "dilation must be nonzero.";
}

// ---------------------------------------------------------------------------- Convolution
template <typename Dtype>
void ConvolutionLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  // base_conv_layer.cpp:15-180, 2-D case
  const ConvolutionParameter& p = this->layer_param_.convolution_param();
  CHECK_EQ(bottom[0]->num_axes(), 4) << "mscnn_b200 Convolution takes 4-D bottoms";
  ParseConvGeometry(p, &kernel_h_, &kernel_w_, &pad_h_, &pad_w_, &stride_h_, &stride_w_, &dilation_h_, &dilation_w_);
  CHECK(stride_h_ <= 4 && stride_w_ <= 4) << "mscnn_b200 Convolution serves strides 1..4 (layer "
                                          << this->layer_param_.name() << ")";
  channels_ = bottom[0]->channels();
  num_output_ = p.num_output();
  CHECK_GT(num_output_, 0);
  group_ = p.group();  // base_conv_layer.cpp:121-124
  CHECK_GT(group_, 0);
  CHECK_EQ(channels_ % group_, 0);
  CHECK_EQ(num_output_ % group_, 0) << "Number of output should be multiples of group.";
  CHECK(group_ == 1 || (channels_ / group_ % 64 == 0 && num_output_ / group_ % 64 == 0))
      << "mscnn_b200 Convolution serves group > 1 only when the input and output channels of one group are multiples "
         "of 64 (layer " << this->layer_param_.name() << ": " << channels_ << " -> " << num_output_ << ", group "
      << group_ << ")";
  bias_term_ = p.bias_term();
  if (this->blobs_.size() > 0) {
    CHECK_EQ((int)this->blobs_.size(), 1 + (bias_term_ ? 1 : 0)) << "Incorrect number of weight blobs.";
  } else {
    this->blobs_.resize(bias_term_ ? 2 : 1);
    this->blobs_[0].reset(new Blob<Dtype>(num_output_, channels_ / group_, kernel_h_, kernel_w_));
    FillBlob(p.weight_filler(), this->blobs_[0].get());
    if (bias_term_) {
      this->blobs_[1].reset(new Blob<Dtype>(vector<int>(1, num_output_)));
      FillBlob(p.bias_filler(), this->blobs_[1].get());
    }
  }
}

template <typename Dtype>
void ConvolutionLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK_EQ(bottom[0]->channels(), channels_) << "Input size incompatible with convolution kernel.";
  // conv_layer.cpp:8-22
  const int ho = (bottom[0]->height() + 2 * pad_h_ - (dilation_h_ * (kernel_h_ - 1) + 1)) / stride_h_ + 1;
  const int wo = (bottom[0]->width() + 2 * pad_w_ - (dilation_w_ * (kernel_w_ - 1) + 1)) / stride_w_ + 1;
  top[0]->Reshape(bottom[0]->num(), num_output_, ho, wo);
}

template <typename Dtype>
void ConvolutionLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const bool split = Caffe::split();
  const int N = bottom[0]->num(), H = bottom[0]->height(), W = bottom[0]->width();
  Blob<Dtype>* wb = this->blobs_[0].get();
  Blob<Dtype>* bias = bias_term_ ? this->blobs_[1].get() : nullptr;
  // Narrow k x k proposal heads (LFCN_*: 9 or 6 outputs, 5x5 / 7x7, "same" padding): the horizontal
  // taps move into the GEMM's N dimension and a 1-D gather sums them (mscnn_head_gather in the C ABI).
  const bool head_path = (num_output_ == 9 || num_output_ == 6) && kernel_h_ == kernel_w_ && kernel_h_ > 1 &&
                         pad_h_ == pad_w_ && 2 * pad_h_ + 1 == kernel_h_ && !fuse_relu_ && channels_ % 64 == 0 &&
                         plain_geometry() && !mscnn::config().no_head_taps;
  if (head_path) {
    const int k = kernel_h_;
    const int n_pad = (k * num_output_ + 63) / 64 * 64;
    packed_.update_weights(wb, {PackedParam::HEAD, split, n_pad, channels_, 0, 0, 0},
                           (size_t)n_pad * k * channels_ * 2, [&](const float* w, void* hi, void* lo) {
      MSCNN_CHECK(mscnn_pack_head_weights(w, hi, lo, num_output_, channels_, k, n_pad, channels_, Caffe::stream()));
    });
    packed_.bias.update(nullptr, 0, n_pad);  // the bias is added by the gather
    packed_.gather_bias.update(bias, num_output_, num_output_);
    typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
    float* P = static_cast<float*>(Caffe::scratch((size_t)N * H * W * n_pad * sizeof(float)));
    // vertical taps stay in K, horizontal taps are columns of P
    mscnn_conv_desc d = conv_desc(x, packed_, N, H, W, x.cpad, n_pad, k, 1, pad_h_, 0, this->dyn_rows_device());
    d.out_mode = MSCNN_OUT_NHWC_F32;
    d.y_f32 = P;
    MSCNN_CHECK(mscnn_conv_forward(&d, Caffe::stream()));
    MSCNN_CHECK(mscnn_head_gather(P, n_pad, packed_.gather_bias.data, top[0]->mutable_gpu_data(), N, H, W, num_output_,
                                  k, pad_h_, Caffe::stream()));
    return;
  }
  // conv1_1 (3 -> 64 channels, 3x3, pad 1): K = 27 is far below one 64-channel tensor-core k-block.
  // One kernel from the fp32 NCHW blob to planes: pixel rows staged once, the horizontal taps are
  // descriptor-shifted views of them (mscnn_conv1_tc_forward, conv_c3_tc.cu).  Its packed image serves
  // both precisions, so a precision switch does not re-pack it.
  if (is_conv1_1()) {
    packed_.update_weights(wb, {PackedParam::CONV1_1, 0, 64, 0, 0, 0, 0}, (size_t)mscnn_conv1_tc_packed_bytes(),
                           [](const float* w, void* hi, void*) {
      MSCNN_CHECK(mscnn_pack_conv1_tc_weights(w, hi, 1, Caffe::stream()));
    });
    packed_.bias.update(bias, 64, 64);
    typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
    MSCNN_CHECK(mscnn_conv1_tc_forward(bottom[0]->gpu_data(), packed_.hi(), packed_.bias.data, y.hi,
                                       split ? y.lo : nullptr, N, H, W, fuse_relu_ ? 1 : 0, Caffe::stream()));
    return;
  }
  // The blob [Cout][Cin / group][kh][kw] packs to planes [Cout_pad][kh][kw][cin_pad]: with groups, group k's rows are
  // [k Cout / group, (k + 1) Cout / group) and their channels are the group's own.
  const int cout_pad = out_pad(num_output_), cin_g = channels_ / group_, cin_pad = pad64(cin_g);
  const size_t bytes = (size_t)cout_pad * kernel_h_ * kernel_w_ * cin_pad * 2;
  packed_.update_weights(wb, {PackedParam::CONV, split, cout_pad, cin_pad, 0, 0, 0}, bytes,
                         [&](const float* w, void* hi, void* lo) {
    MSCNN_CHECK(mscnn_pack_conv_weights(w, hi, lo, num_output_, cin_g, kernel_h_, kernel_w_, cout_pad, cin_pad,
                                        Caffe::stream()));
  });
  packed_.bias.update(bias, num_output_, cout_pad);
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  mscnn_conv_desc d = conv_desc(x, packed_, N, H, W, x.cpad, num_output_, kernel_h_, kernel_w_, pad_h_, pad_w_,
                                this->dyn_rows_device());
  d.relu = fuse_relu_ ? 1 : 0;
  d.stride_h = stride_h_; d.stride_w = stride_w_;
  d.dil_h = dilation_h_; d.dil_w = dilation_w_;
  d.group = group_;
  if (planes_top()) {
    d.out_mode = MSCNN_OUT_NHWC_BF16;
    const int ho = top[0]->height(), wo = top[0]->width();
    const bool pool_here = pools_here(*top[0]);
    if (!pool_here || store_full_) {
      typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
      d.y_hi = y.hi;
      d.y_lo = y.lo;
    }
    if (pool_here) {
      fused_pool_top_->Reshape(top[0]->num(), num_output_, ho / 2, wo / 2);
      typename Blob<Dtype>::Planes q = fused_pool_top_->mutable_planes(split);
      d.pool_hi = q.hi;
      d.pool_lo = q.lo;
    }
  } else {
    d.out_mode = MSCNN_OUT_NCHW_F32;  // narrow heads (LFCN_*): straight into the Caffe layout
    d.y_f32 = top[0]->mutable_gpu_data();
  }
  MSCNN_CHECK(mscnn_conv_forward(&d, Caffe::stream()));
}
LAYER_ACCESSES(ConvolutionLayer) {
  out->push_back(make_pair(bottom[0], is_conv1_1() ? NCHW : PLANES));
  if (!pools_here(*top[0])) return access_all(out, top, planes_top() ? PLANES : NCHW);
  if (store_full_) out->push_back(make_pair(top[0], PLANES));  // else the un-pooled top is not written
  out->push_back(make_pair(fused_pool_top_, PLANES));
  return true;
}

// -------------------------------------------------------------------------- Deconvolution
template <typename Dtype>
void DeconvolutionLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  // base_conv_layer.cpp:15-180, 2-D case, with the channel axes reversed (deconv_layer.hpp: reverse_dimensions)
  const ConvolutionParameter& p = this->layer_param_.convolution_param();
  const std::string& name = this->layer_param_.name();
  CHECK_EQ(bottom[0]->num_axes(), 4) << "mscnn_b200 Deconvolution takes 4-D bottoms";
  ParseConvGeometry(p, &kernel_h_, &kernel_w_, &pad_h_, &pad_w_, &stride_h_, &stride_w_, &dilation_h_, &dilation_w_);
  channels_ = bottom[0]->channels();
  num_output_ = p.num_output();
  CHECK_GT(num_output_, 0);
  group_ = p.group();  // base_conv_layer.cpp:121-124
  CHECK_GT(group_, 0);
  CHECK_EQ(channels_ % group_, 0);
  CHECK_EQ(num_output_ % group_, 0) << "Number of output should be multiples of group.";
  CHECK(stride_h_ <= mscnn::kDeconvMaxStride && stride_w_ <= mscnn::kDeconvMaxStride)
      << "mscnn_b200 Deconvolution serves strides 1..8 (layer " << name << ")";
  CHECK(mscnn::deconv_axis_ok(kernel_h_, stride_h_, pad_h_, dilation_h_) &&
        mscnn::deconv_axis_ok(kernel_w_, stride_w_, pad_w_, dilation_w_))
      << "mscnn_b200 Deconvolution serves pads and dilated kernel reaches up to 2^20 (layer " << name << ")";
  CHECK(!(group_ == channels_ && group_ > 1 && num_output_ != channels_))
      << "mscnn_b200 Deconvolution does not serve a depthwise layer with a channel multiplier (layer " << name << ": "
      << channels_ << " -> " << num_output_ << ", group " << group_ << ")";
  CHECK(group_ == 1 || depthwise() || (channels_ / group_ % 64 == 0 && num_output_ / group_ % 64 == 0))
      << "mscnn_b200 Deconvolution serves group > 1 only when the input and output channels of one group are 1 "
         "(depthwise) or multiples of 64 (layer " << name << ": " << channels_ << " -> " << num_output_ << ", group "
      << group_ << ")";
  bias_term_ = p.bias_term();
  if (this->blobs_.size() > 0) {
    CHECK_EQ((int)this->blobs_.size(), 1 + (bias_term_ ? 1 : 0)) << "Incorrect number of weight blobs.";
  } else {
    this->blobs_.resize(bias_term_ ? 2 : 1);
    this->blobs_[0].reset(new Blob<Dtype>(channels_, num_output_ / group_, kernel_h_, kernel_w_));
    FillBlob(p.weight_filler(), this->blobs_[0].get());
    if (bias_term_) {
      this->blobs_[1].reset(new Blob<Dtype>(vector<int>(1, num_output_)));
      FillBlob(p.bias_filler(), this->blobs_[1].get());
    }
  }
}

template <typename Dtype>
void DeconvolutionLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK_EQ(bottom[0]->channels(), channels_) << "Input size incompatible with convolution kernel.";
  // deconv_layer.cpp:8-22
  const int ho = mscnn::deconv_out_size(bottom[0]->height(), kernel_h_, stride_h_, pad_h_, dilation_h_);
  const int wo = mscnn::deconv_out_size(bottom[0]->width(), kernel_w_, stride_w_, pad_w_, dilation_w_);
  CHECK(ho > 0 && wo > 0) << "mscnn_b200 Deconvolution: the output extent " << ho << " x " << wo
                          << " is not positive (layer " << this->layer_param_.name() << ")";
  top[0]->Reshape(bottom[0]->num(), num_output_, ho, wo);
}

template <typename Dtype>
void DeconvolutionLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const bool split = Caffe::split();
  Blob<Dtype>* wb = this->blobs_[0].get();
  Blob<Dtype>* bias = bias_term_ ? this->blobs_[1].get() : nullptr;
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  // group == channels == num_output: a gather per output pixel straight from the blob [C][1][kh][kw]
  if (depthwise()) {
    typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
    MSCNN_CHECK(mscnn_deconv_depthwise_forward(x.hi, x.lo, wb->gpu_data(), bias ? bias->gpu_data() : nullptr, y.hi,
                                               y.lo, x.n, x.h, x.w, x.cpad, channels_, kernel_h_, kernel_w_, stride_h_,
                                               stride_w_, pad_h_, pad_w_, dilation_h_, dilation_w_, Caffe::stream()));
    return;
  }
  // The blob [Cin][Cout / group][kh][kw] packs into one stride-1 sub-kernel per output phase
  // (mscnn_pack_deconv_weights), each [Cout_pad][m_h][m_w][cin_pad].
  const int cout_pad = pad64(num_output_), cin_pad = pad64(channels_ / group_);
  const long long elems = mscnn_deconv_packed_elems(channels_, num_output_, group_, kernel_h_, kernel_w_, stride_h_,
                                                    stride_w_, pad_h_, pad_w_, dilation_h_, dilation_w_, cout_pad);
  CHECK_GE(elems, 0);
  packed_.update_weights(wb, {PackedParam::DECONV, split, cout_pad, cin_pad, 0, 0, 0,
                              {stride_h_, stride_w_, pad_h_, pad_w_, dilation_h_, dilation_w_}}, (size_t)elems * 2,
                         [&](const float* w, void* hi, void* lo) {
    MSCNN_CHECK(mscnn_pack_deconv_weights(w, hi, lo, channels_, num_output_, group_, kernel_h_, kernel_w_, stride_h_,
                                          stride_w_, pad_h_, pad_w_, dilation_h_, dilation_w_, cout_pad,
                                          Caffe::stream()));
  });
  packed_.bias.update(bias, num_output_, cout_pad);
  mscnn_conv_desc d = conv_desc(x, packed_, x.n, x.h, x.w, x.cpad, num_output_, kernel_h_, kernel_w_, pad_h_, pad_w_,
                                nullptr);
  d.stride_h = stride_h_; d.stride_w = stride_w_;
  d.dil_h = dilation_h_; d.dil_w = dilation_w_;
  d.group = group_;
  d.out_mode = MSCNN_OUT_NHWC_BF16;
  typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
  d.y_hi = y.hi;
  d.y_lo = y.lo;
  MSCNN_CHECK(mscnn_deconv_forward(&d, Caffe::stream()));
}
LAYER_ACCESSES(DeconvolutionLayer) { return access_all(out, bottom, PLANES) && access_all(out, top, PLANES); }

// ----------------------------------------------------------------------------------- ReLU
template <typename Dtype>
void ReLULayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK_EQ(this->layer_param_.relu_param().negative_slope(), 0.f) << "leaky ReLU is not supported";
}
template <typename Dtype>
void ReLULayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  if (fused_) return;  // the producing Convolution / InnerProduct already clamped at zero
  if (top[0] != bottom[0]) top[0]->CopyFrom(*bottom[0], false, true);
  if (top[0]->head_is_planes()) {
    typename Blob<Dtype>::Planes p = top[0]->planes(Caffe::split());
    MSCNN_CHECK(mscnn_relu_planes(p.hi, p.lo, (size_t)p.n * p.h * p.w * p.cpad, Caffe::stream()));
    top[0]->mutable_planes(p.lo != nullptr);  // mark planes as the (modified) head
  } else {
    MSCNN_CHECK(mscnn_relu_f32(top[0]->mutable_gpu_data(), top[0]->count(), Caffe::stream()));
  }
}
LAYER_ACCESSES(ReLULayer) {
  if (fused_) return true;
  if (top[0] == bottom[0]) return access_all(out, top, TOUCH);
  return access_all(out, bottom, NCHW) && access_all(out, top, NCHW);
}

// -------------------------------------------------------------------------------- Pooling
template <typename Dtype>
void PoolingLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const PoolingParameter& p = this->layer_param_.pooling_param();  // pooling_layer.cpp:16-77
  global_pooling_ = p.global_pooling();
  if (global_pooling_) {
    CHECK(!(p.has_kernel_size() || p.has_kernel_h() || p.has_kernel_w()))
        << "With Global_pooling: true Filter size cannot specified";
  } else {
    CHECK(!p.has_kernel_size() != !(p.has_kernel_h() && p.has_kernel_w()))
        << "Filter size is kernel_size OR kernel_h and kernel_w; not both";
    CHECK(p.has_kernel_size() || (p.has_kernel_h() && p.has_kernel_w()))
        << "For non-square filters both kernel_h and kernel_w are required.";
  }
  CHECK((!p.has_pad() && p.has_pad_h() && p.has_pad_w()) || (!p.has_pad_h() && !p.has_pad_w()))
      << "pad is pad OR pad_h and pad_w are required.";
  CHECK((!p.has_stride() && p.has_stride_h() && p.has_stride_w()) || (!p.has_stride_h() && !p.has_stride_w()))
      << "Stride is stride OR stride_h and stride_w are required.";
  if (global_pooling_) {
    kernel_h_ = bottom[0]->height();
    kernel_w_ = bottom[0]->width();
  } else {
    kernel_h_ = p.has_kernel_size() ? p.kernel_size() : p.kernel_h();
    kernel_w_ = p.has_kernel_size() ? p.kernel_size() : p.kernel_w();
  }
  CHECK_GT(kernel_h_, 0) << "Filter dimensions cannot be zero.";
  CHECK_GT(kernel_w_, 0) << "Filter dimensions cannot be zero.";
  pad_h_ = p.has_pad_h() ? p.pad_h() : p.pad();
  pad_w_ = p.has_pad_h() ? p.pad_w() : p.pad();
  stride_h_ = p.has_stride_h() ? p.stride_h() : p.stride();
  stride_w_ = p.has_stride_h() ? p.stride_w() : p.stride();
  CHECK_GT(stride_h_, 0) << "Stride cannot be zero.";
  CHECK_GT(stride_w_, 0) << "Stride cannot be zero.";
  if (global_pooling_)
    CHECK(pad_h_ == 0 && pad_w_ == 0 && stride_h_ == 1 && stride_w_ == 1)
        << "With Global_pooling: true; only pad = 0 and stride = 1";
  CHECK_LT(pad_h_, kernel_h_);
  CHECK_LT(pad_w_, kernel_w_);
  CHECK(p.pool() == PoolingParameter_PoolMethod_MAX || p.pool() == PoolingParameter_PoolMethod_AVE)
      << "MAX and AVE pooling only (STOCHASTIC is a training mode)";
  mode_ = p.pool() == PoolingParameter_PoolMethod_MAX ? MSCNN_POOL_MAX : MSCNN_POOL_AVE;
}
template <typename Dtype>
void PoolingLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK_EQ(4, bottom[0]->num_axes()) << "Input must have 4 axes";
  if (global_pooling_) {  // pooling_layer.cpp:86-89: follows a net that changes its input size
    kernel_h_ = bottom[0]->height();
    kernel_w_ = bottom[0]->width();
  }
  // pooling_layer.cpp:90-105
  pooled_h_ = mscnn_pool_output_size(bottom[0]->height(), kernel_h_, stride_h_, pad_h_);
  pooled_w_ = mscnn_pool_output_size(bottom[0]->width(), kernel_w_, stride_w_, pad_w_);
  CHECK(pooled_h_ > 0 && pooled_w_ > 0) << "Pooling layer " << this->layer_param_.name() << ": kernel " << kernel_h_
                                        << "x" << kernel_w_ << " does not fit the " << bottom[0]->height() << "x"
                                        << bottom[0]->width() << " bottom";
  top[0]->Reshape(bottom[0]->num(), bottom[0]->channels(), pooled_h_, pooled_w_);
}
template <typename Dtype>
void PoolingLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  if (pooled_by_conv(*bottom[0])) return;  // computed in the producing convolution's epilogue
  const bool split = Caffe::split();
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
  MSCNN_CHECK(mscnn_pool2d_forward_dyn(x.hi, x.lo, y.hi, y.lo, x.n, x.h, x.w, x.cpad, kernel_h_, kernel_w_, stride_h_,
                                       stride_w_, pad_h_, pad_w_, mode_, this->dyn_rows_device(), Caffe::stream()));
}
LAYER_ACCESSES(PoolingLayer) {
  if (pooled_by_conv(*bottom[0])) return true;  // the convolution writes the top
  return access_all(out, bottom, PLANES) && access_all(out, top, PLANES);
}

// ---------------------------------------------------------------------------------- Split
template <typename Dtype>
void SplitLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  for (size_t i = 0; i < top.size(); ++i) {
    CHECK_NE(top[i], bottom[0]) << this->type() << " Layer does not allow in-place computation.";
    top[i]->ReshapeLike(*bottom[0]);
  }
}
template <typename Dtype>
void SplitLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  for (size_t i = 0; i < top.size(); ++i) top[i]->ShareData(*bottom[0]);
}
LAYER_ACCESSES(SplitLayer) { return true; }  // the tops are on the bottom's storage (TopsShareBottom)

// --------------------------------------------------------------------------------- Concat
template <typename Dtype>
void ConcatLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const ConcatParameter& p = this->layer_param_.concat_param();
  CHECK(!(p.has_axis() && p.has_concat_dim())) << "Either axis or concat_dim should be specified; not both.";
  const int axis = p.has_concat_dim() ? (int)p.concat_dim() : bottom[0]->CanonicalAxisIndex(p.axis());
  CHECK_EQ(axis, 1) << "mscnn_b200 Concat supports the channel axis only";
}
template <typename Dtype>
void ConcatLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  vector<int> shape = bottom[0]->shape();  // concat_layer.cpp:28-55
  for (size_t i = 1; i < bottom.size(); ++i) {
    CHECK_EQ(bottom[0]->num_axes(), bottom[i]->num_axes()) << "All inputs must have the same #axes.";
    for (int j = 0; j < bottom[0]->num_axes(); ++j)
      if (j != 1) CHECK_EQ(shape[j], bottom[i]->shape(j)) << "All inputs must have the same shape, except at concat_axis.";
    shape[1] += bottom[i]->shape(1);
  }
  top[0]->Reshape(shape);
}
template <typename Dtype>
void ConcatLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  if (fused_) return;  // ROIPooling producers already wrote their channel ranges of top[0]
  if (TopsShareBottom(bottom)) { top[0]->ShareData(*bottom[0]); return; }
  const bool split = Caffe::split();
  if (aligned(bottom)) {
    typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
    int off = 0;
    for (size_t i = 0; i < bottom.size(); ++i) {
      typename Blob<Dtype>::Planes x = bottom[i]->planes(split);
      const size_t pixels = (size_t)x.n * x.h * x.w;
      MSCNN_CHECK(mscnn_concat_planes(x.hi, y.hi, pixels, x.cpad, y.cpad, off, Caffe::stream()));
      if (split) MSCNN_CHECK(mscnn_concat_planes(x.lo, y.lo, pixels, x.cpad, y.cpad, off, Caffe::stream()));
      off += x.cpad;
    }
  } else {
    Dtype* dst = top[0]->mutable_gpu_data();
    const int num = top[0]->num();
    const size_t inner = (size_t)top[0]->count(2);
    const size_t top_row = (size_t)top[0]->channels() * inner;
    size_t off = 0;
    for (size_t i = 0; i < bottom.size(); ++i) {
      const size_t row = (size_t)bottom[i]->channels() * inner;
      CUDA_CHECK(cudaMemcpy2DAsync(dst + off, top_row * sizeof(Dtype), bottom[i]->gpu_data(), row * sizeof(Dtype),
                                   row * sizeof(Dtype), num, cudaMemcpyDeviceToDevice, Caffe::stream()));
      off += row;
    }
  }
}
LAYER_ACCESSES(ConcatLayer) {
  if (fused_ || TopsShareBottom(bottom)) return true;  // fused: the ROIPooling producers write the top
  const Access a = aligned(bottom) ? PLANES : NCHW;
  return access_all(out, bottom, a) && access_all(out, top, a);
}

// --------------------------------------------------------------------------- InnerProduct
template <typename Dtype>
void InnerProductLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const InnerProductParameter& p = this->layer_param_.inner_product_param();  // inner_product_layer.cpp:10-56
  N_ = p.num_output();
  bias_term_ = p.bias_term();
  CHECK(!p.transpose()) << "transpose is not supported";
  const int axis = bottom[0]->CanonicalAxisIndex(p.axis());
  CHECK_EQ(axis, 1) << "mscnn_b200 InnerProduct supports axis 1 only";
  K_ = bottom[0]->count(axis);
  if (this->blobs_.size() > 0) {
    CHECK_EQ((int)this->blobs_.size(), 1 + (bias_term_ ? 1 : 0));
  } else {
    this->blobs_.resize(bias_term_ ? 2 : 1);
    vector<int> ws(2);
    ws[0] = N_;
    ws[1] = K_;
    this->blobs_[0].reset(new Blob<Dtype>(ws));
    FillBlob(p.weight_filler(), this->blobs_[0].get());
    if (bias_term_) {
      this->blobs_[1].reset(new Blob<Dtype>(vector<int>(1, N_)));
      FillBlob(p.bias_filler(), this->blobs_[1].get());
    }
  }
}
template <typename Dtype>
void InnerProductLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const int new_K = bottom[0]->count(1);
  CHECK_EQ(K_, new_K) << "Input size incompatible with inner product parameters.";
  M_ = bottom[0]->count(0, 1);
  vector<int> ts(2);
  ts[0] = M_;
  ts[1] = N_;
  top[0]->Reshape(ts);  // inner_product_layer.cpp:58-74
}
template <typename Dtype>
void InnerProductLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const bool split = Caffe::split();
  const int C = bottom[0]->LegacyShape(1), H = bottom[0]->LegacyShape(2), W = bottom[0]->LegacyShape(3);
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  const int nout_pad = out_pad(N_);
  packed_.update_weights(this->blobs_[0].get(), {PackedParam::FC, split, nout_pad, x.cpad, C, H, W},
                         (size_t)nout_pad * H * W * x.cpad * 2, [&](const float* w, void* hi, void* lo) {
    MSCNN_CHECK(mscnn_pack_fc_weights(w, hi, lo, N_, C, H, W, nout_pad, x.cpad, Caffe::stream()));
  });
  packed_.bias.update(bias_term_ ? this->blobs_[1].get() : nullptr, N_, nout_pad);
  // the NHWC flattening of the bottom is the channel vector of a 1 x 1 "image"
  mscnn_conv_desc d = conv_desc(x, packed_, M_, 1, 1, H * W * x.cpad, N_, 1, 1, 0, 0, this->dyn_rows_device());
  d.relu = fuse_relu_ ? 1 : 0;
  if (planes_top()) {
    typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
    d.out_mode = MSCNN_OUT_NHWC_BF16;
    d.y_hi = y.hi;
    d.y_lo = y.lo;
  } else {
    d.out_mode = MSCNN_OUT_NCHW_F32;  // cls_pred / bbox_pred: [R][N_] fp32, the Caffe layout
    d.y_f32 = top[0]->mutable_gpu_data();
  }
  MSCNN_CHECK(mscnn_conv_forward(&d, Caffe::stream()));
}
LAYER_ACCESSES(InnerProductLayer) {
  return access_all(out, bottom, PLANES) && access_all(out, top, planes_top() ? PLANES : NCHW);
}

// -------------------------------------------------------------------------------- Dropout
template <typename Dtype>
void DropoutLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK(this->phase_ == TEST) << "mscnn_b200 is forward-only: Dropout runs in the TEST phase";
  if (top[0] != bottom[0]) top[0]->ShareData(*bottom[0]);  // dropout_layer.cpp:43-45 copies; sharing is equivalent
}
LAYER_ACCESSES(DropoutLayer) { return true; }  // the top is on the bottom's storage (TopsShareBottom)

// ------------------------------------------------------------------------------ BoxOutput
template <typename Dtype>
BoxOutputLayer<Dtype>::~BoxOutputLayer() {
  if (workspace_) cudaFree(workspace_);
  if (num_out_dev_) cudaFree(num_out_dev_);
  if (num_out_host_) cudaFreeHost(num_out_host_);
  if (rows_event_) cudaEventDestroy(rows_event_);
}
template <typename Dtype>
void BoxOutputLayer<Dtype>::ResolveRows(const vector<Blob<Dtype>*>& top) {
  if (!dyn_.pending) return;
  CUDA_CHECK(cudaEventSynchronize(rows_event_));
  dyn_.pending = false;
  const int rows = num_out_host_[0];
  top[0]->Reshape(rows, 5, 1, 1);
  if (output_proposal_with_score_) top[1]->Reshape(rows, 6, 1, 1);
}
template <typename Dtype>
void BoxOutputLayer<Dtype>::RearmRows() {
  CUDA_CHECK(cudaEventRecord(rows_event_, Caffe::stream()));
  dyn_.pending = true;
}
template <typename Dtype>
void BoxOutputLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const BoxOutputParameter& p = this->layer_param_.box_output_param();  // box_output_layer.cpp:19-26, 79-104
  const int J = (int)bottom.size();
  CHECK_LE(J, MSCNN_MAX_SCALES);
  CHECK_EQ(J, p.field_h_size());
  CHECK_EQ(J, p.field_w_size());
  CHECK_EQ(J, p.downsample_rate_size());
  memset(&cfg_, 0, sizeof(cfg_));
  cfg_.num_scales = J;
  for (int j = 0; j < J; ++j) {
    cfg_.field_w[j] = (float)p.field_w(j);
    cfg_.field_h[j] = (float)p.field_h(j);
    cfg_.downsample_rate[j] = (float)p.downsample_rate(j);
  }
  cfg_.fg_thr = p.fg_thr();
  cfg_.iou_thr = p.iou_thr();
  cfg_.nms_type = p.nms_type() == "IOMU" ? MSCNN_NMS_IOMU : p.nms_type() == "IOFU" ? MSCNN_NMS_IOFU : MSCNN_NMS_IOU;
  cfg_.field_whr = p.field_whr();
  cfg_.field_xyr = p.field_xyr();
  cfg_.min_size = p.min_size();
  cfg_.max_nms_num = p.max_nms_num();
  cfg_.max_post_nms_num = p.max_post_nms_num();
  CHECK(cfg_.max_nms_num > 0 && cfg_.max_nms_num <= 8192)
      << "mscnn_b200 BoxOutput needs 0 < max_nms_num <= 8192 (the reference's 0 = unbounded is not supported)";
  const BBoxRegParameter& r = this->layer_param_.bbox_reg_param();
  cfg_.do_bbox_norm = (r.bbox_mean_size() > 0 && r.bbox_std_size() > 0) ? 1 : 0;
  if (cfg_.do_bbox_norm) {
    CHECK_EQ(r.bbox_mean_size(), 4);
    CHECK_EQ(r.bbox_std_size(), 4);
    for (int k = 0; k < 4; ++k) { cfg_.bbox_mean[k] = r.bbox_mean(k); cfg_.bbox_std[k] = r.bbox_std(k); }
  }
  output_proposal_with_score_ = (top.size() == 2);
}
template <typename Dtype>
void BoxOutputLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  // "dummy reshape" (box_output_layer.cpp:29-36); the real shape is data dependent.  Rows still pending from the
  // last Forward (Net::ResolveRows re-runs Reshape down the net) keep their cap shape until resolved.
  if (dyn_.pending) return;
  top[0]->Reshape(1, 5, 1, 1);
  if (output_proposal_with_score_) top[1]->Reshape(1, 6, 1, 1);
}
template <typename Dtype>
void BoxOutputLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const int N = bottom[0]->num();
  cfg_.channels = bottom[0]->channels();
  const float* maps[MSCNN_MAX_SCALES];
  for (size_t j = 0; j < bottom.size(); ++j) {
    CHECK_EQ(bottom[j]->channels(), cfg_.channels);
    CHECK_EQ(bottom[j]->num(), N);
    cfg_.height[j] = bottom[j]->height();
    cfg_.width[j] = bottom[j]->width();
    maps[j] = bottom[j]->gpu_data();
  }
  size_t need = 0;
  MSCNN_CHECK(mscnn_box_output_workspace_bytes(&cfg_, N, &need));
  if (need > workspace_bytes_) {
    if (workspace_) CUDA_CHECK(cudaFree(workspace_));
    CUDA_CHECK(cudaMalloc(&workspace_, need));
    workspace_bytes_ = need;
  }
  if (2 + N > num_out_cap_) {
    if (num_out_dev_) CUDA_CHECK(cudaFree(num_out_dev_));
    if (num_out_host_) CUDA_CHECK(cudaFreeHost(num_out_host_));
    CUDA_CHECK(cudaMalloc(&num_out_dev_, sizeof(int) * (2 + N)));
    CUDA_CHECK(cudaMallocHost(&num_out_host_, sizeof(int) * (2 + N)));
    num_out_cap_ = 2 + N;
    dyn_.device_rows = num_out_dev_;  // [0] = rows in the top blobs (>= 1)
  }
  if (!rows_event_) CUDA_CHECK(cudaEventCreateWithFlags(&rows_event_, cudaEventDisableTiming));
  dyn_.pending = false;  // a new Forward supersedes counts nobody asked for
  // Size the tops for the cap, let the kernels write in place, then shrink to the true row
  // count (Blob::Reshape never reallocates when shrinking, blob.cpp:40-44).
  ReshapeAsForward(bottom, top);
  Dtype* rois = top[0]->mutable_gpu_data();
  Dtype* rois_score = output_proposal_with_score_ ? top[1]->mutable_gpu_data() : nullptr;
  MSCNN_CHECK(mscnn_box_output_forward(&cfg_, N, maps, workspace_, workspace_bytes_, rois, rois_score,
                                       num_out_dev_, Caffe::stream()));
  CUDA_CHECK(cudaMemcpyAsync(num_out_host_, num_out_dev_, sizeof(int) * (2 + N), cudaMemcpyDeviceToHost,
                             Caffe::stream()));
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(Caffe::stream(), &capturing);
  if (capturing == cudaStreamCaptureStatusNone)  // under capture the Net re-arms after the graph launch (RearmRows)
    CUDA_CHECK(cudaEventRecord(rows_event_, Caffe::stream()));
  dyn_.pending = true;  // tops have `cap` rows; the true count is in num_out_dev_[0] (and soon in num_out_host_[0])
  if (!defer_rows_) ResolveRows(top);
}
LAYER_ACCESSES(BoxOutputLayer) { return access_all(out, bottom, NCHW) && access_all(out, top, NCHW); }

// ----------------------------------------------------------------------------- ROIPooling
template <typename Dtype>
void ROIPoolingLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const ROIPoolingParameter& p = this->layer_param_.roi_pooling_param();  // roi_pooling_layer.cpp:22-34
  CHECK_GT(p.pooled_h(), 0u) << "pooled_h must be > 0";
  CHECK_GT(p.pooled_w(), 0u) << "pooled_w must be > 0";
  pooled_height_ = p.pooled_h();
  pooled_width_ = p.pooled_w();
  spatial_scale_ = p.spatial_scale();
  pad_ratios_.assign(1, p.pad_ratio());
  channel_offsets_.assign(1, 0);
}
template <typename Dtype>
void ROIPoolingLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  channels_ = bottom[0]->channels();
  height_ = bottom[0]->height();
  width_ = bottom[0]->width();
  top[0]->Reshape(bottom[1]->num(), channels_, pooled_height_, pooled_width_);
}
template <typename Dtype>
void ROIPoolingLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  if (fused_) return;  // the group's leader pools this layer's variant in its launch
  const bool split = Caffe::split();
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  const int R = bottom[1]->num();
  const Dtype* rois = bottom[1]->gpu_data();
  Blob<Dtype>* out = output(top);
  if (concat_top_) out->Reshape(R, concat_channels_, pooled_height_, pooled_width_);  // the fused Concat's top
  typename Blob<Dtype>::Planes y = out->mutable_planes(split);
  MSCNN_CHECK(mscnn_roi_pool_multi_forward_dyn(x.hi, x.lo, x.n, x.h, x.w, x.cpad, rois, R, pooled_height_, pooled_width_,
                                               spatial_scale_, (int)pad_ratios_.size(), pad_ratios_.data(),
                                               channel_offsets_.data(), y.hi, y.lo, y.cpad, this->dyn_rows_device(),
                                               Caffe::stream()));
}
LAYER_ACCESSES(ROIPoolingLayer) {
  if (fused_) return true;  // pooled in its leader's launch
  out->push_back(make_pair(bottom[0], PLANES));
  out->push_back(make_pair(bottom[1], NCHW));
  out->push_back(make_pair(output(top), PLANES));
  return true;
}

// ------------------------------------------------------------------------------- ROIAlign
template <typename Dtype>
void ROIAlignLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const ROIPoolingParameter& p = this->layer_param_.roi_pooling_param();  // roi_align_layer.cpp:22-37
  CHECK_GT(p.pooled_h(), 0u) << "pooled_h must be > 0";
  CHECK_GT(p.pooled_w(), 0u) << "pooled_w must be > 0";
  pooled_height_ = p.pooled_h();
  pooled_width_ = p.pooled_w();
  grid_height_ = pooled_height_ + 1;
  grid_width_ = pooled_width_ + 1;
  spatial_scale_ = p.spatial_scale();
  pad_ratio_ = p.pad_ratio();
}
template <typename Dtype>
void ROIAlignLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  channels_ = bottom[0]->channels();
  height_ = bottom[0]->height();
  width_ = bottom[0]->width();
  top[0]->Reshape(bottom[1]->num(), channels_, grid_height_, grid_width_);
}
template <typename Dtype>
void ROIAlignLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const bool split = Caffe::split();
  typename Blob<Dtype>::Planes x = bottom[0]->planes(split);
  typename Blob<Dtype>::Planes y = top[0]->mutable_planes(split);
  MSCNN_CHECK(mscnn_roi_align_forward_dyn(x.hi, x.lo, x.n, x.h, x.w, x.cpad, bottom[1]->gpu_data(), bottom[1]->num(),
                                          pooled_height_, pooled_width_, spatial_scale_, pad_ratio_, y.hi, y.lo,
                                          y.cpad, 0, this->dyn_rows_device(), Caffe::stream()));
}
LAYER_ACCESSES(ROIAlignLayer) {
  out->push_back(make_pair(bottom[0], PLANES));
  out->push_back(make_pair(bottom[1], NCHW));
  return access_all(out, top, PLANES);
}

// ----------------------------------------------------------------------------- DecodeBBox
template <typename Dtype>
void DecodeBBoxLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const BBoxRegParameter& r = this->layer_param_.bbox_reg_param();  // decode_bbox_layer.cpp:20-36
  if (r.bbox_mean_size() > 0 && r.bbox_std_size() > 0) {
    CHECK_EQ(r.bbox_mean_size(), 4);
    CHECK_EQ(r.bbox_std_size(), 4);
    for (int i = 0; i < 4; ++i) {
      bbox_mean_[i] = r.bbox_mean(i);
      bbox_std_[i] = r.bbox_std(i);
      CHECK_GT(bbox_std_[i], 0);
    }
  } else {
    for (int i = 0; i < 4; ++i) { bbox_mean_[i] = 0.f; bbox_std_[i] = 1.f; }
  }
}
template <typename Dtype>
void DecodeBBoxLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK_EQ(bottom[0]->num(), bottom[1]->num());  // decode_bbox_layer.cpp:42-50
  CHECK(bottom.size() < 3) << "mscnn_b200 is forward-only: DecodeBBox takes gt boxes only in the TRAIN phase";
  CHECK_EQ(bottom[0]->channels(), 8);
  CHECK_EQ(bottom[1]->channels(), 5);
  top[0]->ReshapeLike(*bottom[1]);
}
template <typename Dtype>
void DecodeBBoxLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  CHECK(this->phase_ == TEST) << "mscnn_b200 is forward-only: DecodeBBox runs in the TEST phase";
  const int num = bottom[0]->num();
  // TEST phase keeps every row (decode_bbox_layer.cpp:79-110), so the top has the priors' shape
  top[0]->Reshape(num, bottom[1]->channels(), 1, 1);
  MSCNN_CHECK(mscnn_decode_bbox_forward(bottom[0]->gpu_data(), bottom[1]->gpu_data(), num, bottom[0]->channels(),
                                        bbox_mean_, bbox_std_, top[0]->mutable_gpu_data(), Caffe::stream()));
}
LAYER_ACCESSES(DecodeBBoxLayer) { return access_all(out, bottom, NCHW) && access_all(out, top, NCHW); }

// -------------------------------------------------------------------------------- Softmax
template <typename Dtype>
void SoftmaxLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  softmax_axis_ = bottom[0]->CanonicalAxisIndex(this->layer_param_.softmax_param().axis());  // softmax_layer.cpp:10-25
  top[0]->ReshapeLike(*bottom[0]);
  outer_num_ = bottom[0]->count(0, softmax_axis_);
  inner_num_ = bottom[0]->count(softmax_axis_ + 1);
}
template <typename Dtype>
void SoftmaxLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  MSCNN_CHECK(mscnn_softmax_forward(bottom[0]->gpu_data(), outer_num_, bottom[0]->shape(softmax_axis_), inner_num_,
                                    top[0]->mutable_gpu_data(), Caffe::stream()));
}
LAYER_ACCESSES(SoftmaxLayer) { return access_all(out, bottom, NCHW) && access_all(out, top, NCHW); }

// -------------------------------------------------------------------------------- Eltwise
template <typename Dtype>
void EltwiseLayer<Dtype>::LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const EltwiseParameter& p = this->layer_param_.eltwise_param();  // eltwise_layer.cpp:10-28
  CHECK(p.coeff_size() == 0 || p.coeff_size() == (int)bottom.size())
      << "Eltwise Layer takes one coefficient per bottom blob.";
  CHECK(!(p.operation() == EltwiseParameter_EltwiseOp_PROD && p.coeff_size()))
      << "Eltwise layer only takes coefficients for summation.";
  CHECK_LE((int)bottom.size(), MSCNN_MAX_ELTWISE);
  op_ = p.operation() == EltwiseParameter_EltwiseOp_PROD ? MSCNN_ELTWISE_PROD
        : p.operation() == EltwiseParameter_EltwiseOp_MAX ? MSCNN_ELTWISE_MAX
                                                          : MSCNN_ELTWISE_SUM;
  coeffs_.assign(bottom.size(), 1.f);
  for (int i = 0; i < p.coeff_size(); ++i) coeffs_[i] = p.coeff(i);
}
template <typename Dtype>
void EltwiseLayer<Dtype>::Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  for (size_t i = 1; i < bottom.size(); ++i) CHECK(bottom[i]->shape() == bottom[0]->shape());
  top[0]->ReshapeLike(*bottom[0]);
}
template <typename Dtype>
void EltwiseLayer<Dtype>::Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
  const float* in[MSCNN_MAX_ELTWISE];
  for (size_t i = 0; i < bottom.size(); ++i) in[i] = bottom[i]->gpu_data();
  MSCNN_CHECK(mscnn_eltwise_forward(in, (int)bottom.size(), op_, coeffs_.data(), (size_t)top[0]->count(),
                                    top[0]->mutable_gpu_data(), Caffe::stream()));
}
LAYER_ACCESSES(EltwiseLayer) { return access_all(out, bottom, NCHW) && access_all(out, top, NCHW); }

INSTANTIATE_CLASS(InputLayer);
INSTANTIATE_CLASS(ConvolutionLayer);
INSTANTIATE_CLASS(DeconvolutionLayer);
INSTANTIATE_CLASS(ReLULayer);
INSTANTIATE_CLASS(PoolingLayer);
INSTANTIATE_CLASS(SplitLayer);
INSTANTIATE_CLASS(ConcatLayer);
INSTANTIATE_CLASS(InnerProductLayer);
INSTANTIATE_CLASS(DropoutLayer);
INSTANTIATE_CLASS(BoxOutputLayer);
INSTANTIATE_CLASS(ROIPoolingLayer);
INSTANTIATE_CLASS(ROIAlignLayer);
INSTANTIATE_CLASS(DecodeBBoxLayer);
INSTANTIATE_CLASS(SoftmaxLayer);
INSTANTIATE_CLASS(EltwiseLayer);
REGISTER_LAYER_CLASS(Input);
REGISTER_LAYER_CLASS(Convolution);
REGISTER_LAYER_CLASS(Deconvolution);
REGISTER_LAYER_CLASS(ReLU);
REGISTER_LAYER_CLASS(Pooling);
REGISTER_LAYER_CLASS(Split);
REGISTER_LAYER_CLASS(Concat);
REGISTER_LAYER_CLASS(InnerProduct);
REGISTER_LAYER_CLASS(Dropout);
REGISTER_LAYER_CLASS(BoxOutput);
REGISTER_LAYER_CLASS(ROIPooling);
REGISTER_LAYER_CLASS(ROIAlign);
REGISTER_LAYER_CLASS(DecodeBBox);
REGISTER_LAYER_CLASS(Softmax);
REGISTER_LAYER_CLASS(Eltwise);

}  // namespace caffe
