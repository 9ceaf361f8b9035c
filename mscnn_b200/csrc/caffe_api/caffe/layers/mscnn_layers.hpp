// The layer types the MS-CNN and cascade deploy nets instantiate (census: SURVEY.md section 2 and 8(f)), as
// caffe::Layer<Dtype> subclasses whose Forward_gpu calls the C ABI in include/mscnn_b200.h.
// Class names, type() strings, blob layouts and parameter semantics are the reference's
// (/root/reference/include/caffe/layers/*.hpp); the per-layer headers next to this file
// (conv_layer.hpp, ...) only include this one so that existing #include lines keep working.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "caffe/blob.hpp"
#include "caffe/layer.hpp"
#include "caffe/proto/caffe.pb.h"

namespace caffe {

// Fill a parameter blob according to a FillerParameter (include/caffe/filler.hpp).  Supported:
// constant, gaussian, bilinear (the only ones the MS-CNN prototxts name); anything else aborts.
CAFFE_API void FillBlob(const FillerParameter& filler, Blob<float>* blob);

// Device copies of the packed weights (planes) and zero-padded biases owned by Convolution / InnerProduct layers,
// brought up to date in the first forward after a change: a forward with unchanged parameters, precision and shapes
// allocates and copies nothing, so it can be captured into a CUDA graph.
struct PackedBias {
  float* data = nullptr;
  int len = 0;  // padded length
  const Blob<float>* src = nullptr;
  unsigned long version = ~0ul;
  ~PackedBias();
  void update(Blob<float>* b, int n, int n_pad);  // b[0:n], then zeros up to n_pad (b == NULL: all zeros)
};
struct PackedParam {
  enum Route { CONV, HEAD, CONV1_1, FC, DECONV };
  // how the image was packed: the route, the precision (split), its padding, (fc) the bottom's C, H, W and (deconv)
  // the stride, pad and dilation per axis.  With the blob's storage it names one image (Blob::packed_image).
  struct Layout { int route, split, out_pad, in_pad, c, h, w, geom[6]; };
  shared_ptr<PackedImage> img;  // the image the kernels read; it lives with the weight blob's storage
  Layout layout = {-1};
  unsigned long w_version = ~0ul;  // the storage version img held when this layer last made its stream wait for it
  PackedBias bias, gather_bias;  // [layout.out_pad] for the kernel; k x k heads: [Cout] for the tap gather
  // Makes img the image of wb's storage under l, current for wb's version: packs it with pack(w_f32, hi, lo) on this
  // thread's stream when stale (lo = NULL unless l.split), else orders this stream after its last pack.
  template <typename Pack> void update_weights(Blob<float>* wb, const Layout& l, size_t bytes, Pack pack);
  void* hi() const { return img->w.hi; }
  void* lo() const { return layout.split ? img->w.lo : nullptr; }
};

/// InputLayer: /root/reference/src/caffe/layers/input_layer.cpp:8-22
template <typename Dtype>
class CAFFE_API InputLayer : public Layer<Dtype> {
 public:
  explicit InputLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
  virtual inline const char* type() const { return "Input"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 0; }
  virtual inline int MinTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
};

// A Pooling folded into its convolution (Net::FusePooling) is computed in the convolution's epilogue exactly when the
// convolution's output has even height and width; at odd extents the convolution stores its full output and the
// Pooling runs itself.  Both layers decide with this, from the shape of the forward they run in.
template <typename Dtype>
inline bool epilogue_pools(const Blob<Dtype>& conv_top) {
  return conv_top.height() % 2 == 0 && conv_top.width() % 2 == 0;
}

/// ConvolutionLayer: conv_layer.cpp:8-40 / base_conv_layer.cpp:15-254, 2-D, with stride, dilation and groups whose
/// Cin / group and Cout / group are multiples of 64.  blobs_[0] = [Cout, Cin / group, kh, kw], blobs_[1] = [Cout].
template <typename Dtype>
class CAFFE_API ConvolutionLayer : public Layer<Dtype> {
 public:
  explicit ConvolutionLayer(const LayerParameter& param) : Layer<Dtype>(param), fuse_relu_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Convolution"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
  // mscnn_b200 extension: fold the in-place ReLU that follows into the epilogue (set by Net).
  void set_fuse_relu(bool f) { fuse_relu_ = f; }
  bool fuse_relu() const { return fuse_relu_; }
  // mscnn_b200 extension (set by Net): the folded 2x2/2 MAX Pooling that follows is computed in this layer's epilogue
  // and written to `pool_top` whenever epilogue_pools(top); then, unless store_full, nothing else reads this layer's
  // own top, which is not written (its blob holds no data).
  void set_fused_pool(Blob<Dtype>* pool_top, bool store_full) { fused_pool_top_ = pool_top; store_full_ = store_full; }
  // the route whose epilogue can pool: 64-channel-aligned output, not conv1_1's kernel
  bool can_fuse_pool() const { return num_output_ % 64 == 0 && !is_conv1_1(); }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  // the top is planes above 32 outputs, NCHW fp32 for the narrow heads
  bool planes_top() const { return num_output_ > 32; }
  bool pools_here(const Blob<Dtype>& top) const { return fused_pool_top_ && epilogue_pools(top); }
  // stride 1, dilation 1, one group: what conv1_1's kernel and the k x 1 head-tap route compute
  bool plain_geometry() const {
    return stride_h_ == 1 && stride_w_ == 1 && dilation_h_ == 1 && dilation_w_ == 1 && group_ == 1;
  }
  bool is_conv1_1() const {
    return channels_ == 3 && kernel_h_ == 3 && kernel_w_ == 3 && pad_h_ == 1 && pad_w_ == 1 && num_output_ == 64 &&
           plain_geometry();
  }
  Blob<Dtype>* fused_pool_top_ = nullptr;
  bool store_full_ = true;
  int num_output_, channels_, kernel_h_, kernel_w_, pad_h_, pad_w_;
  int stride_h_, stride_w_, dilation_h_, dilation_w_, group_;
  bool bias_term_, fuse_relu_;
  PackedParam packed_;
};

/// DeconvolutionLayer: deconv_layer.cpp:8-40 / base_conv_layer.cpp:15-254, 2-D, with stride, pad, dilation, groups and
/// bias.  blobs_[0] = [Cin, Cout / group, kh, kw], blobs_[1] = [Cout].  Depthwise layers (group == Cin == Cout) run
/// mscnn_deconv_depthwise_forward on the blob as it is; the others mscnn_deconv_forward on weights packed by phase,
/// which needs Cin / group and Cout / group to be multiples of 64 when group > 1.
template <typename Dtype>
class CAFFE_API DeconvolutionLayer : public Layer<Dtype> {
 public:
  explicit DeconvolutionLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Deconvolution"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  bool depthwise() const { return group_ == channels_ && num_output_ == channels_; }
  int num_output_, channels_, kernel_h_, kernel_w_, pad_h_, pad_w_;
  int stride_h_, stride_w_, dilation_h_, dilation_w_, group_;
  bool bias_term_;
  PackedParam packed_;
};

/// ReLULayer: relu_layer.cpp:9-19 (negative_slope 0), in place.
template <typename Dtype>
class CAFFE_API ReLULayer : public Layer<Dtype> {
 public:
  explicit ReLULayer(const LayerParameter& param) : Layer<Dtype>(param), fused_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    top[0]->ReshapeLike(*bottom[0]);
  }
  virtual inline const char* type() const { return "ReLU"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
  void set_fused(bool f) { fused_ = f; }   // producer already applied it
  bool fused() const { return fused_; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  bool fused_;
};

/// PoolingLayer: pooling_layer.cpp:16-220 (MAX / AVE; padding, rectangular kernel / stride, global_pooling).
template <typename Dtype>
class CAFFE_API PoolingLayer : public Layer<Dtype> {
 public:
  explicit PoolingLayer(const LayerParameter& param) : Layer<Dtype>(param), fused_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Pooling"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int MinTopBlobs() const { return 1; }
  virtual inline int MaxTopBlobs() const { return 1; }
  // the one geometry a convolution's epilogue computes: MAX over 2x2 windows, stride 2, no padding
  bool is_max_2x2_s2() const {
    return mode_ == MSCNN_POOL_MAX && !global_pooling_ && kernel_h_ == 2 && kernel_w_ == 2 && stride_h_ == 2 &&
           stride_w_ == 2 && pad_h_ == 0 && pad_w_ == 0;
  }
  void set_fused(bool f) { fused_ = f; }   // folded into the producing convolution: see epilogue_pools
  bool fused() const { return fused_; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  bool pooled_by_conv(const Blob<Dtype>& bottom) const { return fused_ && epilogue_pools(bottom); }
  int kernel_h_, kernel_w_, stride_h_, stride_w_, pad_h_, pad_w_, mode_, pooled_h_, pooled_w_;
  bool global_pooling_, fused_;
};

/// SplitLayer: split_layer.cpp:9-31 (forward = share data).
template <typename Dtype>
class CAFFE_API SplitLayer : public Layer<Dtype> {
 public:
  explicit SplitLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Split"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual bool TopsShareBottom(const vector<Blob<Dtype>*>& bottom) const { return true; }
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int MinTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
};

/// ConcatLayer: concat_layer.cpp:11-74, channel axis.
template <typename Dtype>
class CAFFE_API ConcatLayer : public Layer<Dtype> {
 public:
  explicit ConcatLayer(const LayerParameter& param) : Layer<Dtype>(param), fused_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Concat"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual bool TopsShareBottom(const vector<Blob<Dtype>*>& bottom) const { return bottom.size() == 1; }
  virtual inline int MinBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
  void set_fused(bool f) { fused_ = f; }   // the producers write straight into top[0]
  bool fused() const { return fused_; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  static bool aligned(const vector<Blob<Dtype>*>& bottom) {  // every bottom 64-channel aligned: planes, else NCHW fp32
    return std::all_of(bottom.begin(), bottom.end(), [](const Blob<Dtype>* b) { return b->channels() % 64 == 0; });
  }
  bool fused_;
};

/// InnerProductLayer: inner_product_layer.cpp:10-97 (axis 1, no transpose).
/// blobs_[0] = [N_out, K] with K in the bottom's NCHW flattening, blobs_[1] = [N_out].
template <typename Dtype>
class CAFFE_API InnerProductLayer : public Layer<Dtype> {
 public:
  explicit InnerProductLayer(const LayerParameter& param) : Layer<Dtype>(param), fuse_relu_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "InnerProduct"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
  void set_fuse_relu(bool f) { fuse_relu_ = f; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  bool planes_top() const { return N_ > 32; }  // else [M][N] fp32, the Caffe layout
  int M_, K_, N_;
  bool bias_term_, fuse_relu_;
  PackedParam packed_;
};

/// DropoutLayer: dropout_layer.cpp:31-46 -- TEST phase is the identity.
template <typename Dtype>
class CAFFE_API DropoutLayer : public Layer<Dtype> {
 public:
  explicit DropoutLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    if (top[0] != bottom[0]) top[0]->ReshapeLike(*bottom[0]);
  }
  virtual inline const char* type() const { return "Dropout"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual bool TopsShareBottom(const vector<Blob<Dtype>*>& bottom) const { return true; }
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
};

/// BoxOutputLayer: box_output_layer.cpp:19-234.  top[0] = [R,5,1,1] ROIs, top[1] = [R,6,1,1] with score.
/// Unlike the reference (CPU only) this runs on the device; one small D2H copy of the row count
/// is needed because the Caffe API exposes R as the blobs' shape.
template <typename Dtype>
class CAFFE_API BoxOutputLayer : public Layer<Dtype> {
 public:
  explicit BoxOutputLayer(const LayerParameter& param)
      : Layer<Dtype>(param), workspace_(nullptr), workspace_bytes_(0), num_out_dev_(nullptr),
        num_out_host_(nullptr), num_out_cap_(0) {}
  virtual ~BoxOutputLayer();
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "BoxOutput"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int MinBottomBlobs() const { return 1; }
  virtual inline int MinTopBlobs() const { return 1; }
  virtual inline int MaxTopBlobs() const { return 2; }
  // mscnn_b200 extensions: results of the last Forward
  const int* num_out_device() const { return num_out_dev_; }   // int[2+N], see mscnn_box_output_forward
  int num_proposals() const { return num_out_host_ ? num_out_host_[1] : 0; }
  int image_proposals(int n) const { return num_out_host_[2 + n]; }
  // upper bound of the proposals one image can contribute (box_output_layer.cpp:176-186)
  int max_rows_per_image() const {
    return (cfg_.max_post_nms_num > 0 && cfg_.max_post_nms_num < cfg_.max_nms_num) ? cfg_.max_post_nms_num : cfg_.max_nms_num;
  }
  // Deferred rows (set by Net): Forward leaves the tops at cap rows and does NOT wait for the device; ResolveRows
  // waits for the 12-byte copy of the counts and trims the tops.  Without it (a layer driven directly) Forward
  // synchronises and trims itself, which is the reference's observable behaviour (box_output_layer.cpp:201).
  void set_defer_rows(bool on) { defer_rows_ = on; }
  const DynRows* dyn_rows() const { return &dyn_; }
  bool rows_pending() const { return dyn_.pending; }
  void ResolveRows(const vector<Blob<Dtype>*>& top);
  // after a CUDA-graph replay of this layer's launches (Net::GraphForward): the counts are pending again
  void RearmRows();
  // the tops at cap rows (N x max_nms_num), as Forward sizes them before the count is known
  virtual void ReshapeAsForward(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    const int cap = bottom[0]->num() * cfg_.max_nms_num;
    top[0]->Reshape(cap, 5, 1, 1);
    if (output_proposal_with_score_) top[1]->Reshape(cap, 6, 1, 1);
  }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  mscnn_box_output_cfg cfg_;
  bool output_proposal_with_score_;
  void* workspace_;
  size_t workspace_bytes_;
  int* num_out_dev_;
  int* num_out_host_;
  int num_out_cap_;
  bool defer_rows_ = false;
  DynRows dyn_ = {nullptr, false};
  cudaEvent_t rows_event_ = nullptr;
};

/// ROIPoolingLayer: roi_pooling_layer.cpp:22-139 with the MS-CNN pad_ratio extension.
template <typename Dtype>
class CAFFE_API ROIPoolingLayer : public Layer<Dtype> {
 public:
  explicit ROIPoolingLayer(const LayerParameter& param)
      : Layer<Dtype>(param), concat_top_(nullptr), concat_channels_(0), fused_(false) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "ROIPooling"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int MinBottomBlobs() const { return 2; }
  virtual inline int MaxBottomBlobs() const { return 2; }
  virtual inline int MinTopBlobs() const { return 1; }
  virtual inline int MaxTopBlobs() const { return 1; }
  // mscnn_b200 extensions (set by Net when it folds a Concat into its ROIPooling producers): write into `target` (the
  // Concat top) at a channel offset instead of into top[0]; and, for the group's leader, also pool `follower`'s variant
  // (its pad ratio, at its channel offset) in this layer's launch, after which the follower does nothing.
  void set_concat_target(Blob<Dtype>* target, int channel_offset, int total_channels) {
    concat_top_ = target; channel_offsets_[0] = channel_offset; concat_channels_ = total_channels;
  }
  void add_follower(ROIPoolingLayer<Dtype>* follower) {
    pad_ratios_.push_back(follower->pad_ratios_[0]);
    channel_offsets_.push_back(follower->channel_offsets_[0]);
    follower->fused_ = true;
  }
  bool fused() const { return fused_; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  Blob<Dtype>* output(const vector<Blob<Dtype>*>& top) const { return concat_top_ ? concat_top_ : top[0]; }
  int channels_, height_, width_, pooled_height_, pooled_width_;
  float spatial_scale_;
  vector<float> pad_ratios_;     // one variant per entry, pooled in one launch: this layer's own, then its followers'
  vector<int> channel_offsets_;  // where each variant starts in the output's channels
  Blob<Dtype>* concat_top_;
  int concat_channels_;
  bool fused_;                   // the group's leader pools this layer's variant
};

/// ROIAlignLayer: roi_align_layer.cpp:22-139 (cascade WIDER-face net).  top = [R, C, pooled_h+1, pooled_w+1].
template <typename Dtype>
class CAFFE_API ROIAlignLayer : public Layer<Dtype> {
 public:
  explicit ROIAlignLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "ROIAlign"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int MinBottomBlobs() const { return 2; }
  virtual inline int MaxBottomBlobs() const { return 2; }
  virtual inline int MinTopBlobs() const { return 1; }
  virtual inline int MaxTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  int channels_, height_, width_, pooled_height_, pooled_width_, grid_height_, grid_width_;
  float spatial_scale_, pad_ratio_;
};

/// DecodeBBoxLayer: decode_bbox_layer.cpp:17-124, TEST phase (2 bottoms: bbox_pred [R,8], prior ROIs [R,5]).
/// CPU-only in the reference; here it stays on the device, so the cascade stages do not sync with the host.
template <typename Dtype>
class CAFFE_API DecodeBBoxLayer : public Layer<Dtype> {
 public:
  explicit DecodeBBoxLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "DecodeBBox"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int MinBottomBlobs() const { return 2; }
  virtual inline int MaxBottomBlobs() const { return 3; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  float bbox_mean_[4], bbox_std_[4];
};

/// SoftmaxLayer: softmax_layer.cpp:10-62.
template <typename Dtype>
class CAFFE_API SoftmaxLayer : public Layer<Dtype> {
 public:
  explicit SoftmaxLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Softmax"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int ExactNumBottomBlobs() const { return 1; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  int outer_num_, inner_num_, softmax_axis_;
};

/// EltwiseLayer: eltwise_layer.cpp:10-96 (PROD / SUM with coefficients / MAX).
template <typename Dtype>
class CAFFE_API EltwiseLayer : public Layer<Dtype> {
 public:
  explicit EltwiseLayer(const LayerParameter& param) : Layer<Dtype>(param) {}
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  virtual inline const char* type() const { return "Eltwise"; }
  virtual bool Accesses(const vector<Blob<Dtype>*>&, const vector<Blob<Dtype>*>&, BlobAccesses<Dtype>*) const;
  virtual inline int MinBottomBlobs() const { return 2; }
  virtual inline int ExactNumTopBlobs() const { return 1; }
 protected:
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top);
  int op_;
  vector<float> coeffs_;
};

}  // namespace caffe
