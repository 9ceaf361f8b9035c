// caffe::Layer<Dtype> -- the operator ABI of the reference, restated for the forward path
// (/root/reference/include/caffe/layer.hpp:33-487).  SetUp = CheckBlobCounts -> LayerSetUp ->
// Reshape (:67-74); Forward = Reshape (every call) -> Forward_{cpu,gpu} by Caffe::mode()
// (:451-487).  Backward is declared for source compatibility and is NOT_IMPLEMENTED.
//
// mscnn_b200 rule: Forward_cpu of every layer aborts -- there is no CPU fallback.  (The
// reference does the opposite for BoxOutput: its Forward_gpu falls back to Forward_cpu,
// layer.hpp:341-345.)
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/layer_factory.hpp"
#include "caffe/proto/caffe.pb.h"

namespace caffe {

// mscnn_b200 extension: data-dependent row counts that stay on the device.  BoxOutput's number of proposals R is only
// known after its kernels have run; the reference learns it on the host (its BoxOutput IS host code,
// box_output_layer.cpp:201) and shapes every later blob with it.  Here a Net sizes those blobs for the cap
// (N x max_nms_num rows), every layer behind BoxOutput reads R from device memory (`device_rows`: rows to process,
// >= 1) and skips the rest, and the blob shapes are trimmed to R when the host next needs them (Net::ResolveRows).
// `pending` = the blobs currently have cap rows and device_rows is authoritative.
struct DynRows {
  const int* device_rows;
  bool pending;
};

// mscnn_b200 extension: how a forward touches a blob (Net's activation plan).  PLANES: bf16 hi (+ lo in fp32-faithful
// precision) planes; NCHW: fp32 in the Caffe layout; TOUCH: in place, on whichever representation is current.
enum Access { TOUCH, PLANES, NCHW };
template <typename Dtype> using BlobAccesses = vector<pair<const Blob<Dtype>*, Access> >;

template <typename Dtype>
class CAFFE_API Layer {
 public:
  explicit Layer(const LayerParameter& param) : layer_param_(param) {
    phase_ = param.phase();
    if (layer_param_.blobs_size() > 0) {
      blobs_.resize(layer_param_.blobs_size());
      for (int i = 0; i < layer_param_.blobs_size(); ++i) {
        blobs_[i].reset(new Blob<Dtype>());
        blobs_[i]->FromProto(layer_param_.blobs(i));
      }
    }
  }
  virtual ~Layer() {}

  void SetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    CheckBlobCounts(bottom, top);
    LayerSetUp(bottom, top);
    Reshape(bottom, top);
  }
  virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
  virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;

  inline Dtype Forward(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    Reshape(bottom, top);
    switch (Caffe::mode()) {
      case Caffe::CPU:
        Forward_cpu(bottom, top);
        break;
      case Caffe::GPU:
        Forward_gpu(bottom, top);
        break;
      default:
        LOG(FATAL) << "Unknown caffe mode.";
    }
    return Dtype(0);
  }
  inline void Backward(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down,
                       const vector<Blob<Dtype>*>& bottom) {
    NOT_IMPLEMENTED << " (mscnn_b200 is forward-only)";
  }

  vector<shared_ptr<Blob<Dtype> > >& blobs() { return blobs_; }
  const LayerParameter& layer_param() const { return layer_param_; }
  // mscnn_b200 extension (set by Net for the layers behind a BoxOutput layer): see DynRows
  void set_dyn_rows(const DynRows* d) { dyn_rows_ = d; }
  const int* dyn_rows_device() const { return (dyn_rows_ && dyn_rows_->pending) ? dyn_rows_->device_rows : nullptr; }
  // mscnn_b200 extension: appends each blob a forward on blobs of these shapes reads or writes, with its representation;
  // work a fused layer does for another is stated where it runs.  false: no statement (the net cannot be planned).
  virtual bool Accesses(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top,
                        BlobAccesses<Dtype>* out) const { return false; }
  // mscnn_b200 extension: a forward leaves every top on bottom[0]'s bytes (ShareData): one storage for the net
  virtual bool TopsShareBottom(const vector<Blob<Dtype>*>& bottom) const { return false; }
  // mscnn_b200 extension: shapes top as a forward on bottom writes it, before the host learns any data-dependent row
  // count (Net's activation plan): Reshape's shapes, unless Forward_gpu sizes its tops itself
  virtual void ReshapeAsForward(const vector<Blob<Dtype>*>& b, const vector<Blob<Dtype>*>& t) { Reshape(b, t); }
  virtual inline const char* type() const { return ""; }
  virtual inline int ExactNumBottomBlobs() const { return -1; }
  virtual inline int MinBottomBlobs() const { return -1; }
  virtual inline int MaxBottomBlobs() const { return -1; }
  virtual inline int ExactNumTopBlobs() const { return -1; }
  virtual inline int MinTopBlobs() const { return -1; }
  virtual inline int MaxTopBlobs() const { return -1; }
  virtual inline bool EqualNumBottomTopBlobs() const { return false; }

 protected:
  LayerParameter layer_param_;
  Phase phase_;
  vector<shared_ptr<Blob<Dtype> > > blobs_;
  const DynRows* dyn_rows_ = nullptr;

  virtual void Forward_cpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    LOG(FATAL) << "mscnn_b200: layer " << layer_param_.name() << " (" << type()
               << ") has no CPU implementation; set Caffe::set_mode(Caffe::GPU).";
  }
  virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;

  virtual void CheckBlobCounts(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
    if (ExactNumBottomBlobs() >= 0)
      CHECK_EQ(ExactNumBottomBlobs(), (int)bottom.size())
          << type() << " Layer takes " << ExactNumBottomBlobs() << " bottom blob(s) as input.";
    if (MinBottomBlobs() >= 0)
      CHECK_LE(MinBottomBlobs(), (int)bottom.size())
          << type() << " Layer takes at least " << MinBottomBlobs() << " bottom blob(s) as input.";
    if (MaxBottomBlobs() >= 0)
      CHECK_GE(MaxBottomBlobs(), (int)bottom.size())
          << type() << " Layer takes at most " << MaxBottomBlobs() << " bottom blob(s) as input.";
    if (ExactNumTopBlobs() >= 0)
      CHECK_EQ(ExactNumTopBlobs(), (int)top.size())
          << type() << " Layer produces " << ExactNumTopBlobs() << " top blob(s) as output.";
    if (MinTopBlobs() >= 0)
      CHECK_LE(MinTopBlobs(), (int)top.size())
          << type() << " Layer produces at least " << MinTopBlobs() << " top blob(s) as output.";
    if (MaxTopBlobs() >= 0)
      CHECK_GE(MaxTopBlobs(), (int)top.size())
          << type() << " Layer produces at most " << MaxTopBlobs() << " top blob(s) as output.";
    if (EqualNumBottomTopBlobs())
      CHECK_EQ(bottom.size(), top.size())
          << type() << " Layer produces one top blob as output for each bottom blob input.";
  }

 private:
  DISABLE_COPY_AND_ASSIGN(Layer);
};

}  // namespace caffe
