// caffe::Blob<Dtype> -- source-compatible subset of /root/reference/include/caffe/blob.hpp:24-277
// (forward path: no diff storage), plus the mscnn_b200 extension that lets the hot path keep a
// tensor as NHWC bf16 "planes" on the device without ever materialising the NCHW fp32 array.
//
// A blob has up to two device representations of the same logical N x C x H x W tensor:
//   * the Caffe one: NCHW fp32 in a SyncedMemory (cpu_data()/gpu_data());
//   * planes: NHWC bf16, channels padded to 64, hi (+ lo in fp32-faithful mode).
// `layout_head_` says which one is current.  cpu_data()/gpu_data() convert from planes on
// demand (mscnn_planes_to_nchw_f32), planes() converts from NCHW on demand
// (mscnn_nchw_f32_to_planes), so user code that inspects any blob by name sees ordinary Caffe
// data while layers hand planes to each other with no conversion.
//
// Versions follow the storage.  version() is the counter of the SyncedMemory holding the NCHW bytes, not of the Blob:
// blobs that ShareData (within a net by ParamSpec name, or across nets by Net::ShareTrainedLayersWith) read one
// counter, so a write through any of them (mutable_cpu_data / mutable_gpu_data / mutable_planes / set_cpu_data, and
// so CopyTrainedLayersFrom and mscnn_net_set_param) is seen by every layer that caches something derived from the
// data.  Values come from one process-wide clock and never repeat, so ShareData itself changes the version a blob
// reports.  The packed weight images live next to that counter (packed_image), one per packing key, so layers whose
// weight blobs share storage pack once and read one image.
#pragma once
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "caffe/common.hpp"
#include "caffe/proto/caffe.pb.h"
#include "caffe/syncedmem.hpp"

const int kMaxBlobAxes = 32;

namespace caffe {

// Device buffer pair for the planes representation (grow-only, like Blob::Reshape).  A store that is not `owned`
// points into a net's activation arena (Net::set_activation_reuse): it never allocates or frees, and a request
// beyond its slot is a planning bug, so reserve aborts instead of allocating.
struct CAFFE_API PlaneStore {
  void* hi = nullptr;
  void* lo = nullptr;
  size_t capacity = 0;     // bytes per plane
  size_t lo_capacity = 0;
  bool owned = true;
  ~PlaneStore();
  void reserve(size_t bytes, bool need_lo);
};

// A packed device image of a parameter blob's bytes (the weights a Convolution / InnerProduct / Deconvolution kernel
// reads), kept with the storage (SyncedMemory::packed_image).  A layer that finds it stale re-packs it under `mu` on
// its own stream and records `ready` there; a layer on another stream that finds it current waits for `ready` on the
// device before its first launch that reads this version.  No host thread waits for the device.
struct CAFFE_API PackedImage {
  std::mutex mu;
  PlaneStore w;                      // bf16 hi (+ lo on the fp32-faithful path)
  unsigned long version = ~0ul;      // the storage version it holds (~0: never packed)
  cudaEvent_t ready = nullptr;       // recorded after the last pack, on the stream that ran it
  ~PackedImage();
};

template <typename Dtype>
class CAFFE_API Blob {
 public:
  Blob() : data_(), count_(0), capacity_(0), layout_head_(HEAD_NCHW), planes_split_(false) {}
  explicit Blob(const int num, const int channels, const int height, const int width);
  explicit Blob(const vector<int>& shape);

  void Reshape(const int num, const int channels, const int height, const int width);
  void Reshape(const vector<int>& shape);
  void Reshape(const BlobShape& shape);
  void ReshapeLike(const Blob& other);
  inline string shape_string() const {
    std::ostringstream stream;
    for (size_t i = 0; i < shape_.size(); ++i) stream << shape_[i] << " ";
    stream << "(" << count_ << ")";
    return stream.str();
  }
  inline const vector<int>& shape() const { return shape_; }
  inline int shape(int index) const { return shape_[CanonicalAxisIndex(index)]; }
  inline int num_axes() const { return (int)shape_.size(); }
  inline int count() const { return count_; }
  inline int count(int start_axis, int end_axis) const {
    CHECK_LE(start_axis, end_axis);
    CHECK_GE(start_axis, 0);
    CHECK_LE(end_axis, num_axes());
    int count = 1;
    for (int i = start_axis; i < end_axis; ++i) count *= shape(i);
    return count;
  }
  inline int count(int start_axis) const { return count(start_axis, num_axes()); }
  inline int CanonicalAxisIndex(int axis_index) const {
    CHECK_GE(axis_index, -num_axes()) << "axis " << axis_index << " out of range";
    CHECK_LT(axis_index, num_axes()) << "axis " << axis_index << " out of range";
    if (axis_index < 0) return axis_index + num_axes();
    return axis_index;
  }
  inline int num() const { return LegacyShape(0); }
  inline int channels() const { return LegacyShape(1); }
  inline int height() const { return LegacyShape(2); }
  inline int width() const { return LegacyShape(3); }
  inline int LegacyShape(int index) const {
    CHECK_LE(num_axes(), 4) << "Cannot use legacy accessors on Blobs with > 4 axes.";
    CHECK_LT(index, 4);
    CHECK_GE(index, -4);
    if (index >= num_axes() || index < -num_axes()) return 1;
    return shape(index);
  }
  inline int offset(const int n, const int c = 0, const int h = 0, const int w = 0) const {
    return ((n * channels() + c) * height() + h) * width() + w;
  }
  void CopyFrom(const Blob<Dtype>& source, bool copy_diff = false, bool reshape = false);
  inline Dtype data_at(const int n, const int c, const int h, const int w) const {
    return const_cast<Blob*>(this)->cpu_data()[offset(n, c, h, w)];
  }

  const Dtype* cpu_data();
  void set_cpu_data(Dtype* data);
  const Dtype* gpu_data();
  Dtype* mutable_cpu_data();
  Dtype* mutable_gpu_data();
  void FromProto(const BlobProto& proto, bool reshape = true);
  void ToProto(BlobProto* proto, bool write_diff = false);
  Dtype asum_data();
  Dtype sumsq_data();
  void ShareData(const Blob& other);
  bool ShapeEquals(const BlobProto& other);

  // ---- mscnn_b200 extension: planes -----------------------------------------------------
  struct Planes {
    void* hi;
    void* lo;   // NULL on the plain-bf16 path
    int n, h, w, cpad;
  };
  // Current contents as planes (converted from NCHW fp32 if that is where the head is).
  Planes planes(bool split);
  // Storage for a producer to fill: sets the head to planes and invalidates the NCHW copy.
  Planes mutable_planes(bool split);
  bool head_is_planes() const { return layout_head_ == HEAD_PLANES; }
  // The storage's version (see the file comment): changed by every mutable_* accessor and by ShareData; layers use it
  // to re-pack cached weights lazily.
  unsigned long version() const { return data_ ? data_->version() : 0; }
  // The packed image of this blob's storage under `key` (see PackedImage); the blob must have storage.
  shared_ptr<PackedImage> packed_image(const std::string& key) {
    CHECK(data_);
    return data_->packed_image(key);
  }

  // ---- mscnn_b200 extension: activation arena (Net::set_activation_reuse) ----------------------------------
  // Storage in a net's arena instead of its own: planes at hi (+ lo) of plane_bytes each (hi NULL: none), NCHW fp32
  // at nchw for nchw_count values (NULL: none; the NCHW side then allocates lazily as before).  The contents are
  // undefined until a producer writes them.
  void UseArena(void* hi, void* lo, size_t plane_bytes, Dtype* nchw, int nchw_count);
  // back to storage of its own, allocated on first use
  void LeaveArena();
  // whether the arena storage set by UseArena(hi, ..., nchw, ...) is still what this blob holds, and (nchw NULL) no
  // NCHW device buffer of its own has been allocated since
  bool OnArena(const void* hi, const void* nchw) const;
  // frees an NCHW device buffer the blob allocated itself (the planes stay)
  void DropDeviceNchw();
  // A released blob's storage has been handed to a later blob: every data accessor aborts with `message`; the shape
  // stays readable.  "" = readable.
  void set_released(const string& message) { released_ = message; }
  const string& released() const { return released_; }

 protected:
  enum LayoutHead { HEAD_NCHW, HEAD_PLANES, HEAD_BOTH };
  void planes_dims(int* n, int* c, int* h, int* w) const;
  void sync_to_nchw();
  void bump_version() {
    if (data_) data_->bump_version();
  }
  void check_readable() const { CHECK(released_.empty()) << released_; }
  shared_ptr<SyncedMemory> data_;
  shared_ptr<PlaneStore> planes_;
  vector<int> shape_;
  int count_;
  int capacity_;
  LayoutHead layout_head_;
  bool planes_split_;
  string released_;
  DISABLE_COPY_AND_ASSIGN(Blob);
};

}  // namespace caffe
