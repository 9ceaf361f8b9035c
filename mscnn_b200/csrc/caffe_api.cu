// Implementation of the Caffe-API mirror's core types: Caffe context, SyncedMemory, Blob.
// Semantics follow /root/reference/src/caffe/{common,syncedmem,blob}.cpp; citations inline.
#include <algorithm>
#include <cstring>

#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/syncedmem.hpp"

#include "caffe/layer_factory.hpp"

namespace caffe {

// ------------------------------------------------------------------------------- Caffe
Caffe& Caffe::Get() {
  // one context per thread, like boost::thread_specific_ptr<Caffe> in common.cpp:13-22
  // (a host thread per net, started and joined per call, must not leave its scratch behind)
  static thread_local std::unique_ptr<Caffe> instance(new Caffe());
  return *instance;
}

Caffe::~Caffe() {
  if (scratch_) cudaFree(scratch_);  // not checked: at process exit the runtime may already be gone
}

Caffe::Caffe() : mode_(Caffe::GPU), precision_(Caffe::FP32_SPLIT), stream_(0), scratch_(nullptr), scratch_bytes_(0) {
  if (const char* e = std::getenv("MSCNN_PRECISION")) {
    const std::string v(e);
    if (v == "bf16" || v == "BF16") precision_ = BF16;
  }
}

void* Caffe::scratch(size_t bytes) {
  Caffe& c = Get();
  if (bytes > c.scratch_bytes_) {
    // the old buffer may still be in use by queued kernels: free is stream-ordered by the driver
    if (c.scratch_) CUDA_CHECK(cudaFree(c.scratch_));
    CUDA_CHECK(cudaMalloc(&c.scratch_, bytes));
    c.scratch_bytes_ = bytes;
  }
  return c.scratch_;
}

void Caffe::SetDevice(const int device_id) { CUDA_CHECK(cudaSetDevice(device_id)); }

void Caffe::DeviceQuery() {
  cudaDeviceProp prop;
  int device;
  CUDA_CHECK(cudaGetDevice(&device));
  CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  std::cerr << "Device id: " << device << "\nName: " << prop.name << "\nMajor.minor: " << prop.major << "."
            << prop.minor << "\nSMs: " << prop.multiProcessorCount
            << "\nTotal global memory: " << prop.totalGlobalMem << std::endl;
}

// -------------------------------------------------------------------------- SyncedMemory
// Host STORAGE (not compute) also works without a CUDA device, so that nets can be constructed
// and inspected on a GPU-less machine (graph / shape logic is testable there); any Forward still
// needs the device and aborts without one.
static bool g_host_pinned = true;
static void* host_alloc(size_t bytes) {
  void* p = nullptr;
  if (g_host_pinned && cudaMallocHost(&p, bytes) == cudaSuccess) return p;
  cudaGetLastError();
  g_host_pinned = false;
  p = malloc(bytes);
  CHECK(p) << "host allocation of " << bytes << " bytes failed";
  return p;
}
static void host_free(void* p) {
  if (g_host_pinned) cudaFreeHost(p);
  else free(p);
}

static std::atomic<unsigned long> g_storage_clock{0};
unsigned long next_storage_version() { return g_storage_clock.fetch_add(1, std::memory_order_relaxed) + 1; }

SyncedMemory::~SyncedMemory() {
  if (cpu_ptr_ && own_cpu_data_) host_free(cpu_ptr_);
  if (gpu_ptr_ && own_gpu_data_) cudaFree(gpu_ptr_);
  if (upload_) cudaEventDestroy(upload_);
}

inline void SyncedMemory::wait_upload() {
  if (!upload_pending_) return;
  const cudaStream_t s = Caffe::stream();
  if (s == upload_stream_ || std::find(upload_waited_.begin(), upload_waited_.end(), s) != upload_waited_.end()) return;
  CUDA_CHECK(cudaStreamWaitEvent(s, upload_, 0));
  upload_waited_.push_back(s);
}

shared_ptr<PackedImage> SyncedMemory::packed_image(const std::string& key) {
  std::lock_guard<std::mutex> lk(packed_mu_);
  shared_ptr<PackedImage>& p = packed_[key];
  if (!p) p.reset(new PackedImage());
  return p;
}

inline void SyncedMemory::to_cpu() {  // syncedmem.cpp:25-49
  switch (head_) {
    case UNINITIALIZED:
      cpu_ptr_ = host_alloc(size_ ? size_ : 1);
      memset(cpu_ptr_, 0, size_);
      head_ = HEAD_AT_CPU;
      own_cpu_data_ = true;
      break;
    case HEAD_AT_GPU:
      if (cpu_ptr_ == NULL) {
        cpu_ptr_ = host_alloc(size_ ? size_ : 1);
        own_cpu_data_ = true;
      }
      wait_upload();
      CUDA_CHECK(cudaMemcpyAsync(cpu_ptr_, gpu_ptr_, size_, cudaMemcpyDeviceToHost, Caffe::stream()));
      CUDA_CHECK(cudaStreamSynchronize(Caffe::stream()));
      head_ = SYNCED;
      break;
    case HEAD_AT_CPU:
    case SYNCED:
      break;
  }
}

inline void SyncedMemory::to_gpu() {  // syncedmem.cpp:51-77
  switch (head_) {
    case UNINITIALIZED:
      CUDA_CHECK(cudaMalloc(&gpu_ptr_, size_ ? size_ : 1));
      CUDA_CHECK(cudaMemsetAsync(gpu_ptr_, 0, size_, Caffe::stream()));
      head_ = HEAD_AT_GPU;
      own_gpu_data_ = true;
      break;
    case HEAD_AT_CPU:
      if (gpu_ptr_ == NULL) {
        CUDA_CHECK(cudaMalloc(&gpu_ptr_, size_ ? size_ : 1));
        own_gpu_data_ = true;
      }
      CUDA_CHECK(cudaMemcpyAsync(gpu_ptr_, cpu_ptr_, size_, cudaMemcpyHostToDevice, Caffe::stream()));
      {
        // another thread's stream may read these bytes next (storage shared between nets): mark where they land
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        CUDA_CHECK(cudaStreamIsCapturing(Caffe::stream(), &cap));
        if (cap == cudaStreamCaptureStatusNone) {
          if (!upload_) CUDA_CHECK(cudaEventCreateWithFlags(&upload_, cudaEventDisableTiming));
          CUDA_CHECK(cudaEventRecord(upload_, Caffe::stream()));
          upload_stream_ = Caffe::stream();
          upload_pending_ = true;
          upload_waited_.clear();
        }
      }
      head_ = SYNCED;
      break;
    case HEAD_AT_GPU:
    case SYNCED:
      break;
  }
}

const void* SyncedMemory::cpu_data() {
  std::lock_guard<std::mutex> lk(mu_);
  to_cpu();
  return (const void*)cpu_ptr_;
}
void SyncedMemory::set_cpu_data(void* data) {
  CHECK(data);
  std::lock_guard<std::mutex> lk(mu_);
  if (own_cpu_data_) host_free(cpu_ptr_);
  cpu_ptr_ = data;
  head_ = HEAD_AT_CPU;
  own_cpu_data_ = false;
}
const void* SyncedMemory::gpu_data() {
  std::lock_guard<std::mutex> lk(mu_);
  to_gpu();
  wait_upload();
  return (const void*)gpu_ptr_;
}
void SyncedMemory::set_gpu_data(void* data) {
  CHECK(data);
  std::lock_guard<std::mutex> lk(mu_);
  if (own_gpu_data_) cudaFree(gpu_ptr_);
  gpu_ptr_ = data;
  head_ = HEAD_AT_GPU;
  own_gpu_data_ = false;
  upload_pending_ = false;
}
void* SyncedMemory::mutable_cpu_data() {
  std::lock_guard<std::mutex> lk(mu_);
  to_cpu();
  head_ = HEAD_AT_CPU;
  return cpu_ptr_;
}
void* SyncedMemory::mutable_gpu_data() {
  std::lock_guard<std::mutex> lk(mu_);
  to_gpu();
  wait_upload();
  head_ = HEAD_AT_GPU;
  return gpu_ptr_;
}

// ---------------------------------------------------------------------------- PlaneStore
PlaneStore::~PlaneStore() {
  if (!owned) return;
  if (hi) cudaFree(hi);
  if (lo) cudaFree(lo);
}
void PlaneStore::reserve(size_t bytes, bool need_lo) {
  if (!owned) {
    CHECK(hi && bytes <= capacity && (!need_lo || (lo && bytes <= lo_capacity)))
        << "activation arena miss: a planned blob needs " << bytes << " bytes per plane" << (need_lo ? " (hi and lo)" : "")
        << " but its arena slot holds " << capacity << (lo ? " (hi and lo)" : " (hi only)")
        << "; the activation plan does not describe this forward";
    return;
  }
  if (bytes > capacity) {
    if (hi) CUDA_CHECK(cudaFree(hi));
    CUDA_CHECK(cudaMalloc(&hi, bytes));
    capacity = bytes;
  }
  if (need_lo && bytes > lo_capacity) {
    if (lo) CUDA_CHECK(cudaFree(lo));
    CUDA_CHECK(cudaMalloc(&lo, bytes));
    lo_capacity = bytes;
  }
}

PackedImage::~PackedImage() {
  if (ready) cudaEventDestroy(ready);
}

// ---------------------------------------------------------------------------------- Blob
template <typename Dtype>
Blob<Dtype>::Blob(const int num, const int channels, const int height, const int width)
    : count_(0), capacity_(0), layout_head_(HEAD_NCHW), planes_split_(false) {
  Reshape(num, channels, height, width);
}
template <typename Dtype>
Blob<Dtype>::Blob(const vector<int>& shape)
    : count_(0), capacity_(0), layout_head_(HEAD_NCHW), planes_split_(false) {
  Reshape(shape);
}

template <typename Dtype>
void Blob<Dtype>::Reshape(const int num, const int channels, const int height, const int width) {
  vector<int> shape(4);
  shape[0] = num;
  shape[1] = channels;
  shape[2] = height;
  shape[3] = width;
  Reshape(shape);
}

template <typename Dtype>
void Blob<Dtype>::Reshape(const vector<int>& shape) {  // blob.cpp:23-45: grow-only capacity
  CHECK_LE(shape.size(), (size_t)kMaxBlobAxes);
  bool same = (shape == shape_);
  // a trim along axis 0 keeps the leading rows of BOTH layouts valid (NCHW rows and NHWC planes are row-major in n):
  // that is what Net::ResolveRows does to the blobs behind BoxOutput once the data-dependent row count is known
  if (!same && shape.size() == shape_.size() && !shape.empty() && shape[0] <= shape_[0] &&
      std::equal(shape.begin() + 1, shape.end(), shape_.begin() + 1))
    same = true;
  count_ = 1;
  shape_.resize(shape.size());
  for (size_t i = 0; i < shape.size(); ++i) {
    CHECK_GE(shape[i], 0);
    if (count_ != 0) CHECK_LE(shape[i], INT_MAX / count_) << "blob size exceeds INT_MAX";
    count_ *= shape[i];
    shape_[i] = shape[i];
  }
  if (count_ > capacity_) {
    capacity_ = count_;
    data_.reset(new SyncedMemory(capacity_ * sizeof(Dtype)));
    if (layout_head_ == HEAD_BOTH) layout_head_ = HEAD_PLANES;
  }
  if (!same && layout_head_ != HEAD_NCHW) {
    // a planes image of the old shape does not describe the new one
    layout_head_ = HEAD_NCHW;
  }
}

template <typename Dtype>
void Blob<Dtype>::Reshape(const BlobShape& shape) {
  CHECK_LE(shape.dim_size(), kMaxBlobAxes);
  vector<int> shape_vec(shape.dim_size());
  for (int i = 0; i < shape.dim_size(); ++i) shape_vec[i] = (int)shape.dim(i);
  Reshape(shape_vec);
}

template <typename Dtype>
void Blob<Dtype>::ReshapeLike(const Blob<Dtype>& other) {
  Reshape(other.shape());
}

template <typename Dtype>
void Blob<Dtype>::planes_dims(int* n, int* c, int* h, int* w) const {
  CHECK_LE(num_axes(), 4) << "planes need a blob with at most 4 axes";
  *n = LegacyShape(0);
  *c = LegacyShape(1);
  *h = LegacyShape(2);
  *w = LegacyShape(3);
}

template <typename Dtype>
void Blob<Dtype>::sync_to_nchw() {
  if (layout_head_ != HEAD_PLANES) return;
  int n, c, h, w;
  planes_dims(&n, &c, &h, &w);
  CHECK(data_);
  Dtype* dst = static_cast<Dtype*>(data_->mutable_gpu_data());
  if (count_ > 0) {
    const int cpad = (c + 63) / 64 * 64;
    MSCNN_CHECK(mscnn_planes_to_nchw_f32(planes_->hi, planes_split_ ? planes_->lo : nullptr, dst, n, c, h, w,
                                         cpad, Caffe::stream()));
  }
  layout_head_ = HEAD_BOTH;
}

template <typename Dtype>
const Dtype* Blob<Dtype>::cpu_data() {
  check_readable();
  CHECK(data_);
  sync_to_nchw();
  return (const Dtype*)data_->cpu_data();
}
template <typename Dtype>
void Blob<Dtype>::set_cpu_data(Dtype* data) {
  CHECK(data);
  check_readable();
  data_->set_cpu_data(data);
  layout_head_ = HEAD_NCHW;
  bump_version();
}
template <typename Dtype>
const Dtype* Blob<Dtype>::gpu_data() {
  check_readable();
  CHECK(data_);
  sync_to_nchw();
  return (const Dtype*)data_->gpu_data();
}
template <typename Dtype>
Dtype* Blob<Dtype>::mutable_cpu_data() {
  check_readable();
  CHECK(data_);
  sync_to_nchw();
  layout_head_ = HEAD_NCHW;
  bump_version();
  return static_cast<Dtype*>(data_->mutable_cpu_data());
}
template <typename Dtype>
Dtype* Blob<Dtype>::mutable_gpu_data() {
  check_readable();
  CHECK(data_);
  sync_to_nchw();
  layout_head_ = HEAD_NCHW;
  bump_version();
  return static_cast<Dtype*>(data_->mutable_gpu_data());
}

template <typename Dtype>
typename Blob<Dtype>::Planes Blob<Dtype>::planes(bool split) {
  check_readable();
  int n, c, h, w;
  planes_dims(&n, &c, &h, &w);
  const int cpad = (c + 63) / 64 * 64;
  if (layout_head_ == HEAD_NCHW || (split && !planes_split_)) {
    // (re)build planes from the fp32 data
    if (layout_head_ == HEAD_PLANES) sync_to_nchw();
    if (!planes_) planes_.reset(new PlaneStore());
    const size_t bytes = (size_t)n * h * w * cpad * 2;
    planes_->reserve(bytes ? bytes : 2, split);
    if (count_ > 0) {
      const Dtype* src = static_cast<const Dtype*>(data_->gpu_data());
      MSCNN_CHECK(mscnn_nchw_f32_to_planes(src, planes_->hi, split ? planes_->lo : nullptr, n, c, h, w, cpad,
                                           Caffe::stream()));
    }
    planes_split_ = split;
    layout_head_ = HEAD_BOTH;
  }
  Planes p;
  p.hi = planes_->hi;
  p.lo = (split && planes_split_) ? planes_->lo : nullptr;
  p.n = n; p.h = h; p.w = w; p.cpad = cpad;
  return p;
}

template <typename Dtype>
typename Blob<Dtype>::Planes Blob<Dtype>::mutable_planes(bool split) {
  check_readable();
  int n, c, h, w;
  planes_dims(&n, &c, &h, &w);
  const int cpad = (c + 63) / 64 * 64;
  if (!planes_) planes_.reset(new PlaneStore());
  const size_t bytes = (size_t)n * h * w * cpad * 2;
  planes_->reserve(bytes ? bytes : 2, split);
  planes_split_ = split;
  layout_head_ = HEAD_PLANES;
  bump_version();
  Planes p;
  p.hi = planes_->hi;
  p.lo = split ? planes_->lo : nullptr;
  p.n = n; p.h = h; p.w = w; p.cpad = cpad;
  return p;
}

template <typename Dtype>
void Blob<Dtype>::UseArena(void* hi, void* lo, size_t plane_bytes, Dtype* nchw, int nchw_count) {
  if (hi) {
    planes_.reset(new PlaneStore());
    planes_->owned = false;
    planes_->hi = hi;
    planes_->lo = lo;
    planes_->capacity = plane_bytes;
    planes_->lo_capacity = lo ? plane_bytes : 0;
  } else {
    planes_.reset();
  }
  if (nchw) {
    // the slot holds nchw_count values: that is the capacity now, so a Reshape within it keeps the slot
    capacity_ = nchw_count;
    data_.reset(new SyncedMemory((size_t)nchw_count * sizeof(Dtype)));
    data_->set_gpu_data(nchw);
  } else {
    data_.reset(new SyncedMemory((size_t)capacity_ * sizeof(Dtype)));
  }
  layout_head_ = HEAD_NCHW;
  planes_split_ = false;
}
template <typename Dtype>
void Blob<Dtype>::LeaveArena() {
  planes_.reset();
  data_.reset(new SyncedMemory((size_t)capacity_ * sizeof(Dtype)));
  layout_head_ = HEAD_NCHW;
  planes_split_ = false;
  released_.clear();
}
template <typename Dtype>
bool Blob<Dtype>::OnArena(const void* hi, const void* nchw) const {
  if (hi && !(planes_ && !planes_->owned && planes_->hi == hi)) return false;
  if (nchw) return data_ && data_->gpu_ptr() == nchw;
  return !(data_ && data_->owns_gpu_data());
}
template <typename Dtype>
void Blob<Dtype>::DropDeviceNchw() {
  if (!data_ || !data_->owns_gpu_data()) return;
  data_.reset(new SyncedMemory((size_t)capacity_ * sizeof(Dtype)));
  if (layout_head_ == HEAD_BOTH) layout_head_ = HEAD_PLANES;
}

template <typename Dtype>
void Blob<Dtype>::ShareData(const Blob& other) {  // blob.cpp:149-153
  CHECK_EQ(count_, other.count());
  data_ = other.data_;
  planes_ = other.planes_;
  layout_head_ = other.layout_head_;
  planes_split_ = other.planes_split_;
  // the version now is the shared storage's (a value this blob never had: the clock never repeats), so every cache
  // keyed on it, packed weights and CUDA graphs included, sees the change without a write
}

template <typename Dtype>
void Blob<Dtype>::CopyFrom(const Blob& source, bool copy_diff, bool reshape) {  // blob.cpp:415-446
  if (source.count() != count_ || source.shape() != shape_) {
    if (reshape) ReshapeLike(source);
    else LOG(FATAL) << "Trying to copy blobs of different sizes.";
  }
  CHECK(!copy_diff) << "mscnn_b200 blobs carry no diff";
  Blob& src = const_cast<Blob&>(source);
  if (count_ > 0)
    CUDA_CHECK(cudaMemcpyAsync(mutable_gpu_data(), src.gpu_data(), sizeof(Dtype) * count_,
                               cudaMemcpyDeviceToDevice, Caffe::stream()));
}

template <typename Dtype>
bool Blob<Dtype>::ShapeEquals(const BlobProto& other) {  // blob.cpp:392-413
  if (other.has_num() || other.has_channels() || other.has_height() || other.has_width()) {
    return shape_.size() <= 4 && LegacyShape(-4) == other.num() && LegacyShape(-3) == other.channels() &&
           LegacyShape(-2) == other.height() && LegacyShape(-1) == other.width();
  }
  vector<int> other_shape(other.shape().dim_size());
  for (int i = 0; i < other.shape().dim_size(); ++i) other_shape[i] = (int)other.shape().dim(i);
  return shape_ == other_shape;
}

template <typename Dtype>
void Blob<Dtype>::FromProto(const BlobProto& proto, bool reshape) {  // blob.cpp:448-500
  if (reshape) {
    vector<int> shape;
    if (proto.has_num() || proto.has_channels() || proto.has_height() || proto.has_width()) {
      shape.resize(4);
      shape[0] = proto.num();
      shape[1] = proto.channels();
      shape[2] = proto.height();
      shape[3] = proto.width();
    } else {
      shape.resize(proto.shape().dim_size());
      for (int i = 0; i < proto.shape().dim_size(); ++i) shape[i] = (int)proto.shape().dim(i);
    }
    Reshape(shape);
  } else {
    CHECK(ShapeEquals(proto)) << "shape mismatch (reshape not set)";
  }
  Dtype* data_vec = mutable_cpu_data();
  if (proto.double_data_size() > 0) {
    CHECK_EQ(count_, proto.double_data_size());
    for (int i = 0; i < count_; ++i) data_vec[i] = (Dtype)proto.double_data(i);
  } else {
    CHECK_EQ(count_, proto.data_size());
    for (int i = 0; i < count_; ++i) data_vec[i] = proto.data(i);
  }
}

template <typename Dtype>
void Blob<Dtype>::ToProto(BlobProto* proto, bool write_diff) {  // blob.cpp:502-520
  proto->clear_shape();
  for (size_t i = 0; i < shape_.size(); ++i) proto->mutable_shape()->add_dim(shape_[i]);
  proto->clear_data();
  proto->clear_diff();
  const Dtype* data_vec = cpu_data();
  for (int i = 0; i < count_; ++i) proto->add_data(data_vec[i]);
}

template <typename Dtype>
Dtype Blob<Dtype>::asum_data() {
  const Dtype* d = cpu_data();
  double s = 0;
  for (int i = 0; i < count_; ++i) s += std::fabs(d[i]);
  return (Dtype)s;
}
template <typename Dtype>
Dtype Blob<Dtype>::sumsq_data() {
  const Dtype* d = cpu_data();
  double s = 0;
  for (int i = 0; i < count_; ++i) s += (double)d[i] * d[i];
  return (Dtype)s;
}

INSTANTIATE_CLASS(Blob);

// The one layer-type table of the process and its accessors (layer_factory.hpp).
template <typename Dtype>
typename LayerRegistry<Dtype>::CreatorRegistry& LayerRegistry<Dtype>::Registry() {
  static CreatorRegistry* table = new CreatorRegistry();  // never destroyed: layers may be created during shutdown
  return *table;
}

template <typename Dtype>
void LayerRegistry<Dtype>::AddCreator(const string& type, Creator creator) {
  const bool fresh = Registry().insert(std::make_pair(type, creator)).second;
  CHECK(fresh) << "Layer type " << type << " already registered.";
}

template <typename Dtype>
vector<string> LayerRegistry<Dtype>::LayerTypeList() {
  vector<string> names;
  for (const auto& entry : Registry()) names.push_back(entry.first);
  return names;
}

template <typename Dtype>
shared_ptr<Layer<Dtype> > LayerRegistry<Dtype>::CreateLayer(const LayerParameter& param) {
  const CreatorRegistry& table = Registry();
  const typename CreatorRegistry::const_iterator it = table.find(param.type());
  if (it == table.end()) {
    string known;
    for (const string& t : LayerTypeList()) known += (known.empty() ? "" : ", ") + t;
    LOG(FATAL) << "Unknown layer type: " << param.type() << " (known types: " << known << ")";
  }
  return it->second(param);
}

template <typename Dtype>
LayerRegisterer<Dtype>::LayerRegisterer(const string& type, typename LayerRegistry<Dtype>::Creator creator) {
  LayerRegistry<Dtype>::AddCreator(type, creator);
}

template class LayerRegistry<float>;
template struct LayerRegisterer<float>;

}  // namespace caffe
