// SyncedMemory: lazily allocated host/device mirror with the reference's head state machine
// (/root/reference/include/caffe/syncedmem.hpp:45-83, src/caffe/syncedmem.cpp:25-139).
// Host memory is pinned (cudaMallocHost) as the reference does in GPU mode (syncedmem.hpp:15-26).
//
// mscnn_b200 additions, for storage that blobs of several nets share (Blob::ShareData, Net::ShareTrainedLayersWith):
//   * the version counter of the bytes (Blob::version), so that a write through any sharing blob is seen by all;
//   * the packed device images derived from the bytes (Blob::packed_image), one per packing key;
//   * thread safety: the head state machine runs under a mutex, and a host -> device upload issued on one stream is
//     waited for, on the device, by the first access from any other stream.
#pragma once
#include <atomic>
#include <cstdlib>
#include <mutex>

#include "caffe/common.hpp"

namespace caffe {

struct PackedImage;  // blob.hpp

// One process-wide clock for storage versions: every storage starts at a fresh value and every write takes the next,
// so a version names one state of one storage and never recurs, even across storages.
CAFFE_API unsigned long next_storage_version();

class CAFFE_API SyncedMemory {
 public:
  SyncedMemory() : cpu_ptr_(NULL), gpu_ptr_(NULL), size_(0), head_(UNINITIALIZED), own_cpu_data_(false),
                   own_gpu_data_(false), version_(next_storage_version()) {}
  explicit SyncedMemory(size_t size) : cpu_ptr_(NULL), gpu_ptr_(NULL), size_(size), head_(UNINITIALIZED),
                                       own_cpu_data_(false), own_gpu_data_(false), version_(next_storage_version()) {}
  ~SyncedMemory();
  const void* cpu_data();
  void set_cpu_data(void* data);
  const void* gpu_data();
  void set_gpu_data(void* data);
  void* mutable_cpu_data();
  void* mutable_gpu_data();
  enum SyncedHead { UNINITIALIZED, HEAD_AT_CPU, HEAD_AT_GPU, SYNCED };
  SyncedHead head() { return head_; }
  size_t size() { return size_; }
  const void* gpu_ptr() const { return gpu_ptr_; }  // the device buffer as it is (NULL: none yet); allocates nothing
  bool owns_gpu_data() const { return gpu_ptr_ && own_gpu_data_; }  // a device buffer it allocated itself

  // mscnn_b200 extension: see the file comment.
  unsigned long version() const { return version_.load(std::memory_order_acquire); }
  void bump_version() { version_.store(next_storage_version(), std::memory_order_release); }
  // The packed image of these bytes under `key` (created empty on first request); every holder of the storage gets
  // the same image.
  shared_ptr<PackedImage> packed_image(const std::string& key);

 private:
  void to_cpu();
  void to_gpu();
  void wait_upload();  // the calling thread's stream waits for the last upload if another stream issued it
  void* cpu_ptr_;
  void* gpu_ptr_;
  size_t size_;
  SyncedHead head_;
  bool own_cpu_data_;
  bool own_gpu_data_;
  std::atomic<unsigned long> version_;
  std::mutex mu_;                        // head transitions
  cudaEvent_t upload_ = nullptr;         // recorded after the last host -> device upload ...
  cudaStream_t upload_stream_ = nullptr; // ... on this stream
  bool upload_pending_ = false;
  vector<cudaStream_t> upload_waited_;   // streams already ordered after it
  std::mutex packed_mu_;
  map<string, shared_ptr<PackedImage> > packed_;
  DISABLE_COPY_AND_ASSIGN(SyncedMemory);
};

}  // namespace caffe
