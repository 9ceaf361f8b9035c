// Process-wide count of the kernels this library has launched (every `<<<>>>` site calls
// note_launch()).  bench.py reads it through mscnn_kernel_launch_count() to report `gpu_launches`
// from a count, not an estimate.  Also the count of weight images packed (PackedParam::update_weights), which shows
// that nets sharing their weights pack each image once (mscnn_weight_pack_count()).
#pragma once
#include <atomic>

namespace mscnn {
extern std::atomic<unsigned long long> g_kernel_launches;
inline void note_launch() { g_kernel_launches.fetch_add(1, std::memory_order_relaxed); }
extern std::atomic<unsigned long long> g_weight_packs;
}  // namespace mscnn
