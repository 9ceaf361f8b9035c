// Environment switches, read once (config.h).
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "config.h"
#include "mscnn_b200.h"

namespace mscnn {

static Config g_cfg;
static std::atomic<bool> g_loaded{false};
static std::mutex g_mu;

static void load_locked() {
  auto on = [](const char* k) { return std::getenv(k) != nullptr; };
  Config c;
  memset(&c, 0, sizeof(c));
  c.no_fat = on("MSCNN_NO_FAT");
  c.no_rowshare = on("MSCNN_NO_ROWSHARE");
  c.no_head_taps = on("MSCNN_NO_HEAD_TAPS");
  c.verbose_conv = on("MSCNN_VERBOSE_CONV");
  c.epoch = g_cfg.epoch + 1;
  g_cfg = c;
  g_loaded.store(true, std::memory_order_release);
}

const Config& config() {
  if (!g_loaded.load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_loaded.load(std::memory_order_relaxed)) load_locked();
  }
  return g_cfg;
}

void conv_plan_cache_clear();  // conv_igemm.cu

}  // namespace mscnn

extern "C" void mscnn_config_reload(void) {
  {
    std::lock_guard<std::mutex> lk(mscnn::g_mu);
    mscnn::load_locked();
  }
  mscnn::conv_plan_cache_clear();
}
