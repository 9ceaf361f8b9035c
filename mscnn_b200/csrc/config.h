// Process-wide switches of the library, read from the environment ONCE (first use) instead of with getenv() on every
// launch.  mscnn_config_reload() re-reads them and drops every cached launch plan: it exists for the tests, which hold
// each operand-delivery variant of the convolution kernel to the fp64 convolution (DESIGN.md 4.1c).
#pragma once

namespace mscnn {

struct Config {
  bool no_fat;      // MSCNN_NO_FAT: term-major k-blocks for every fp32-faithful layer
  bool no_rowshare; // MSCNN_NO_ROWSHARE: one activation tile per tap, also where three horizontal taps could share one
  bool no_head_taps;
  bool verbose_conv;
  unsigned epoch;  // bumped by every reload: cached plans carry the epoch they were built under
};

const Config& config();

}  // namespace mscnn
