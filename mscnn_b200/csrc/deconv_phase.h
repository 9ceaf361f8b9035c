// Deconvolution (transposed convolution) split by output phase: host-side arithmetic shared by the weight packer
// (layout.cu) and the launches (conv_igemm.cu).
//
// Caffe's deconvolution along one axis (col2im form, deconv_layer.cpp:25-40) is y[i s - p + t d] += x[i] w[t], t in
// [0, k), output extent s (in - 1) + d (k - 1) + 1 - 2 p (deconv_layer.cpp:8-22).  Write the output index o = q s + r
// with phase r in [0, s).  Tap t reaches phase r when (r + p - t d) mod s == 0; those taps t_0 < ... < t_{m-1} are
// s / gcd(s, d) apart.  With the tap order reversed, phase r is a stride-1 convolution of x:
//   y[q s + r] = sum_u x[q - P + u d'] w[t_{m-1-u}],   d' = d / gcd(s, d),   P = -(r + p - t_{m-1} d) / s,
// with m taps, a signed pad P and Q = ceil((out - r) / s) outputs.  Each tap belongs to exactly one phase.
#pragma once

namespace mscnn {

constexpr int kDeconvMaxStride = 8;
constexpr int kDeconvMaxReach = 1 << 20;  // pad and dilated kernel reach: tap coordinates stay far inside int32

struct DeconvAxis {
  int taps;   // m (0: no tap reaches the phase)
  int t0;     // first (smallest) tap of the phase
  int tstep;  // s / gcd(s, d): distance between its taps
  int dil;    // d / gcd(s, d): the sub-convolution's dilation
  int pad;    // P, signed
  int ext;    // Q: outputs of the phase
};

inline int deconv_gcd(int a, int b) {
  while (b) {
    const int t = a % b;
    a = b;
    b = t;
  }
  return a;
}

inline int deconv_out_size(int in, int k, int s, int p, int d) { return s * (in - 1) + d * (k - 1) + 1 - 2 * p; }

// one axis of one phase r of a deconvolution with kernel k, stride s, pad p, dilation d and output extent out
inline DeconvAxis deconv_axis(int k, int s, int p, int d, int out, int r) {
  DeconvAxis a = {0, 0, 1, 1, 0, 0};
  const int g = deconv_gcd(s, d);
  a.tstep = s / g;
  a.dil = d / g;
  a.ext = out > r ? (out - r + s - 1) / s : 0;
  for (int t = 0; t < a.tstep && t < k; ++t) {  // the residues of t d mod s repeat with period s / g
    if (((r + p - t * d) % s + s) % s == 0) {
      a.t0 = t;
      a.taps = (k - 1 - t) / a.tstep + 1;
      a.pad = -(r + p - (t + (a.taps - 1) * a.tstep) * d) / s;  // exact: s divides it
      break;
    }
  }
  return a;
}

// kernel, stride, pad and dilation of one axis are in the served range
inline bool deconv_axis_ok(int k, int s, int p, int d) {
  return k >= 1 && s >= 1 && s <= kDeconvMaxStride && p >= 0 && p < kDeconvMaxReach && d >= 1 &&
         d <= kDeconvMaxReach / k;
}

// Packed deconvolution weights (one plane): the phases (r_h, r_w) in row-major order, each the sub-kernel
// [Cout_pad][m_h][m_w][cin_g] in mscnn_pack_conv_weights' layout, cin_g = Cin / group padded to 64.  The offset in
// elements of phase number `phase` = r_h s_w + r_w; phase = s_h s_w gives the size (KH KW Cout_pad cin_g, since every
// tap lies in exactly one phase).  -1 when the geometry is not served.
inline long long deconv_phase_offset(int Cin, int group, int KH, int KW, int sh, int sw, int ph, int pw, int dh, int dw,
                                     int Cout_pad, int phase) {
  if (group < 1 || Cin < 1 || Cin % group || Cout_pad < 1 || !deconv_axis_ok(KH, sh, ph, dh) ||
      !deconv_axis_ok(KW, sw, pw, dw))
    return -1;
  const long long per_tap = (long long)Cout_pad * ((Cin / group + 63) / 64 * 64);
  long long taps = 0;
  for (int i = 0; i < phase && i < sh * sw; ++i)
    taps += (long long)deconv_axis(KH, sh, ph, dh, 0, i / sw).taps * deconv_axis(KW, sw, pw, dw, 0, i % sw).taps;
  return taps * per_tap;
}

}  // namespace mscnn
