/*
 * mscnn_b200 -- C ABI of the H100-native (sm_90a) MS-CNN detection forward path.
 *
 * The reference (zhaoweicai/mscnn, a Caffe fork) has no C ABI: its boundary for this path is
 * the C++ class caffe::Layer<Dtype> (include/caffe/layer.hpp:33-445) whose Forward_gpu
 * virtuals call cuDNN / cuBLAS / ad-hoc kernels.  Every entry point below is what one such
 * Forward_gpu would bind instead; the reference call site it replaces is cited per function.
 * INTEGRATION.md shows the Caffe-side Layer::Forward_gpu stubs.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless named host_*;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - every function returns MSCNN_OK (0) or a negative MSCNN_ERR_* code and never aborts;
 *     the C++ Caffe-API mirror wraps them in CHECK_EQ(rc, 0) to keep Caffe's abort-on-error
 *     convention (include/caffe/util/device_alternate.hpp:48-53);
 *   - no CPU fallback exists: without a CUDA device the compute calls return MSCNN_ERR_CUDA.
 *
 * Activation storage ("planes")
 *   Internal activations are NHWC bf16 with the channel count padded to a multiple of 64.
 *   An fp32-faithful tensor is a PAIR of planes (hi, lo): x ~= hi + lo with hi = bf16(x),
 *   lo = bf16(x - hi) (relative error <= 2^-17).  Passing lo == NULL everywhere selects the
 *   plain bf16 path.  Caffe-visible blobs are NCHW fp32; the mscnn_nchw_* / mscnn_nhwc_*
 *   converters move between the two.
 */
#ifndef MSCNN_B200_H_
#define MSCNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Only the C ABI is exported from libmscnn_b200.so (the library is built with hidden visibility
 * so that its internal C++ symbols cannot collide with another Caffe in the same process). */
#if defined(__GNUC__)
#define MSCNN_API __attribute__((visibility("default")))
#else
#define MSCNN_API
#endif

#define MSCNN_OK 0
#define MSCNN_ERR_INVALID (-1) /* bad argument / unsupported shape */
#define MSCNN_ERR_CUDA (-2)    /* CUDA runtime or driver error (message on stderr) */
#define MSCNN_ERR_NOMEM (-3)

#define MSCNN_OUT_NHWC_BF16 0 /* planes, via TMA store */
#define MSCNN_OUT_NCHW_F32 1  /* Caffe blob layout, fp32 */
#define MSCNN_OUT_NHWC_F32 2  /* pixel-major fp32 rows [N*Ho*Wo][Cout_pad] (head-tap partial sums) */

#define MSCNN_POOL_MAX 0
#define MSCNN_POOL_AVE 1

#define MSCNN_NMS_IOU 0  /* intersection / union            */
#define MSCNN_NMS_IOMU 1 /* intersection / min(area)        */
#define MSCNN_NMS_IOFU 2 /* intersection / area(first box)  */

#define MSCNN_MAX_SCALES 16

/* library / device ------------------------------------------------------------------ */
MSCNN_API const char* mscnn_version(void);
MSCNN_API int mscnn_sm_count(void);
/* Number of CUDA kernels this library has launched in this process so far (all entry points). */
MSCNN_API unsigned long long mscnn_kernel_launch_count(void);
/* Number of packed weight images this process has (re-)packed so far: nets that share their weights
 * (mscnn_net_share_trained_layers) pack each image once between them. */
MSCNN_API unsigned long long mscnn_weight_pack_count(void);
/* The MSCNN_* environment switches (DESIGN.md 4.1c) are read once, not per launch.  This re-reads them and drops the
 * cached convolution launch plans; mscnn_net_create calls it.  The reference reads its switches (Caffe::mode, cuDNN
 * engine choice) at layer set-up too (src/caffe/layer_factory.cpp:37-65). */
MSCNN_API void mscnn_config_reload(void);

/* ------------------------------------------------------------------------------------
 * Convolution (stride, dilation, groups) / InnerProduct with fused bias and optional ReLU.
 * Replaces ConvolutionLayer::Forward_gpu (src/caffe/layers/conv_layer.cu:8-23,
 * cudnn_conv_layer.cu:11-46), InnerProductLayer::Forward_gpu (inner_product_layer.cu:10-31)
 * and the in-place ReLULayer::Forward_gpu that follows them (relu_layer.cu:9-26).
 *   x   : planes [N][H][W][C], C % 64 == 0
 *   w   : planes [Cout_pad][KH][KW][C / group]  (mscnn_pack_conv_weights / mscnn_pack_fc_weights)
 *   bias: fp32 [Cout_pad]
 *   out : MSCNN_OUT_NHWC_BF16 -> y planes [N][Ho][Wo][Cout_pad] (Cout_pad % 64 == 0)
 *         MSCNN_OUT_NCHW_F32  -> y_f32 [N][Cout][Ho][Wo]
 *         MSCNN_OUT_NHWC_F32  -> y_f32 [N][Ho][Wo][Cout_pad]
 *   Ho = (H + 2 pad_h - (dil_h (KH - 1) + 1)) / stride_h + 1, Wo likewise (conv_layer.cpp:8-22); tap (dy, dx) of
 *   output pixel (ho, wo) reads input pixel (ho stride_h + dy dil_h - pad_h, wo stride_w + dx dil_w - pad_w), zero
 *   outside the image.  InnerProduct = KH = KW = H = W = 1.
 *   group = g > 1 (base_conv_layer.cpp:108-120): output channels [k Cout/g, (k+1) Cout/g) see input channels
 *   [k C/g, (k+1) C/g); C / g and Cout / g must be multiples of 64 and Cout_pad == Cout.  The weight planes are
 *   mscnn_pack_conv_weights of the Caffe blob [Cout][C/g][KH][KW] with Cin = Cin_pad = C / g.
 *   Served: strides 1..4, any dilation whose taps fit a tensor map's coordinate range; anything else returns
 *   MSCNN_ERR_INVALID with a message on stderr.
 */
typedef struct mscnn_conv_desc {
  const void* x_hi;
  const void* x_lo; /* NULL -> single-term bf16 */
  int N, H, W, C;
  const void* w_hi;
  const void* w_lo;
  const float* bias;
  int Cout, Cout_pad, KH, KW, pad_h, pad_w;
  int relu;
  int out_mode;
  void* y_hi;
  void* y_lo; /* may be NULL even when x_lo is set (bf16-only output) */
  float* y_f32;
  /* Optional fused PoolingLayer (MAX, 2x2, stride 2; pooling_layer.cu:158-190) on the NHWC_BF16
   * output: pool planes [N][Ho/2][Wo/2][Cout_pad] (Ho, Wo even).  With pool_hi set, y_hi may be
   * NULL: the un-pooled tensor is then never written to HBM. */
  void* pool_hi;
  void* pool_lo;
  /* Optional data-dependent batch size (device int, may be NULL): the kernel processes min(*dyn_n, N) images / rows
   * and leaves the rest of y untouched.  The detection head runs on BoxOutput's R proposals, a count that only exists
   * on the device when the head is launched (the reference learns it on the host, box_output_layer.cpp:201): the
   * launch is sized for the cap N and R is read by the kernel. */
  const int* dyn_n;
  /* Geometry beyond stride 1 / dilation 1 / group 1.  0 means 1, so a zero-initialised descriptor without these
   * fields set is the plain convolution. */
  int stride_h, stride_w, dil_h, dil_w, group;
} mscnn_conv_desc;
MSCNN_API int mscnn_conv_forward(const mscnn_conv_desc* d, void* stream);
/* Host-only: the launch plan mscnn_conv_forward would use for `d` as one line of text (kernel instantiation, pixel box,
 * operand staging, pipeline depth); no CUDA call, the pointers only have to be non-NULL. */
MSCNN_API int mscnn_conv_plan_describe(const mscnn_conv_desc* d, char* buf, int cap);
/* Host-only: the number of launch plans mscnn_conv_forward holds in its cache (one per distinct descriptor, including
 * the tensor addresses).  A net that changes input size adds its convolutions' plans once per new shape; the cache is
 * emptied when it reaches 4096 entries. */
MSCNN_API int mscnn_conv_plan_count(void);

/* Weight packing (done once at load time; replaces nothing in the reference -- Caffe keeps
 * [Cout][Cin][KH][KW] fp32, blob layout base_conv_layer.cpp:135-142).
 *   conv: w_f32 [Cout][Cin][KH][KW] -> planes [Cout_pad][KH][KW][Cin_pad], zero padded.
 *   fc  : w_f32 [Nout][C*H*W] (Caffe flattening c*H*W + h*W + w, inner_product_layer.cpp:32-48)
 *         -> planes [Nout_pad][(h*W + w)*Cpad + c], the NHWC flattening of the bottom. */
MSCNN_API int mscnn_pack_conv_weights(const float* w_f32, void* w_hi, void* w_lo, int Cout, int Cin, int KH,
                            int KW, int Cout_pad, int Cin_pad, void* stream);
MSCNN_API int mscnn_pack_fc_weights(const float* w_f32, void* w_hi, void* w_lo, int Nout, int C, int H, int W,
                          int Nout_pad, int Cpad, void* stream);

/* ------------------------------------------------------------------------------------
 * Deconvolution (transposed convolution) with any kernel, stride, pad, dilation and group whose channels are 64-aligned,
 * with fused bias and optional ReLU.  Replaces DeconvolutionLayer::Forward_gpu (src/caffe/layers/deconv_layer.cu,
 * deconv_layer.cpp:25-40: col2im of w^T x, then the bias) for every layer but the depthwise ones
 * (mscnn_deconv_depthwise_forward).
 *   The descriptor is the convolution's: KH, KW, pad_*, stride_*, dil_*, group are the Deconvolution's parameters,
 *   N, H, W, C the input planes [N][H][W][C] (C % 64 == 0), w_* the planes of mscnn_pack_deconv_weights, bias fp32
 *   [Cout_pad], y planes [N][Ho][Wo][Cout_pad] (Cout_pad % 64 == 0, out_mode MSCNN_OUT_NHWC_BF16), with
 *   Ho = stride_h (H - 1) + dil_h (KH - 1) + 1 - 2 pad_h, Wo likewise (deconv_layer.cpp:8-22):
 *     y[n][i stride_h - pad_h + ky dil_h][j stride_w - pad_w + kx dil_w][co] += x[n][i][j][ci] w[ci][co][ky][kx].
 *   The output is computed by phase (ho mod stride_h, wo mod stride_w): each phase is a stride-1 convolution with its
 *   own sub-kernel, signed pad and extent, one conv_igemm_kernel launch writing that phase's pixels; a phase no tap
 *   reaches holds the bias (plus ReLU).  The sums run in the convolution kernel's K order, not col2im's.
 *   group = g > 1: C / g and Cout / g must be multiples of 64 and Cout_pad == Cout.
 *   Served: strides 1..8, pad >= 0, dilation >= 1, pad and dilated kernel reach up to 2^20, a positive output extent;
 *   pool_*, y_f32 and dyn_n unused (NULL).  Anything else returns MSCNN_ERR_INVALID with a message on stderr and
 *   writes nothing. */
MSCNN_API int mscnn_deconv_forward(const mscnn_conv_desc* d, void* stream);
/* Host-only: one line per output phase, in (r_h, r_w) row-major order,
 *   "phase=<r_h>x<r_w> taps=<m_h>x<m_w> dil=<d_h>x<d_w> pad=<P_h>x<P_w> out=<Q_h>x<Q_w> plan=<plan>\n"
 * with the sub-convolution's taps, dilation, signed pad and extent, and as <plan> the mscnn_conv_plan_describe text of
 * its launch, "bias_fill" where no tap reaches the phase or "none" where it has no output pixel.  No CUDA call. */
MSCNN_API int mscnn_deconv_plan_describe(const mscnn_conv_desc* d, char* buf, int cap);
/* Weight packing for mscnn_deconv_forward: the Caffe blob [Cin][Cout / group][KH][KW] (deconv blob layout,
 * base_conv_layer.cpp:135-142 with the channel axes reversed) -> every phase's sub-kernel, phases (r_h, r_w) in row-major
 * order, each [Cout_pad][m_h][m_w][cin_g] (mscnn_pack_conv_weights' layout; cin_g = Cin / group padded to 64), taps
 * reversed.  mscnn_deconv_packed_elems (host-only): elements of one plane (w_hi or w_lo), -1 for a geometry not served. */
MSCNN_API long long mscnn_deconv_packed_elems(int Cin, int Cout, int group, int KH, int KW, int stride_h, int stride_w,
                                              int pad_h, int pad_w, int dil_h, int dil_w, int Cout_pad);
MSCNN_API int mscnn_pack_deconv_weights(const float* w_f32, void* w_hi, void* w_lo, int Cin, int Cout, int group,
                                        int KH, int KW, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                        int dil_w, int Cout_pad, void* stream);

/* conv1_1 as one tensor-core kernel (mscnn_b200/csrc/conv_c3_tc.cu): 3 -> 64 channels, 3x3, pad 1, straight
 * from the fp32 NCHW input blob to NHWC bf16 planes [N][H][W][64] (+ReLU).  Same reference call sites as
 * mscnn_conv_forward (conv_layer.cpp:25-40, relu_layer.cpp:9-19).  The horizontal taps are overlapping views
 * of one staged pixel row, expressed in the wgmma shared-memory descriptor (no im2col tensor, no padded copy).
 * packed_w: mscnn_conv1_tc_packed_bytes() bytes filled by mscnn_pack_conv1_tc_weights from fp32 [64][3][3][3];
 * y_lo == NULL selects the plain bf16 path (pack with split = 0 or 1, the lo plane is simply unused). */
MSCNN_API int mscnn_conv1_tc_packed_bytes(void);
MSCNN_API int mscnn_pack_conv1_tc_weights(const float* w_f32, void* packed, int split, void* stream);
MSCNN_API int mscnn_conv1_tc_forward(const float* x, const void* packed_w, const float* bias64, void* y_hi,
                                     void* y_lo, int N, int H, int W, int relu, void* stream);

/* Narrow-output k x k heads (LFCN_*: Cout = 9, k = 5 / 7).  A direct k x k conv with tiny Cout
 * wastes the tensor core (N = 16..32) and re-reads the activation tile once per tap.  Instead the
 * horizontal taps move into the GEMM's N dimension and only the vertical taps stay in K:
 *   P[pixel][dx*Cout + co] = sum_dy sum_c x[pixel + dy - pad rows][c] * w[co][c][dy][dx]
 *                            (mscnn_conv_forward as a k x 1 conv, pad_w = 0, N = k*Cout -> 64,
 *                             MSCNN_OUT_NHWC_F32)
 *   y[n][co][h][w] = bias[co] + sum_dx P[(n, h, w + dx - pad)][dx*Cout + co]   (mscnn_head_gather)
 * Same FLOPs as the convolution, k instead of k*k activation reads, a 64-column fp32 intermediate;
 * the summation order differs from im2col+sgemm only in fp32 rounding.  Replaces
 * ConvolutionLayer::Forward_gpu for those layers.  mscnn_pack_head_weights writes planes
 * [N_pad][k][1][Cin_pad] with row n = dx*Cout + co. */
MSCNN_API int mscnn_pack_head_weights(const float* w_f32 /*[Cout][Cin][k][k]*/, void* w_hi, void* w_lo, int Cout,
                            int Cin, int k, int N_pad, int Cin_pad, void* stream);
MSCNN_API int mscnn_head_gather(const float* P, int ld, const float* bias, float* y /*[N][Cout][H][W]*/, int N, int H,
                      int W, int Cout, int k, int pad, void* stream);

/* Layout converters between Caffe blobs (NCHW fp32, blob.hpp:153-164) and planes. */
MSCNN_API int mscnn_nchw_f32_to_planes(const float* x, void* hi, void* lo, int N, int C, int H, int W,
                             int Cpad, void* stream);
MSCNN_API int mscnn_planes_to_nchw_f32(const void* hi, const void* lo, float* y, int N, int C, int H, int W,
                             int Cpad, void* stream);

/* ------------------------------------------------------------------------------------
 * Pooling, ceil-mode output size.  Replaces PoolingLayer::Forward_gpu
 * (src/caffe/layers/pooling_layer.cu:158-190; shape pooling_layer.cpp:79-123).
 *   x planes [N][H][W][C] (C % 8 == 0) -> y planes [N][Ho][Wo][C],
 *   mode = MSCNN_POOL_MAX | MSCNN_POOL_AVE (STOCHASTIC is a training mode and is not served).
 * mscnn_pool_output_size (host-only): Ho = ceil((H + 2 pad - kernel) / stride) + 1, one less when pad > 0 and that
 *   last window would start in the bottom / right padding (pooling_layer.cpp:90-105); MSCNN_ERR_INVALID unless
 *   kernel, stride > 0, 0 <= pad < kernel and Ho >= 1.
 * mscnn_pool_forward: square kernel and stride, pad 0.
 * mscnn_pool2d_forward_dyn: every PoolingParameter geometry.  Window (ho, wo) starts at (ho stride_h - pad_h,
 *   wo stride_w - pad_w); MAX ignores padded positions; AVE divides by the window clipped to the padded extent
 *   (pooling_layer.cpp:196-204), so padded positions count as zeros.  global_pooling is kernel = (H, W), stride 1,
 *   pad 0: a single window over at least 32 pixels is reduced by a whole CTA per image and 64 channels.
 *   dyn_n: see below (may be NULL). */
MSCNN_API int mscnn_pool_output_size(int in, int kernel, int stride, int pad);
MSCNN_API int mscnn_pool_forward(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H, int W,
                       int C, int kernel, int stride, int mode, void* stream);
MSCNN_API int mscnn_pool2d_forward_dyn(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H, int W,
                                       int C, int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h,
                                       int pad_w, int mode, const int* dyn_n, void* stream);

/* Data-dependent row counts.  The three per-ROI kernels behind BoxOutput (ROI pooling / ROI align / the pooling
 * that follows ROI align in the cascade nets) and mscnn_conv_desc.dyn_n take an optional DEVICE count: the launch is
 * sized for the cap (N resp. R) and the kernel processes min(cap, *dyn) rows.  The reference knows R on the host at this
 * point because its BoxOutput is host code (box_output_layer.cpp:201); here nothing waits for the device mid-forward. */
MSCNN_API int mscnn_pool_forward_dyn(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int N, int H, int W,
                           int C, int kernel, int stride, int mode, const int* dyn_n, void* stream);
MSCNN_API int mscnn_roi_pool_multi_forward_dyn(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                     const float* rois, int R, int pooled_h, int pooled_w, float spatial_scale,
                                     int num_variants, const float* pad_ratios, const int* out_channel_offsets,
                                     void* y_hi, void* y_lo, int out_channels_total, const int* dyn_R, void* stream);
MSCNN_API int mscnn_roi_align_forward_dyn(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                const float* rois, int R, int pooled_h, int pooled_w, float spatial_scale,
                                float pad_ratio, void* y_hi, void* y_lo, int out_channels_total,
                                int out_channel_offset, const int* dyn_R, void* stream);

/* Stand-alone ReLU (in place) and channel Concat for planes / fp32 blobs.  mscnn_b200's Net fuses
 * ReLU into the producing convolution and Concat into ROIPooling; these serve unfused use.
 * Replace ReLULayer::Forward_gpu (relu_layer.cu:9-26) and ConcatLayer::Forward_gpu
 * (concat_layer.cu:9-46).  count = elements per plane (multiple of 8). */
MSCNN_API int mscnn_relu_planes(void* hi, void* lo, size_t count, void* stream);
MSCNN_API int mscnn_relu_f32(float* x, size_t count, void* stream);
MSCNN_API int mscnn_concat_planes(const void* x, void* y, size_t pixels, int C, int Ctot, int offset, void* stream);

/* Depthwise transposed convolution (group == channels == num_output): DeconvolutionLayer::Forward_gpu
 * (src/caffe/layers/deconv_layer.cu) for those layers, any kernel, stride 1..8, pad >= 0 and dilation >= 1 per axis.
 *   w: fp32 [Creal][1][KH][KW] (layer blob 0), bias: fp32 [Creal] (blob 1) or NULL.
 *   x planes [N][H][W][C] -> y planes [N][Ho][Wo][C], Ho = stride_h (H - 1) + dil_h (KH - 1) + 1 - 2 pad_h, Wo likewise;
 *   channels from Creal up to C are zero.  Each output sums its taps in col2im's increasing (ky, kx) order
 *   (util/im2col.cpp:col2im_cpu), then adds the bias.
 * mscnn_deconv2x_forward: kernel 4 / stride 2 / pad 1 / no bias, the "conv4_3_2x" layer of the -2x nets
 *   (y planes [N][2H][2W][C]). */
MSCNN_API int mscnn_deconv_depthwise_forward(const void* x_hi, const void* x_lo, const float* w, const float* bias,
                                             void* y_hi, void* y_lo, int N, int H, int W, int C, int Creal, int KH,
                                             int KW, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                             int dil_w, void* stream);
MSCNN_API int mscnn_deconv2x_forward(const void* x_hi, const void* x_lo, const float* w, void* y_hi, void* y_lo,
                           int N, int H, int W, int C, int Creal, void* stream);

/* ------------------------------------------------------------------------------------
 * BoxOutput: anchor decode + score, joint top-N over all scales, greedy NMS, outputs.
 * Replaces BoxOutputLayer::Forward_cpu (src/caffe/layers/box_output_layer.cpp:66-234; the
 * reference has no GPU version) with parameters of BoxOutputParameter / BBoxRegParameter
 * (src/caffe/proto/caffe.proto:1315-1329,1346-1350).
 *   maps[j]        : fp32 [N][channels][height[j]][width[j]], channels = cls_num + 4
 *   proposals      : fp32 [rows][5] = [img x1 y1 x2 y2]      (top[0]), capacity N*max_nms_num rows
 *   proposals_score: fp32 [rows][6] = [... score] (top[1]) or NULL
 *   num_out (device int[2+N]): [0] rows in the blobs (>= 1: a dummy ROI [0 1 1 10 10] / zero
 *                  row is emitted when nothing survives, :195-199,214-218), [1] true proposal
 *                  count, [2+n] proposals of image n.
 * max_nms_num must be in 1..8192 (the reference's 0 = "unbounded" is not supported on device). */
typedef struct mscnn_box_output_cfg {
  int num_scales;
  int channels;
  int height[MSCNN_MAX_SCALES], width[MSCNN_MAX_SCALES];
  float field_w[MSCNN_MAX_SCALES], field_h[MSCNN_MAX_SCALES], downsample_rate[MSCNN_MAX_SCALES];
  float fg_thr, iou_thr;
  int nms_type; /* MSCNN_NMS_* */
  float field_whr, field_xyr, min_size;
  int max_nms_num, max_post_nms_num;
  int do_bbox_norm;
  float bbox_mean[4], bbox_std[4];
} mscnn_box_output_cfg;
MSCNN_API int mscnn_box_output_workspace_bytes(const mscnn_box_output_cfg* cfg, int N, size_t* bytes);
MSCNN_API int mscnn_box_output_forward(const mscnn_box_output_cfg* cfg, int N, const float* const* maps /*host array*/,
                             void* workspace, size_t workspace_bytes, float* proposals,
                             float* proposals_score, int* num_out, void* stream);

/* ------------------------------------------------------------------------------------
 * ROIPooling with the MS-CNN pad_ratio context extension, writing at a channel offset of a wider
 * output so that org || ctx are concatenated in place.  Replaces ROIPoolingLayer::Forward_gpu
 * (src/caffe/layers/roi_pooling_layer.cu:19-104; CPU semantics roi_pooling_layer.cpp:49-139) and
 * ConcatLayer::Forward_gpu (concat_layer.cu:28-46).
 *   x planes [N][H][W][C]; rois fp32 [R][5] = [img x1 y1 x2 y2];
 *   y planes [R][pooled_h][pooled_w][out_channels_total], channels [offset, offset + C). */
MSCNN_API int mscnn_roi_pool_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                           const float* rois, int R, int pooled_h, int pooled_w, float spatial_scale,
                           float pad_ratio, void* y_hi, void* y_lo, int out_channels_total,
                           int out_channel_offset, void* stream);

/* Same, for up to 4 pad_ratio variants of one ROI set in a single launch (MS-CNN's object + context
 * pooling): variant i is written at channel offset out_channel_offsets[i] of y. */
MSCNN_API int mscnn_roi_pool_multi_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                                 const float* rois, int R, int pooled_h, int pooled_w, float spatial_scale,
                                 int num_variants, const float* pad_ratios, const int* out_channel_offsets,
                                 void* y_hi, void* y_lo, int out_channels_total, void* stream);

/* ------------------------------------------------------------------------------------
 * ROIAlign (cascade WIDER-face nets): bilinear samples on the (pooled_h+1) x (pooled_w+1) grid of bin
 * corners of each (pad_ratio-extended) ROI.  Replaces ROIAlignLayer::Forward_gpu
 * (src/caffe/layers/roi_align_layer.cu:21-98; CPU semantics roi_align_layer.cpp:49-139).
 *   x planes [N][H][W][C]; rois fp32 [R][5];
 *   y planes [R][pooled_h+1][pooled_w+1][out_channels_total], channels [offset, offset + C). */
MSCNN_API int mscnn_roi_align_forward(const void* x_hi, const void* x_lo, int N, int H, int W, int C,
                            const float* rois, int R, int pooled_h, int pooled_w, float spatial_scale,
                            float pad_ratio, void* y_hi, void* y_lo, int out_channels_total,
                            int out_channel_offset, void* stream);

/* ------------------------------------------------------------------------------------
 * Per-ROI layers of the cascade deploy nets, all on NCHW fp32 device arrays.
 * DecodeBBox: replaces DecodeBBoxLayer::Forward_cpu (src/caffe/layers/decode_bbox_layer.cpp:53-124, CPU
 *   only in the reference) + DecodeBBoxesWithPrior (src/caffe/util/math_functions.cpp:46-77), TEST
 *   phase: out[i] = [img, x1, y1, x2, y2] = prior[i] moved by the class-1 deltas bbox_pred[i][4..8).
 *   mean4 / std4 may be NULL (0 / 1, decode_bbox_layer.cpp:33-35).
 * Softmax: replaces SoftmaxLayer::Forward_cpu (softmax_layer.cpp:28-62) over `channels` with
 *   `outer` x `inner` independent positions.
 * Eltwise: replaces EltwiseLayer::Forward_cpu (eltwise_layer.cpp:46-96); `bottoms` is a HOST array
 *   of 2..MSCNN_MAX_ELTWISE device pointers, coeffs (host, SUM only) may be NULL (all 1). */
#define MSCNN_MAX_ELTWISE 8
#define MSCNN_ELTWISE_PROD 0
#define MSCNN_ELTWISE_SUM 1
#define MSCNN_ELTWISE_MAX 2
MSCNN_API int mscnn_decode_bbox_forward(const float* bbox_pred, const float* prior, int R, int bbox_dim,
                              const float* mean4, const float* std4, float* out, void* stream);
MSCNN_API int mscnn_softmax_forward(const float* x, int outer, int channels, int inner, float* y, void* stream);
MSCNN_API int mscnn_eltwise_forward(const float* const* bottoms, int num_bottoms, int op, const float* coeffs,
                          size_t count, float* y, void* stream);

/* ------------------------------------------------------------------------------------
 * Final detections for one class: softmax probability, bbox-delta decode, clip, greedy NMS.
 * Replaces the MATLAB code after net.forward in the reference driver
 * (examples/kitti_car/run_mscnn_detection.m:75-120, utils/bbNms.m:112-126).
 *   proposals_score [R][6], cls_pred [R][num_cls], bbox_pred [R][4*num_cls], num_rois = the
 *   num_out array written by mscnn_box_output_forward (per-image row ranges).
 *   dets fp32 [N][max_rois_per_image][5] = [x y w h prob] in kept order; det_counts int[N]. */
typedef struct mscnn_detect_cfg {
  int num_cls;
  int cls_id; /* 1-based, 2 = car in the KITTI nets */
  float bbox_mean[4], bbox_std[4];
  float proposal_thr; /* -10 */
  float nms_overlap;  /* 0.5 */
  float ratio_h, ratio_w; /* net input size / original image size */
  float org_h, org_w;
  int max_rois_per_image; /* 1..8192 */
} mscnn_detect_cfg;
MSCNN_API int mscnn_detect_workspace_bytes(const mscnn_detect_cfg* cfg, int N, size_t* bytes);
MSCNN_API int mscnn_detect_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                             const float* cls_pred, const float* bbox_pred, const int* num_rois,
                             void* workspace, size_t workspace_bytes, float* dets, int* det_counts,
                             void* stream);
/* Batches of images with different ORIGINAL sizes (all resized to the one net input).  The reference drivers handle
 * one frame at a time and rescale / clip its detections with that frame's own ratios
 * (examples/kitti_car/run_mscnn_detection.m:64-65 and :111-116, run_cascademscnn.m:77-80 and :101-105); the *_sized
 * entries take them per image instead of from the cfg:
 *   geom: HOST float [N][4] = ratio_h, ratio_w, org_h, org_w of each image (every value > 0, finite); the cfg's four
 *   geometry fields are ignored.  Image n's result equals bit for bit the cfg entry's with image n's four values.
 * mscnn_detect_image_geometry (host-only, no CUDA call): geom from the net input size and the original sizes
 *   org_hw [N][2] = h, w: ratio = (float)((double)net / (double)org), org = (float)org, the values the MATLAB drivers
 *   compute (run_mscnn_detection.m:65). */
MSCNN_API int mscnn_detect_image_geometry(int net_h, int net_w, int N, const int* org_hw, float* geom);
MSCNN_API int mscnn_detect_postprocess_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                             const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                             void* workspace, size_t workspace_bytes, float* dets, int* det_counts,
                                             const float* geom, void* stream);

/* The drivers' proposal list (examples/kitti_car/run_mscnn_detection.m:75-91, the same lines in kitti_ped_cyc, caltech
 * :83-96, widerface :96-109), on the device: for image n, the rows of BoxOutput's proposals_score [R][6] (num_rois:
 * its DEVICE row counts, read as the post-process reads them, so a lazy row count needs no host wait) with
 * w = x2 - x1, h = y2 - y1 in single, kept iff score >= cfg->proposal_thr && w != 0 && h != 0 (single compares; a NaN
 * score is dropped), in row order, written as float64 props[n][k] = [x y w h score] with x and w divided by
 * (double)net_w / org_w and y and h by (double)net_h / org_h in double, without clipping.  counts[n] = rows kept.
 * cap = cfg->max_rois_per_image; props is [N][cap][5].  org_hw: HOST int [N][2] = h, w per image, or NULL for
 * cfg->org_h / org_w.  Reads cfg->proposal_thr, max_rois_per_image and (org_hw NULL) org_h, org_w only.  An image
 * with more kept rows than cap gets counts[n] = -1 (mscnn_net_proposals refuses such a cap before any launch). */
MSCNN_API int mscnn_proposals_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                          const int* num_rois, int net_h, int net_w, const int* org_hw, double* props,
                                          int* counts, void* stream);

/* Packed output of the same post-process, for the multi-GPU exchange below: `payload` (device,
 * mscnn_detect_payload_floats(N, max_rois_per_image) floats) = int32 header [N, total, counts[0..N)] padded to a
 * multiple of 4 words, then the kept rows of all N images back to back, [total][5] = [x y w h prob] in image order. */
MSCNN_API size_t mscnn_detect_payload_floats(int N, int max_rois_per_image);
MSCNN_API int mscnn_detect_postprocess_packed(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                    const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                    void* workspace, size_t workspace_bytes, float* payload, void* stream);
/* Per-image geometry as in mscnn_detect_postprocess_sized (run_mscnn_detection.m:111-116). */
MSCNN_API int mscnn_detect_postprocess_packed_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                                    const float* cls_pred, const float* bbox_pred, const int* num_rois,
                                                    void* workspace, size_t workspace_bytes, float* payload,
                                                    const float* geom, void* stream);

/* Cascade variant: replaces the MATLAB code after net.forward in examples/kitti_car/run_cascademscnn.m:99-126
 * (+ utils/bbNms.m:112-126).  The net already holds decoded boxes and probabilities:
 *   proposals [R][5] (the stage's ROIs: rows whose width or height is 0 are dropped), cls_prob [R][num_cls]
 *   (Softmax output), output_bbox [R][5] (DecodeBBox output).  Boxes are rescaled by ratio_*, clipped to
 *   [0, org_*], converted to [x y w h] with w = x2 - x1 + 1, and NMS'ed; cfg->bbox_mean/std and
 *   proposal_thr are unused.  Same workspace size and outputs as mscnn_detect_postprocess. */
MSCNN_API int mscnn_cascade_detect_postprocess(const mscnn_detect_cfg* cfg, int N, const float* proposals,
                                     const float* cls_prob, const float* output_bbox, const int* num_rois,
                                     void* workspace, size_t workspace_bytes, float* dets, int* det_counts,
                                     void* stream);
/* Per-image geometry as in mscnn_detect_postprocess_sized (run_cascademscnn.m:77-80, :101-105). */
MSCNN_API int mscnn_cascade_detect_postprocess_sized(const mscnn_detect_cfg* cfg, int N, const float* proposals,
                                                     const float* cls_prob, const float* output_bbox,
                                                     const int* num_rois, void* workspace, size_t workspace_bytes,
                                                     float* dets, int* det_counts, const float* geom, void* stream);

/* Final detections for several classes in one post-process, as the KITTI pedestrian / cyclist driver loops over
 * cls_ids = [2 3] (examples/kitti_ped_cyc/run_mscnn_detection.m:48,93-121), with the WIDER drivers' detection
 * threshold (examples/widerface/run_mscnn_detection.m:139-143: keep prob >= det_thr before bbNms when det_thr > 0).
 * The pipeline runs over N x num_ids slots, slot n * num_ids + c = image n with class cls_ids[c]; each slot's result
 * equals bit for bit the single-class entry's with cls_id = cls_ids[c] (and, with det_thr > 0, that result without its
 * rows of prob < det_thr: greedy NMS only lets a box suppress lower-ranked ones).
 *   dets fp32 [N][num_ids][max_rois_per_image][5], det_counts int[N][num_ids]; geom NULL (the cfg's ratio_* / org_*)
 *   or HOST [N][4] as in the *_sized entries.  cfg->cls_id is ignored.
 *   _packed: the payload layout above over N * num_ids slots, mscnn_detect_payload_floats(N * num_ids, cap) floats.
 *   Workspace: mscnn_detect_classes_workspace_bytes (= the single-class plan of N * num_ids images).
 * Every argument is checked on the host before any CUDA call: num_ids outside 1..MSCNN_MAX_DETECT_CLASSES, an id
 * outside 1..cfg->num_cls, repeated ids, a non-finite det_thr or N outside 1..1024 return MSCNN_ERR_INVALID. */
#define MSCNN_MAX_DETECT_CLASSES 8
typedef struct mscnn_detect_classes {
  int num_ids;                           /* 1..MSCNN_MAX_DETECT_CLASSES */
  int cls_ids[MSCNN_MAX_DETECT_CLASSES]; /* 1-based, distinct, each <= cfg->num_cls; output order = this order */
  float det_thr;                         /* > 0: keep prob >= det_thr before NMS; <= 0: off (the drivers' -1) */
} mscnn_detect_classes;
MSCNN_API int mscnn_detect_classes_workspace_bytes(const mscnn_detect_cfg* cfg, int N,
                                                   const mscnn_detect_classes* classes, size_t* bytes);
MSCNN_API int mscnn_detect_postprocess_classes(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, int N,
                                               const float* proposals_score, const float* cls_pred,
                                               const float* bbox_pred, const int* num_rois, void* workspace,
                                               size_t workspace_bytes, float* dets, int* det_counts,
                                               const float* geom, void* stream);
MSCNN_API int mscnn_cascade_detect_postprocess_classes(const mscnn_detect_cfg* cfg,
                                                       const mscnn_detect_classes* classes, int N,
                                                       const float* proposals, const float* cls_prob,
                                                       const float* output_bbox, const int* num_rois, void* workspace,
                                                       size_t workspace_bytes, float* dets, int* det_counts,
                                                       const float* geom, void* stream);
MSCNN_API int mscnn_detect_postprocess_classes_packed(const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                                      int N, const float* proposals_score, const float* cls_pred,
                                                      const float* bbox_pred, const int* num_rois, void* workspace,
                                                      size_t workspace_bytes, float* payload, const float* geom,
                                                      void* stream);

/* ------------------------------------------------------------------------------------
 * Image pre-processing (the step in front of the path, SURVEY.md 8(f)-3).  Replaces the MATLAB code
 * before net.forward in examples/kitti_car/run_mscnn_detection.m:64-69 and
 * examples/widerface/run_mscnn_detection.m:70-86:
 *   imresize(uint8 image, [out_h out_w]) (bicubic, antialiased, uint8 result) -> channel order [3 2 1]
 *   (RGB -> BGR) -> single -> minus mean [104 117 123] -> W-fastest planes = the net's `data` blob.
 * images: uint8 [N][in_h][in_w][3] interleaved (what an image decoder returns), all N of one size;
 * data: fp32 [N][3][out_h][out_w].  mean[] is indexed by OUTPUT channel (after the swap).
 * A plan has one output size, mean and channel order.  It caches the fp64 tap tables of every input size it has
 * seen on the device (built once per distinct size); the size it was created with is the first. */
typedef struct mscnn_preprocess_desc {
  int in_h, in_w;   /* original image */
  int out_h, out_w; /* net input */
  float mean[3];
  int swap_rb; /* 1: input is RGB (imread), output BGR as the reference nets expect */
} mscnn_preprocess_desc;
MSCNN_API int mscnn_preprocess_create(const mscnn_preprocess_desc* d, void** plan);
MSCNN_API int mscnn_preprocess_destroy(void* plan);
MSCNN_API int mscnn_preprocess_get_desc(void* plan, mscnn_preprocess_desc* d);
MSCNN_API int mscnn_preprocess_forward(void* plan, int N, const unsigned char* images /*device*/, float* data,
                                       void* stream);
/* Same with HOST images: one async H2D copy of the ORIGINAL uint8 pixels into a staging buffer owned by
 * the plan (pinned host memory makes it asynchronous), then the kernels. */
MSCNN_API int mscnn_preprocess_forward_host(void* plan, int N, const unsigned char* host_images, float* data,
                                            void* stream);
/* Images of different original sizes in one batch, all resized to the plan's output size.  The reference reads each
 * frame's size inside its loop (examples/kitti_car/run_mscnn_detection.m:64-65, run_cascademscnn.m:77-80).
 *   in_hw: HOST int [N][2] = h, w of each image (>= 1); images packed back to back in batch order, image n starting
 *   at byte sum_{m<n} h_m * w_m * 3.  Each slot of `data` equals the result of a plan made for that image's size.
 *   A size the plan has not seen yet builds and uploads its tap tables first (synchronous, once per size).
 * _host: the same with HOST images, one async H2D copy into the plan's staging buffer. */
MSCNN_API int mscnn_preprocess_forward_sized(void* plan, int N, const int* in_hw, const unsigned char* images,
                                             float* data, void* stream);
MSCNN_API int mscnn_preprocess_forward_sized_host(void* plan, int N, const int* in_hw,
                                                  const unsigned char* host_images, float* data, void* stream);
/* Grayscale frames ([h][w] or [h][w][1] uint8, as imread returns them) beside colour ones, in any mix and sizes.  The
 * cascade drivers repmat a gray frame to three channels (examples/kitti_car/run_cascademscnn.m:76,
 * examples/citypersons/run_cascademscnn.m:82); slot n of `data` equals bit for bit the result for that repmat'ed frame.
 *   in_c: HOST int [N] = channels of each image, 1 (gray) or 3 (RGB); NULL = all 3, which is the _sized entry.  Image n
 *   starts at byte sum_{m<n} h_m * w_m * c_m.  Any other channel count returns MSCNN_ERR_INVALID before any CUDA call.
 * A plan's staging and intermediate buffers are rewritten by every call: a call on another stream than the plan's
 * previous one first waits, on the device, for that call's launches (an event the plan records behind them). */
MSCNN_API int mscnn_preprocess_forward_sized_c(void* plan, int N, const int* in_hw, const int* in_c,
                                               const unsigned char* images, float* data, void* stream);
MSCNN_API int mscnn_preprocess_forward_sized_c_host(void* plan, int N, const int* in_hw, const int* in_c,
                                                    const unsigned char* host_images, float* data, void* stream);
/* Host-only helpers (no CUDA call; usable on a GPU-less box):
 * imresize's tap tables for one dimension: returns the tap count P (<= cap_taps) and fills
 * host_weights / host_indices as [out_len][cap_taps] (0-based indices); mscnn_imresize_taps = P alone. */
MSCNN_API int mscnn_imresize_taps(int in_len, int out_len);
MSCNN_API int mscnn_imresize_contributions(int in_len, int out_len, double* host_weights, int* host_indices,
                                           int cap_taps);
/* WIDER FACE net input size: round to multiples of 32, cap the longer side at max_size
 * (examples/widerface/run_mscnn_detection.m:72-80); img_h / img_w = 0 keeps the original size. */
MSCNN_API int mscnn_widerface_net_size(int org_h, int org_w, int img_h, int img_w, int max_size, int* rz_h,
                                       int* rz_w);

/* ------------------------------------------------------------------------------------
 * KITTI result writer / evaluator glue (the step behind the path, SURVEY.md 8(f)-4).  Host-only: plain
 * files in, plain files out, no CUDA call (usable on a GPU-less box), as in the reference, where these are
 * MATLAB scripts and a stand-alone C++ tool.
 *
 * mscnn_kitti_write_det_file: examples/kitti_car/run_mscnn_detection.m:150-161 -- one text row
 *   "img,x,y,w,h,score" per final detection (dlmwrite defaults: ',' and %.5g); host_dets [N][max_rois][5] and
 *   host_counts [N] are HOST copies of mscnn_detect_postprocess's outputs, img = first_image_index + n (1-based
 *   position in the image list).
 * mscnn_kitti_write_labels: examples/kitti_result/writeDetForEval.m:19-95 -- reads up to three such files
 *   (NULL or missing = no detections of that class), and writes <save_dir>/<%06d image id>.txt in the KITTI
 *   label format (x2 = x + w, y2 = y + h, score * score_scale; reference: 1000).
 * mscnn_kitti_evaluate: examples/kitti_result/eval/evaluate_object.cpp (main -> eval): reads
 *   <gt_dir>/<id>.txt and <result_dir>/data/<id>.txt for every id in list_path and writes
 *   <result_dir>/stats_<class>_detection.txt and <result_dir>/plot/<class>_detection.txt byte-identical to the
 *   reference tool (the gnuplot / pdf calls are not reproduced).  ap (may be NULL) receives
 *   [car, pedestrian, cyclist] x [easy, moderate, hard] 11-point AP in percent as writeDetForEval.m:104-108
 *   computes it, or -1 for a class without detections.  Unlike the reference tool, a missing file returns
 *   MSCNN_ERR_INVALID instead of deleting result_dir. */
MSCNN_API int mscnn_kitti_write_det_file(const char* path, int N, const float* host_dets, const int* host_counts,
                                         int max_rois, int first_image_index, int append);
MSCNN_API int mscnn_kitti_write_labels(const char* car_det_file, const char* ped_det_file, const char* cyc_det_file,
                                       const char* list_path, const char* save_dir, double score_scale);
MSCNN_API int mscnn_kitti_evaluate(const char* gt_dir, const char* result_dir, const char* list_path, double* ap);

/* WIDER FACE result files (examples/widerface/run_mscnn_detection.m:177-196, run_cascademscnn.m:165-184), host-only:
 * creates event_dir (and any missing parent) and writes <event_dir>/<image_names[n]>.txt for every image n: the name,
 * the detection count, then one "%d %d %d %d %f" row per detection = x y w h rounded half away from zero (MATLAB
 * round), and the probability.  host_dets [N][max_rois_per_image][5] = [x y w h prob] and host_counts [N] are host
 * copies of a post-process's outputs (one class).  An empty name, a name with '/', a count outside
 * 0..max_rois_per_image or a non-finite value in a kept row returns MSCNN_ERR_INVALID before anything is created. */
MSCNN_API int mscnn_widerface_write_results(const char* event_dir, int N, const char* const* image_names,
                                            const float* host_dets, const int* host_counts, int max_rois_per_image);

/* ------------------------------------------------------------------------------------
 * Net facade: caffe::Net<float> of the Caffe-API mirror (mscnn_b200/csrc/caffe_api) for hosts that
 * cannot include C++ headers.  Mirrors what matcaffe / pycaffe expose of Net
 * (/root/reference/matlab/+caffe/private/caffe_.cpp, python/caffe/_caffe.cpp):
 * create from a deploy prototxt (TEST phase), copy parameters by layer name, set inputs, forward,
 * read any blob in Caffe layout (NCHW fp32).  C++ hosts use caffe::Net directly (INTEGRATION.md).
 * Structural errors (bad prototxt graph, shape mismatch) abort like Caffe's CHECKs. */
MSCNN_API int mscnn_set_device(int device);
MSCNN_API int mscnn_set_stream(void* stream);      /* stream used by all layers of this thread's context */
MSCNN_API int mscnn_set_precision(int bf16);       /* 0: fp32-faithful split-bf16 (default), 1: plain bf16 */
MSCNN_API int mscnn_get_precision(void);
MSCNN_API void* mscnn_net_create(const char* prototxt_path_or_text, int is_path);
MSCNN_API void mscnn_net_destroy(void* net);
MSCNN_API int mscnn_net_num_layers(void* net);
MSCNN_API const char* mscnn_net_layer_name(void* net, int i);
MSCNN_API const char* mscnn_net_layer_type(void* net, int i);
MSCNN_API int mscnn_net_layer_param_string(void* net, int i, char* buf, int cap);
MSCNN_API int mscnn_net_num_params(void* net, const char* layer);
MSCNN_API int mscnn_net_param_shape(void* net, const char* layer, int idx, int* shape4); /* returns #axes */
MSCNN_API int mscnn_net_set_param(void* net, const char* layer, int idx, const float* host, long count);
MSCNN_API int mscnn_net_get_param(void* net, const char* layer, int idx, float* host, long count);
MSCNN_API int mscnn_net_copy_trained(void* net, const char* caffemodel_path); /* Net::CopyTrainedLayersFrom */
/* Net::ShareTrainedLayersWith (net.cpp:682-712, pycaffe's share_with): every parameter blob of `net` whose layer name
 * `other` also has shares `other`'s storage (ShareData); layers `net` lacks are ignored.  Afterwards a write through
 * either net is seen by both, and both read one packed image of each weight, so the second net allocates no weight
 * memory.  The nets may then run forwards concurrently from different host threads, each on its own stream; write
 * parameters only while no forward of a sharing net is in flight.  MSCNN_ERR_INVALID, with the reference's message
 * on stderr and nothing shared, when a layer's blob count or a blob's shape differs, or the nets were created on
 * different devices. */
MSCNN_API int mscnn_net_share_trained_layers(void* net, const void* other);
MSCNN_API int mscnn_net_device(void* net);   /* the device current when the net was created (-1: none) */
MSCNN_API int mscnn_net_num_blobs(void* net);
MSCNN_API const char* mscnn_net_blob_name(void* net, int i);
MSCNN_API int mscnn_net_num_inputs(void* net);
MSCNN_API int mscnn_net_num_outputs(void* net);
MSCNN_API const char* mscnn_net_input_name(void* net, int i);
MSCNN_API const char* mscnn_net_output_name(void* net, int i);
MSCNN_API int mscnn_net_blob_shape(void* net, const char* blob, int* shape4); /* returns #axes */
MSCNN_API int mscnn_net_reshape_blob(void* net, const char* blob, int n, int c, int h, int w);
MSCNN_API int mscnn_net_reshape(void* net);
MSCNN_API int mscnn_net_set_blob(void* net, const char* blob, const float* host, long count);       /* async H2D */
MSCNN_API int mscnn_net_set_blob_device(void* net, const char* blob, const float* dev, long count); /* async D2D */
/* Upload for the NEXT forward while the current one still runs: H2D on a private copy stream that waits (on the
 * device) until the layers reading `blob` in the forward in flight have run; the next mscnn_net_forward waits
 * for the copy.  `host` should be pinned and must stay valid until that forward has been issued. */
MSCNN_API int mscnn_net_set_blob_async(void* net, const char* blob, const float* host, long count);
MSCNN_API int mscnn_net_get_blob(void* net, const char* blob, float* host, long count);             /* D2H + sync */
MSCNN_API const float* mscnn_net_blob_device(void* net, const char* blob);
/* pycaffe's Blob.data (_caffe.cpp binds it to mutable_cpu_data): the host side of a blob, or of parameter blob i of
 * `layer`, NCHW fp32 in the blob's shape, after the net's stream has drained (no queued copy reads or writes it).  The
 * memory is valid until that blob's next reshape.  As with every mutable_* accessor the storage's version changes, so
 * what is written there is uploaded by the next forward that reads the blob, and a weight written there is packed
 * again before the next forward.  NULL for an unknown name or index, and, with mscnn_net_last_error saying why, for a
 * blob released by activation reuse. */
MSCNN_API float* mscnn_net_blob_cpu_data(void* net, const char* blob);
MSCNN_API float* mscnn_net_param_cpu_data(void* net, const char* layer, int i);
/* The blob indices (mscnn_net_blob_name order) layer i reads and writes (Net::bottom_ids / top_ids, pycaffe's
 * _bottom_ids / _top_ids), split blobs included: up to cap of them into ids; returns how many the layer has, or
 * MSCNN_ERR_INVALID for a layer index out of range. */
MSCNN_API int mscnn_net_layer_bottoms(void* net, int i, int* ids, int cap);
MSCNN_API int mscnn_net_layer_tops(void* net, int i, int* ids, int cap);
/* The registered layer types (LayerRegistry::LayerTypeList), in name order, one per line, into buf; returns how many
 * there are, or MSCNN_ERR_INVALID when cap is too small. */
MSCNN_API int mscnn_layer_type_list(char* buf, int cap);
/* uint8 host images -> pre-processing kernels -> the input blob (N, in size and out size from the plan / blob). */
MSCNN_API int mscnn_net_set_input_images(void* net, const char* blob, void* preprocess_plan, int N,
                                         const unsigned char* host_images);
/* Batches of frames with different original sizes (run_mscnn_detection.m:64-65 reads each frame's size; the frames
 * are resized to the one net input size).
 * mscnn_net_set_input_images_sized: mscnn_preprocess_forward_sized_host into the blob, and records in_hw [N][2] as
 *   the original sizes of the images the NEXT forward consumes.
 * mscnn_net_set_input_geometry: records org_hw [N][2] (host) alone, for hosts that resize themselves and fill the
 *   input with mscnn_net_set_blob*; N = 0 or org_hw = NULL clears it.
 * A forward from the first layer turns the recorded sizes into the per-image geometry of its outputs (net size = the
 * input blob's H and W; N must match the input blob) and clears them; without recorded sizes its geometry is "none".
 * mscnn_net_detect, _gather, _push and _cascade rescale and clip with the last forward's per-image geometry when it
 * has one (run_mscnn_detection.m:111-116), with the cfg's ratio_* / org_* otherwise.  So the pipelined order "set
 * batch k + 1, detect batch k" pairs each batch with its own sizes.  mscnn_net_set_input_images drops recorded sizes. */
MSCNN_API int mscnn_net_set_input_images_sized(void* net, const char* blob, void* preprocess_plan, int N,
                                               const int* in_hw, const unsigned char* host_images);
/* The same with gray frames among them: in_c [N] as in mscnn_preprocess_forward_sized_c (NULL = all colour). */
MSCNN_API int mscnn_net_set_input_images_sized_c(void* net, const char* blob, void* preprocess_plan, int N,
                                                 const int* in_hw, const int* in_c, const unsigned char* host_images);
/* Pre-processing of the NEXT forward's frames while the current forward runs: what mscnn_net_set_input_images /
 * _sized_c do (staging copy, both resize passes into the blob, recorded sizes), issued on the net's private copy stream
 * (mscnn_net_copy_stream) exactly as mscnn_net_set_blob_async orders its copy.  That stream first waits, on the device,
 * for the point where the forward in flight has stopped reading `blob` (the whole graph of a replayed forward); the next
 * mscnn_net_forward waits for the work on the device, never on the host.  The recorded sizes are the geometry of that
 * next forward, so "forward k, set k + 1, detect k" pairs each batch with its own sizes.  The blob must already have
 * the batch's shape (N x 3 x out_h x out_w).
 * Who waits for what: the plan's device staging and intermediate buffers are reused in stream order (another stream
 * waits for the plan's previous call, see mscnn_preprocess_forward_sized_c).  host_images is read by the H2D copy on the
 * copy stream: it must stay valid until that copy has run, which a host wait on an event recorded on
 * mscnn_net_copy_stream after this call, or on anything queued behind the next forward, guarantees (pageable memory is
 * copied out before the call returns). */
MSCNN_API int mscnn_net_set_input_images_async(void* net, const char* blob, void* preprocess_plan, int N,
                                               const unsigned char* host_images);
MSCNN_API int mscnn_net_set_input_images_sized_async(void* net, const char* blob, void* preprocess_plan, int N,
                                                     const int* in_hw, const int* in_c,
                                                     const unsigned char* host_images);
/* The copy stream of the *_async entries (a cudaStream_t, created on first use; NULL if it cannot be created). */
MSCNN_API void* mscnn_net_copy_stream(void* net);
MSCNN_API int mscnn_net_set_input_geometry(void* net, int N, const int* org_hw);
MSCNN_API int mscnn_net_forward(void* net, int from_layer, int to_layer); /* inclusive; to < 0 = last */
/* mscnn_net_forward returns with the forward QUEUED on the stream: no layer waits for the device, not even BoxOutput,
 * whose data-dependent row count R stays on the device for the layers behind it (mscnn_conv_desc.dyn_n and the *_dyn
 * entries).  The blobs behind BoxOutput have cap rows until the host asks: every accessor of this facade that returns a
 * shape or a value first waits for the 12-byte count and trims them to R (= mscnn_net_resolve_rows), which is the
 * shape the reference reports (box_output_layer.cpp:201).
 * mscnn_net_set_graph(net, 1): after one eager forward the launches of a whole forward are captured into a CUDA graph
 * and replayed while input shapes, parameter versions, precision and stream stay the same (a non-default stream is
 * required); mscnn_net_graph_replayed tells whether the last forward was a replay. */
MSCNN_API int mscnn_net_resolve_rows(void* net);
MSCNN_API int mscnn_net_set_graph(void* net, int on);
MSCNN_API int mscnn_net_graph_replayed(void* net);
/* Activation reuse (off by default).  With on != 0 the blobs whose lifetimes in a forward do not overlap share one
 * device arena, planned at the first forward after a change of input shapes, precision or keep set.  Net inputs,
 * outputs and the n blobs named in `names` stay outside it and readable; after a forward any other blob whose storage
 * a later blob took is released: its shape stays readable, and mscnn_net_get_blob, mscnn_net_blob_device, the set
 * entries and mscnn_net_detect* on it return MSCNN_ERR_INVALID (NULL) with a message naming the blob, the layer after
 * which its storage is reused and how to keep it (mscnn_net_last_error).  mscnn_net_forward(from > 0, ...) is refused
 * the same way when the range reads a planned blob written before `from`.  A name that is not a blob of the net is
 * refused (MSCNN_ERR_INVALID, nothing changed).  on == 0 gives every blob its own storage back. */
MSCNN_API int mscnn_net_set_activation_reuse(void* net, int on, const char* const* names, int n);
/* Host only (nothing allocated): the arena the plan for the current input shapes and this thread's precision needs,
 * and what its planned blobs take without reuse.  Both 0 with reuse off. */
MSCNN_API int mscnn_net_activation_bytes(void* net, size_t* arena, size_t* unplanned);
/* Host only: the plan, one line per storage (a blob with its Split and in-place tops): "<blob> <bytes> <first>-<last>
 * @<offset>", first and last being the layers of its first write and last read, or "... input|output|kept" for a
 * storage outside the arena.  MSCNN_ERR_INVALID when cap is too small. */
MSCNN_API int mscnn_net_activation_plan_describe(void* net, char* buf, int cap);
/* Planned blobs an eager forward found without their arena storage, or with device storage of their own the plan did
 * not give them (a planning bug; each is logged). */
MSCNN_API unsigned long long mscnn_net_activation_misses(void* net);
/* The message of the last call this net refused with a message ("" if none). */
MSCNN_API const char* mscnn_net_last_error(void* net);
/* Fused groups: the layer that does layer i's work (a Pooling folded into its convolution's epilogue, a sibling
 * ROIPooling pooled by the group's leader), i itself otherwise.  mscnn_net_forward(from, ...) widens `from` back to it. */
MSCNN_API int mscnn_net_fused_producer(void* net, int layer);
MSCNN_API int mscnn_net_set_layer_timing(void* net, int on);
MSCNN_API int mscnn_net_layer_times(void* net, float* ms);                 /* ms per layer, last forward */
MSCNN_API int mscnn_net_num_proposals(void* net, int image);               /* image < 0: whole batch */
MSCNN_API int mscnn_net_detect(void* net, const mscnn_detect_cfg* cfg, float* dets_dev, int* det_counts_dev);
/* cascade nets: the caller names the stage's blobs like run_cascademscnn.m:36-48 does
 * (e.g. "proposals_3rd", "cls_prob_3rd", "output_bbox_3rd"). */
MSCNN_API int mscnn_net_detect_cascade(void* net, const mscnn_detect_cfg* cfg, const char* proposals_blob,
                             const char* cls_prob_blob, const char* output_bbox_blob, float* dets_dev,
                             int* det_counts_dev);
/* Several classes of the last forward in one post-process (mscnn_detect_postprocess_classes): dets_dev
 * [N][num_ids][max_rois_per_image][5], det_counts_dev [N][num_ids], the last forward's per-image geometry applied per
 * slot.  _push: packed over N * num_ids slots into an exchange created with mscnn_detect_payload_floats(N * num_ids,
 * cap) floats per rank (any other size is refused). */
MSCNN_API int mscnn_net_detect_classes(void* net, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                       float* dets_dev, int* det_counts_dev);
MSCNN_API int mscnn_net_detect_cascade_classes(void* net, const mscnn_detect_cfg* cfg,
                                               const mscnn_detect_classes* classes, const char* proposals_blob,
                                               const char* cls_prob_blob, const char* output_bbox_blob,
                                               float* dets_dev, int* det_counts_dev);
MSCNN_API int mscnn_net_detect_push_classes(void* net, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                            void* xchg);
/* mscnn_proposals_postprocess on the last forward's proposals_score, with its per-image original sizes (or cfg's
 * org_h / org_w when it had none) and the net input size, on the net's stream: props_dev [N][max_rois_per_image][5]
 * float64, counts_dev [N].  Refused like mscnn_net_detect* (MSCNN_ERR_INVALID, nothing launched): a cap below what
 * BoxOutput can emit per image, or proposals_score released under activation reuse (mscnn_net_last_error). */
MSCNN_API int mscnn_net_proposals(void* net, const mscnn_detect_cfg* cfg, double* props_dev, int* counts_dev);


/* ------------------------------------------------------------------------------------
 * Multi-GPU exchange (SURVEY.md 8(e)).  The reference has no multi-GPU inference (P2PSync is training-only,
 * src/caffe/parallel.cpp:421-439); images are independent, so batches are sharded by image with no data-path
 * collective, and the ONE exchange is an all-gather of the final detections.  What is mirrored is the reference's
 * threading model: one Caffe context per host thread (src/caffe/common.cpp:13-22) = one communicator rank per host
 * thread (mscnn_comm_init_all, one process) or per process (mscnn_comm_init_rank; the 128-byte id from rank 0's
 * mscnn_comm_get_unique_id travels by whatever the host has: MPI, torch.distributed, a file).
 * NCCL is bound at run time (libnccl.so.2 already in the process, else $MSCNN_NCCL_LIB, else the loader path).
 *
 * mscnn_comm_all_gather: in-place ncclAllGather of `floats_per_rank` floats per rank (rank r's part at
 *   buf_all + r * floats_per_rank, produced on `producer_stream`); it runs on the communicator's own stream behind
 *   the producer's current tail, so the producer continues with the next step while the gather is in flight.
 * mscnn_comm_stream_wait / mscnn_comm_synchronize: order a stream / the host behind the last gather.
 * mscnn_net_detect_gather: mscnn_net_detect in packed form straight into this rank's slot of payload_all
 *   ([nranks][mscnn_detect_payload_floats(N, cap)] floats, device) + the all-gather: one collective per step, the
 *   per-image counts ride in the payload header.  All ranks must use the same N and max_rois_per_image. */
#define MSCNN_COMM_ID_BYTES 128
MSCNN_API int mscnn_comm_nccl_version(void); /* 0 if NCCL cannot be loaded */
MSCNN_API int mscnn_comm_get_unique_id(void* host_id128);
MSCNN_API int mscnn_comm_init_rank(void** comm, int nranks, int rank, const void* host_id128); /* current device */
MSCNN_API int mscnn_comm_init_all(void** comms, int ndev, const int* devices /* NULL = 0..ndev-1 */);
MSCNN_API int mscnn_comm_destroy(void* comm);
MSCNN_API int mscnn_comm_info(void* comm, int* nranks, int* rank, int* device);
MSCNN_API int mscnn_comm_all_gather(void* comm, float* buf_all, size_t floats_per_rank, void* producer_stream);
MSCNN_API int mscnn_comm_stream_wait(void* comm, void* stream);
MSCNN_API int mscnn_comm_synchronize(void* comm);
/* device durations (ms) of the last <= 64 collectives on the communicator's stream, oldest first (each includes the
 * wait for the slowest peer); returns the number written, waits for the last collective */
MSCNN_API int mscnn_comm_gather_times(void* comm, float* host_ms, int cap);
MSCNN_API int mscnn_net_detect_gather(void* net, const mscnn_detect_cfg* cfg, void* comm, float* payload_all);


/* Peer-memory exchange: the same all-gather of the packed final detections WITHOUT a collective kernel.  The
 * post-process kernel of rank r stores its payload directly into slot r of every rank's gather buffer through
 * peer-mapped pointers over NVLink and then publishes the step's sequence number in every rank's flag word; receiving
 * is cuStreamWaitValue32 on the local flags.  No launch, no SM held, no rendezvous (an ncclAllGather kernel spins on
 * its SMs until the slowest peer joins, which stalls one persistent convolution CTA per occupied SM).  This is the default exchange of bench.py; mscnn_net_detect_gather stays as the
 * NCCL baseline.
 *   mscnn_xchg_create: one per rank on its device ([generations][nranks][floats_per_rank] + flags); generations
 *   >= 2 = how many steps the ranks may drift apart (step s uses generation s mod G; a sender reuses a generation only
 *   after every peer has pushed step s - G + 1).  Ranks that must meet every step pay E[max over ranks] of the per-step
 *   jitter per step; with G = 16 they pay it once per 16 steps.
 *   same process (one host thread per GPU): mscnn_xchg_connect_local(all objects);
 *   other processes: mscnn_xchg_ipc_handle -> (host transport) -> mscnn_xchg_open_peer_ipc for every peer.
 *   mscnn_net_detect_push / mscnn_detect_postprocess_push: post-process + push + flags, on the net's / given stream.
 *   mscnn_xchg_wait(x, stream): the stream waits until all ranks' payloads of the last push are in mscnn_xchg_buffer(x)
 *   ([nranks][floats_per_rank]); consume them on that stream before the next push. */
#define MSCNN_XCHG_HANDLE_BYTES 64
MSCNN_API int mscnn_xchg_create(void** xchg, int nranks, int rank, size_t floats_per_rank, int generations);
MSCNN_API int mscnn_xchg_destroy(void* xchg);
MSCNN_API int mscnn_xchg_ipc_handle(void* xchg, void* host_handle64);
MSCNN_API int mscnn_xchg_open_peer_ipc(void* xchg, int peer_rank, const void* host_handle64);
MSCNN_API int mscnn_xchg_connect_local(void** xchgs, int n);
MSCNN_API int mscnn_xchg_info(void* xchg, int* nranks, int* rank, size_t* floats_per_rank);
MSCNN_API const float* mscnn_xchg_buffer(void* xchg);
MSCNN_API int mscnn_xchg_wait(void* xchg, void* stream);
MSCNN_API int mscnn_detect_postprocess_push(const mscnn_detect_cfg* cfg, int N, const float* proposals_score,
                                  const float* cls_pred, const float* bbox_pred, const int* num_rois, void* workspace,
                                  size_t workspace_bytes, void* xchg, void* stream);
MSCNN_API int mscnn_net_detect_push(void* net, const mscnn_detect_cfg* cfg, void* xchg);

#ifdef __cplusplus
}
#endif
#endif /* MSCNN_B200_H_ */
