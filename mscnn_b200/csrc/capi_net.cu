// C facade over caffe::Net<float> for non-C++ hosts (Python ctypes here; the role matcaffe's MEX
// gateway matlab/+caffe/private/caffe_.cpp and pycaffe's _caffe.cpp play in the reference).
// Lookup failures return MSCNN_ERR_INVALID; structural errors abort like Caffe (LOG(FATAL)).
#include <cstring>
#include <sstream>
#include <string>

#include "caffe/layer_factory.hpp"
#include "caffe/layers/mscnn_layers.hpp"
#include "caffe/net.hpp"
#include "mscnn_b200.h"
#include "xchg.h"

using caffe::Blob;
using caffe::Caffe;
using caffe::Net;

namespace {
struct NetHandle {
  std::shared_ptr<Net<float> > net;
  caffe::BoxOutputLayer<float>* box = nullptr;
  void* det_ws = nullptr;
  size_t det_ws_bytes = 0;
  // asynchronous input upload (mscnn_net_set_blob_async): a copy stream plus two events order the H2D copy
  // of the NEXT forward's input against the layers of the CURRENT forward that still read the blob.
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t input_ready = nullptr, inputs_consumed = nullptr;
  bool pending_input = false, consumed_valid = false, graph_mode = false;
  int pending_consumer = -1;
  // Original image sizes: recorded for the next forward ([N][2], empty = none), and the per-image geometry of the
  // last forward's outputs ([N][4] = ratio_h, ratio_w, org_h, org_w; empty = the detect cfg's scalars).  The
  // geometry belongs to the forward, so "set batch k + 1, then detect batch k" pairs each batch with its own sizes.
  std::vector<int> next_org_hw;
  std::vector<float> geom;
  std::string last_error;  // the message of the last call this net refused (mscnn_net_last_error)
  ~NetHandle() {
    if (det_ws) cudaFree(det_ws);
    if (input_ready) cudaEventDestroy(input_ready);
    if (inputs_consumed) cudaEventDestroy(inputs_consumed);
    if (copy_stream) cudaStreamDestroy(copy_stream);
  }
};
NetHandle* H(void* h) { return static_cast<NetHandle*>(h); }
// A refusal with a message: kept for mscnn_net_last_error and printed, as the other refusals print theirs.
bool refuse(NetHandle* nh, const char* what, const std::string& msg) {
  nh->last_error = msg;  // a check that passes clears the last message
  if (msg.empty()) return false;
  fprintf(stderr, "%s: %s\n", what, msg.c_str());
  return true;
}
// Whether `name` is a blob whose storage activation reuse handed to a later blob (its data is gone).
bool released(NetHandle* nh, const char* what, const char* name) {
  return refuse(nh, what, nh->net->released_message(name));
}
// A synchronous input write issued after an asynchronous upload must land after it (the newer write wins).
int settle_pending(NetHandle* nh) {
  if (!nh->pending_input) return MSCNN_OK;
  nh->pending_input = false;
  return cudaStreamWaitEvent(Caffe::stream(), nh->input_ready, 0) == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}
// The input blob `name` as the destination of plan's pre-processing of N images: it must hold exactly N images of the
// plan's output size.
int images_target(NetHandle* nh, const char* name, void* plan, int N, Blob<float>** dst) {
  nh->net->ResolveRowsFor(name);
  if (!nh->net->has_blob(name)) return MSCNN_ERR_INVALID;
  mscnn_preprocess_desc d;
  if (mscnn_preprocess_get_desc(plan, &d) != MSCNN_OK) return MSCNN_ERR_INVALID;
  Blob<float>* b = nh->net->blob_by_name(name).get();
  if (b->count() != (long)N * 3 * d.out_h * d.out_w) return MSCNN_ERR_INVALID;
  *dst = b;
  return MSCNN_OK;
}
// The same for a synchronous write: a pending asynchronous upload is settled first.
int preprocess_target(NetHandle* nh, const char* name, void* plan, int N, float** dst) {
  Blob<float>* b = nullptr;
  const int rc = images_target(nh, name, plan, N, &b);
  if (rc) return rc;
  if (settle_pending(nh) != MSCNN_OK) return MSCNN_ERR_CUDA;
  *dst = b->mutable_gpu_data();
  return MSCNN_OK;
}
// Asynchronous input writes (mscnn_net_set_blob_async, mscnn_net_set_input_images*_async) go on the net's copy stream,
// which first waits, on the device, for the point where the forward in flight no longer reads the input blob.
int async_begin(NetHandle* nh) {
  if (!nh->copy_stream) {
    if (cudaStreamCreateWithFlags(&nh->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&nh->input_ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&nh->inputs_consumed, cudaEventDisableTiming) != cudaSuccess)
      return MSCNN_ERR_CUDA;
  }
  if (nh->consumed_valid && cudaStreamWaitEvent(nh->copy_stream, nh->inputs_consumed, 0) != cudaSuccess) return MSCNN_ERR_CUDA;
  if (!nh->consumed_valid) {
    // no forward has recorded a consumption point yet: order after everything queued on the net stream
    if (cudaEventRecord(nh->inputs_consumed, Caffe::stream()) != cudaSuccess ||
        cudaStreamWaitEvent(nh->copy_stream, nh->inputs_consumed, 0) != cudaSuccess)
      return MSCNN_ERR_CUDA;
  }
  return MSCNN_OK;
}
// ... and mark the write as the next forward's input: that forward waits for input_ready on the device.
int async_end(NetHandle* nh, const char* name) {
  if (cudaEventRecord(nh->input_ready, nh->copy_stream) != cudaSuccess) return MSCNN_ERR_CUDA;
  nh->pending_input = true;
  nh->pending_consumer = nh->net->last_reader(name);
  return MSCNN_OK;
}
// The post-process inputs of the last forward, as every mscnn_net_detect* entry needs them.
struct DetectInputs {
  int N;
  const float *prop, *cls, *bbox;
  const float* geom;  // per-image geometry of the last forward, NULL when it had none (= the cfg's scalars)
};
// Checks that the box layer and the three input blobs exist and that cfg keeps every proposal, grows the workspace (for
// N x classes->num_ids slots; classes NULL = cfg->cls_id alone) and looks up the last forward's geometry.
int detect_inputs(NetHandle* h, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes, const char* prop,
                  const char* cls, const char* bbox, DetectInputs* in) {
  if (!h || !h->box || !cfg || !prop || !cls || !bbox || !h->net->has_blob(prop) || !h->net->has_blob(cls) ||
      !h->net->has_blob(bbox))
    return MSCNN_ERR_INVALID;
  const int N = h->net->input_blobs()[0]->num();
  // The post-process keeps every proposal of an image (run_mscnn_detection.m:75-120 has no cap): a cfg whose
  // max_rois_per_image is below what BoxOutput can emit would silently drop rows, so it is refused instead.
  if (cfg->max_rois_per_image < h->box->max_rows_per_image()) {
    fprintf(stderr, "mscnn_net_detect: max_rois_per_image = %d < %d proposals an image can carry (BoxOutput max_nms_num / "
            "max_post_nms_num)\n", cfg->max_rois_per_image, h->box->max_rows_per_image());
    return MSCNN_ERR_INVALID;
  }
  size_t need = 0;
  const int rc = classes ? mscnn_detect_classes_workspace_bytes(cfg, N, classes, &need)
                         : mscnn_detect_workspace_bytes(cfg, N, &need);
  if (rc) return rc;
  if (need > h->det_ws_bytes) {
    if (h->det_ws) cudaFree(h->det_ws);
    if (cudaMalloc(&h->det_ws, need) != cudaSuccess) return MSCNN_ERR_NOMEM;
    h->det_ws_bytes = need;
  }
  if (!h->geom.empty() && h->geom.size() != (size_t)4 * N) return MSCNN_ERR_INVALID;
  if (released(h, "mscnn_net_detect", prop) || released(h, "mscnn_net_detect", cls) ||
      released(h, "mscnn_net_detect", bbox))
    return MSCNN_ERR_INVALID;
  in->N = N;
  in->prop = h->net->blob_by_name(prop)->gpu_data();
  in->cls = h->net->blob_by_name(cls)->gpu_data();
  in->bbox = h->net->blob_by_name(bbox)->gpu_data();
  in->geom = h->geom.empty() ? nullptr : h->geom.data();
  return MSCNN_OK;
}
// Whether the net's stream has finished all it was given (a net built without a device has no stream: it holds host
// data only).
bool drained(NetHandle* nh) {
  return nh->net->device() < 0 || cudaStreamSynchronize(Caffe::stream()) == cudaSuccess;
}
int fill_shape(const std::vector<int>& s, int* shape4) {
  for (size_t d = 0; d < s.size() && d < 4; ++d) shape4[d] = s[d];
  return (int)s.size();
}
}  // namespace

extern "C" {

int mscnn_set_precision(int bf16) {
  Caffe::set_precision(bf16 ? Caffe::BF16 : Caffe::FP32_SPLIT);
  return MSCNN_OK;
}
int mscnn_get_precision(void) { return Caffe::precision() == Caffe::BF16 ? 1 : 0; }
int mscnn_set_stream(void* stream) {
  Caffe::set_stream((cudaStream_t)stream);
  return MSCNN_OK;
}
int mscnn_set_device(int device) {
  return cudaSetDevice(device) == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}

void* mscnn_net_create(const char* prototxt, int is_path) {
  mscnn_config_reload();  // the MSCNN_* switches are read when a net is created (and never per launch)
  Caffe::set_mode(Caffe::GPU);
  NetHandle* h = new NetHandle();
  if (is_path) {
    h->net.reset(new Net<float>(std::string(prototxt), caffe::TEST));
  } else {
    caffe::NetParameter np;
    try {
      caffe::proto_text_read_string(prototxt, &np);
    } catch (const std::exception& e) {
      fprintf(stderr, "mscnn_net_create: %s\n", e.what());
      delete h;
      return nullptr;
    }
    np.mutable_state()->set_phase(caffe::TEST);
    h->net.reset(new Net<float>(np));
  }
  for (size_t i = 0; i < h->net->layers().size(); ++i)
    if (caffe::BoxOutputLayer<float>* b = dynamic_cast<caffe::BoxOutputLayer<float>*>(h->net->layers()[i].get()))
      h->box = b;
  // mscnn_net_forward returns with the forward merely queued; every accessor below that needs a shape or a value on
  // the host resolves the data-dependent row count first (Net::ResolveRows)
  h->net->set_lazy_rows(true);
  return h;
}
void mscnn_net_destroy(void* h) { delete H(h); }

int mscnn_net_num_layers(void* h) { return (int)H(h)->net->layers().size(); }
const char* mscnn_net_layer_name(void* h, int i) { return H(h)->net->layer_names()[i].c_str(); }
const char* mscnn_net_layer_type(void* h, int i) { return H(h)->net->layers()[i]->type(); }
// canonical one-line dump of the parameters of layer i that matter for the forward path (used to
// compare a generated prototxt with a shipped one field by field)
int mscnn_net_layer_param_string(void* h, int i, char* buf, int cap) {
  const caffe::LayerParameter& p = H(h)->net->layers()[i]->layer_param();
  std::ostringstream o;
  o << p.name() << "|" << p.type();
  for (int k = 0; k < p.bottom_size(); ++k) o << "|b:" << p.bottom(k);
  for (int k = 0; k < p.top_size(); ++k) o << "|t:" << p.top(k);
  const caffe::ConvolutionParameter& c = p.convolution_param();
  o << "|conv:" << c.num_output() << "," << c.bias_term() << "," << c.group();
  for (int k = 0; k < c.kernel_size_size(); ++k) o << ",k" << c.kernel_size(k);
  for (int k = 0; k < c.pad_size(); ++k) o << ",p" << c.pad(k);
  for (int k = 0; k < c.stride_size(); ++k) o << ",s" << c.stride(k);
  // fillers only matter where no trained weights exist: the fixed bilinear upsampling layer
  if (p.type() == "Deconvolution") o << "," << c.weight_filler().type();
  const caffe::PoolingParameter& q = p.pooling_param();
  o << "|pool:" << (int)q.pool() << "," << q.kernel_size() << "," << q.stride() << "," << q.pad();
  o << "|ip:" << p.inner_product_param().num_output();
  o << "|drop:" << p.dropout_param().dropout_ratio();
  const caffe::ROIPoolingParameter& r = p.roi_pooling_param();
  o << "|roi:" << r.pooled_h() << "," << r.pooled_w() << "," << r.spatial_scale() << "," << r.pad_ratio();
  const caffe::BoxOutputParameter& b = p.box_output_param();
  o << "|box:" << b.fg_thr() << "," << b.iou_thr() << "," << b.nms_type() << "," << b.field_whr() << ","
    << b.field_xyr() << "," << b.max_nms_num() << "," << b.max_post_nms_num() << "," << b.min_size();
  for (int k = 0; k < b.field_w_size(); ++k) o << ",w" << b.field_w(k);
  for (int k = 0; k < b.field_h_size(); ++k) o << ",h" << b.field_h(k);
  for (int k = 0; k < b.downsample_rate_size(); ++k) o << ",d" << b.downsample_rate(k);
  const caffe::BBoxRegParameter& g = p.bbox_reg_param();
  o << "|reg:";
  for (int k = 0; k < g.bbox_mean_size(); ++k) o << "m" << g.bbox_mean(k);
  for (int k = 0; k < g.bbox_std_size(); ++k) o << "s" << g.bbox_std(k);
  o << "|softmax:" << p.softmax_param().axis();
  const caffe::EltwiseParameter& e = p.eltwise_param();
  o << "|elt:" << (int)e.operation();
  for (int k = 0; k < e.coeff_size(); ++k) o << "," << e.coeff(k);
  o << "|share:";
  for (int k = 0; k < p.param_size(); ++k)
    if (!p.param(k).name().empty()) o << k << "=" << p.param(k).name() << ",";
  const std::string s = o.str();
  if ((int)s.size() + 1 > cap) return MSCNN_ERR_INVALID;
  memcpy(buf, s.c_str(), s.size() + 1);
  return MSCNN_OK;
}

int mscnn_net_num_params(void* h, const char* layer) {
  if (!H(h)->net->has_layer(layer)) return MSCNN_ERR_INVALID;
  return (int)H(h)->net->layer_by_name(layer)->blobs().size();
}
int mscnn_net_param_shape(void* h, const char* layer, int idx, int* shape4) {
  if (!H(h)->net->has_layer(layer)) return MSCNN_ERR_INVALID;
  auto& blobs = H(h)->net->layer_by_name(layer)->blobs();
  if (idx < 0 || idx >= (int)blobs.size()) return MSCNN_ERR_INVALID;
  return fill_shape(blobs[idx]->shape(), shape4);
}
int mscnn_net_set_param(void* h, const char* layer, int idx, const float* host, long count) {
  if (!H(h)->net->has_layer(layer)) return MSCNN_ERR_INVALID;
  auto& blobs = H(h)->net->layer_by_name(layer)->blobs();
  if (idx < 0 || idx >= (int)blobs.size() || blobs[idx]->count() != count) return MSCNN_ERR_INVALID;
  memcpy(blobs[idx]->mutable_cpu_data(), host, sizeof(float) * count);
  return MSCNN_OK;
}
// host copy of a parameter blob (count must match)
int mscnn_net_get_param(void* h, const char* layer, int idx, float* host, long count) {
  if (!H(h)->net->has_layer(layer)) return MSCNN_ERR_INVALID;
  auto& blobs = H(h)->net->layer_by_name(layer)->blobs();
  if (idx < 0 || idx >= (int)blobs.size() || blobs[idx]->count() != count) return MSCNN_ERR_INVALID;
  memcpy(host, blobs[idx]->cpu_data(), sizeof(float) * count);
  return MSCNN_OK;
}
int mscnn_net_copy_trained(void* h, const char* caffemodel_path) {
  H(h)->net->CopyTrainedLayersFrom(std::string(caffemodel_path));
  return MSCNN_OK;
}

int mscnn_net_share_trained_layers(void* h, const void* other) {
  if (!h || !other) return MSCNN_ERR_INVALID;
  const Net<float>* src = static_cast<const NetHandle*>(other)->net.get();
  const std::string err = H(h)->net->ShareTrainedLayersError(src);
  if (!err.empty()) {
    fprintf(stderr, "mscnn_net_share_trained_layers: %s\n", err.c_str());
    return MSCNN_ERR_INVALID;
  }
  H(h)->net->ShareTrainedLayersWith(src);
  return MSCNN_OK;
}

int mscnn_net_device(void* h) { return H(h)->net->device(); }

int mscnn_net_num_blobs(void* h) { return (int)H(h)->net->blob_names().size(); }
const char* mscnn_net_blob_name(void* h, int i) { return H(h)->net->blob_names()[i].c_str(); }
int mscnn_net_num_inputs(void* h) { return H(h)->net->num_inputs(); }
int mscnn_net_num_outputs(void* h) { return H(h)->net->num_outputs(); }
const char* mscnn_net_input_name(void* h, int i) {
  return H(h)->net->blob_names()[H(h)->net->input_blob_indices()[i]].c_str();
}
const char* mscnn_net_output_name(void* h, int i) {
  return H(h)->net->blob_names()[H(h)->net->output_blob_indices()[i]].c_str();
}
int mscnn_net_blob_shape(void* h, const char* name, int* shape4) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name)) return MSCNN_ERR_INVALID;
  return fill_shape(H(h)->net->blob_by_name(name)->shape(), shape4);
}
int mscnn_net_reshape_blob(void* h, const char* name, int n, int c, int hh, int w) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name)) return MSCNN_ERR_INVALID;
  H(h)->net->blob_by_name(name)->Reshape(n, c, hh, w);
  return MSCNN_OK;
}
int mscnn_net_reshape(void* h) {
  H(h)->net->ResolveRows();
  H(h)->net->Reshape();
  return MSCNN_OK;
}
// host -> blob (pinned staging inside SyncedMemory; the H2D copy is issued on the net stream)
int mscnn_net_set_blob(void* h, const char* name, const float* host, long count) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name)) return MSCNN_ERR_INVALID;
  Blob<float>* b = H(h)->net->blob_by_name(name).get();
  if (b->count() != count || released(H(h), "mscnn_net_set_blob", name)) return MSCNN_ERR_INVALID;
  if (settle_pending(H(h)) != MSCNN_OK) return MSCNN_ERR_CUDA;
  float* dst = b->mutable_gpu_data();
  return cudaMemcpyAsync(dst, host, sizeof(float) * count, cudaMemcpyHostToDevice, Caffe::stream()) == cudaSuccess
             ? MSCNN_OK
             : MSCNN_ERR_CUDA;
}
// uint8 host images -> device pre-processing -> input blob (run_mscnn_detection.m:64-69 on the device)
int mscnn_net_set_input_images(void* h, const char* name, void* plan, int N, const unsigned char* host_images) {
  float* dst = nullptr;
  const int rc = preprocess_target(H(h), name, plan, N, &dst);
  if (rc) return rc;
  H(h)->next_org_hw.clear();  // these images replace any sized batch set before them
  return mscnn_preprocess_forward_host(plan, N, host_images, dst, Caffe::stream());
}
// The same for images of different original sizes (run_mscnn_detection.m:64-65 reads each frame's size): records
// them as the geometry of the next forward.  in_c: channels per image (1 = gray, 3 = colour), NULL = all colour.
int mscnn_net_set_input_images_sized_c(void* h, const char* name, void* plan, int N, const int* in_hw, const int* in_c,
                                       const unsigned char* host_images) {
  if (N < 1 || !in_hw || !host_images) return MSCNN_ERR_INVALID;
  for (int n = 0; n < N; ++n)
    if (in_hw[2 * n] < 1 || in_hw[2 * n + 1] < 1 || (in_c && in_c[n] != 1 && in_c[n] != 3)) return MSCNN_ERR_INVALID;
  float* dst = nullptr;
  int rc = preprocess_target(H(h), name, plan, N, &dst);
  if (rc) return rc;
  rc = mscnn_preprocess_forward_sized_c_host(plan, N, in_hw, in_c, host_images, dst, Caffe::stream());
  if (rc != MSCNN_OK) return rc;
  H(h)->next_org_hw.assign(in_hw, in_hw + 2 * N);
  return MSCNN_OK;
}
int mscnn_net_set_input_images_sized(void* h, const char* name, void* plan, int N, const int* in_hw,
                                     const unsigned char* host_images) {
  return mscnn_net_set_input_images_sized_c(h, name, plan, N, in_hw, nullptr, host_images);
}
// The pre-processing of the NEXT forward's images while the current one runs: the staging copy and both resize passes
// go on the copy stream, behind the point where the forward in flight has stopped reading the blob; the next
// mscnn_net_forward waits for them on the device.  in_hw NULL = N images of the plan's own size (no recorded sizes).
static int set_input_images_async(void* h, const char* name, void* plan, int N, const int* in_hw, const int* in_c,
                                  const unsigned char* host_images) {
  NetHandle* nh = H(h);
  if (N < 1 || !host_images) return MSCNN_ERR_INVALID;
  if (in_hw)
    for (int n = 0; n < N; ++n)
      if (in_hw[2 * n] < 1 || in_hw[2 * n + 1] < 1 || (in_c && in_c[n] != 1 && in_c[n] != 3)) return MSCNN_ERR_INVALID;
  Blob<float>* b = nullptr;
  int rc = images_target(nh, name, plan, N, &b);
  if (rc) return rc;
  if ((rc = async_begin(nh)) != MSCNN_OK) return rc;
  float* dst = b->mutable_gpu_data();
  rc = in_hw ? mscnn_preprocess_forward_sized_c_host(plan, N, in_hw, in_c, host_images, dst, nh->copy_stream)
             : mscnn_preprocess_forward_host(plan, N, host_images, dst, nh->copy_stream);
  if (rc != MSCNN_OK) return rc;
  if ((rc = async_end(nh, name)) != MSCNN_OK) return rc;
  if (in_hw)
    nh->next_org_hw.assign(in_hw, in_hw + 2 * N);
  else
    nh->next_org_hw.clear();
  return MSCNN_OK;
}
int mscnn_net_set_input_images_async(void* h, const char* name, void* plan, int N, const unsigned char* host_images) {
  return set_input_images_async(h, name, plan, N, nullptr, nullptr, host_images);
}
int mscnn_net_set_input_images_sized_async(void* h, const char* name, void* plan, int N, const int* in_hw,
                                           const int* in_c, const unsigned char* host_images) {
  if (!in_hw) return MSCNN_ERR_INVALID;
  return set_input_images_async(h, name, plan, N, in_hw, in_c, host_images);
}
void* mscnn_net_copy_stream(void* h) {
  NetHandle* nh = H(h);
  if (!nh->copy_stream && async_begin(nh) != MSCNN_OK) return nullptr;
  return nh->copy_stream;
}
int mscnn_net_set_input_geometry(void* h, int N, const int* org_hw) {
  if (N < 0) return MSCNN_ERR_INVALID;
  if (N == 0 || !org_hw) {
    H(h)->next_org_hw.clear();
    return MSCNN_OK;
  }
  for (int n = 0; n < N; ++n)
    if (org_hw[2 * n] < 1 || org_hw[2 * n + 1] < 1) return MSCNN_ERR_INVALID;
  H(h)->next_org_hw.assign(org_hw, org_hw + 2 * N);
  return MSCNN_OK;
}
int mscnn_net_set_blob_device(void* h, const char* name, const float* dev, long count) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name)) return MSCNN_ERR_INVALID;
  Blob<float>* b = H(h)->net->blob_by_name(name).get();
  if (b->count() != count || released(H(h), "mscnn_net_set_blob_device", name)) return MSCNN_ERR_INVALID;
  if (settle_pending(H(h)) != MSCNN_OK) return MSCNN_ERR_CUDA;
  return cudaMemcpyAsync(b->mutable_gpu_data(), dev, sizeof(float) * count, cudaMemcpyDeviceToDevice,
                         Caffe::stream()) == cudaSuccess
             ? MSCNN_OK
             : MSCNN_ERR_CUDA;
}
int mscnn_net_get_blob(void* h, const char* name, float* host, long count) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name)) return MSCNN_ERR_INVALID;
  Blob<float>* b = H(h)->net->blob_by_name(name).get();
  if (b->count() != count || released(H(h), "mscnn_net_get_blob", name)) return MSCNN_ERR_INVALID;
  const float* src = b->gpu_data();
  if (cudaMemcpyAsync(host, src, sizeof(float) * count, cudaMemcpyDeviceToHost, Caffe::stream()) != cudaSuccess)
    return MSCNN_ERR_CUDA;
  return cudaStreamSynchronize(Caffe::stream()) == cudaSuccess ? MSCNN_OK : MSCNN_ERR_CUDA;
}
const float* mscnn_net_blob_device(void* h, const char* name) {
  H(h)->net->ResolveRowsFor(name);
  if (!H(h)->net->has_blob(name) || released(H(h), "mscnn_net_blob_device", name)) return nullptr;
  return H(h)->net->blob_by_name(name)->gpu_data();
}
// pycaffe's Blob.data.  The stream is drained first: the view may be written as soon as it is returned, and an upload
// of its previous contents may still be queued (SyncedMemory uploads from the pinned host side asynchronously).
float* mscnn_net_blob_cpu_data(void* h, const char* name) {
  NetHandle* nh = H(h);
  nh->net->ResolveRowsFor(name);
  nh->last_error.clear();
  if (!nh->net->has_blob(name) || released(nh, "mscnn_net_blob_cpu_data", name)) return nullptr;
  if (settle_pending(nh) != MSCNN_OK) return nullptr;
  float* p = nh->net->blob_by_name(name)->mutable_cpu_data();
  return drained(nh) ? p : nullptr;
}
float* mscnn_net_param_cpu_data(void* h, const char* layer, int i) {
  NetHandle* nh = H(h);
  nh->last_error.clear();
  if (!nh->net->has_layer(layer)) return nullptr;
  auto& blobs = nh->net->layer_by_name(layer)->blobs();
  if (i < 0 || i >= (int)blobs.size()) return nullptr;
  float* p = blobs[i]->mutable_cpu_data();
  return drained(nh) ? p : nullptr;
}
static int copy_ids(const std::vector<int>& v, int* ids, int cap) {
  for (int k = 0; k < (int)v.size() && k < cap; ++k) ids[k] = v[k];
  return (int)v.size();
}
int mscnn_net_layer_bottoms(void* h, int i, int* ids, int cap) {
  if (i < 0 || i >= (int)H(h)->net->layers().size() || (cap > 0 && !ids)) return MSCNN_ERR_INVALID;
  return copy_ids(H(h)->net->bottom_ids(i), ids, cap);
}
int mscnn_net_layer_tops(void* h, int i, int* ids, int cap) {
  if (i < 0 || i >= (int)H(h)->net->layers().size() || (cap > 0 && !ids)) return MSCNN_ERR_INVALID;
  return copy_ids(H(h)->net->top_ids(i), ids, cap);
}
int mscnn_layer_type_list(char* buf, int cap) {
  const std::vector<std::string> types = caffe::LayerRegistry<float>::LayerTypeList();
  std::string s;
  for (const std::string& t : types) s += t + "\n";
  if (!buf || (int)s.size() + 1 > cap) return MSCNN_ERR_INVALID;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int)types.size();
}

// layers [from, to] inclusive; to < 0 = last (Net::ForwardFromTo, net.cpp:544-555)
int mscnn_net_forward(void* h, int from, int to) {
  NetHandle* nh = H(h);
  Net<float>* net = nh->net.get();
  if (to < 0) to = (int)net->layers().size() - 1;
  if (from < 0 || from > to || to >= (int)net->layers().size()) return MSCNN_ERR_INVALID;
  if (refuse(nh, "mscnn_net_forward", net->ForwardRangeError(net->fused_producer(from), to))) return MSCNN_ERR_INVALID;
  if (from == 0) {
    // a forward from the first layer consumes the sizes recorded for it; the net input's H and W are the net size
    const int n = (int)nh->next_org_hw.size() / 2;
    std::vector<float> geom((size_t)4 * n);
    if (n > 0) {
      if (net->input_blobs().empty() || net->input_blobs()[0]->num() != n) return MSCNN_ERR_INVALID;
      const Blob<float>* in = net->input_blobs()[0];
      if (mscnn_detect_image_geometry(in->height(), in->width(), n, nh->next_org_hw.data(), geom.data()) != MSCNN_OK)
        return MSCNN_ERR_INVALID;
    }
    nh->geom.swap(geom);
    nh->next_org_hw.clear();
  }
  if (nh->pending_input) {
    // the upload issued by mscnn_net_set_blob_async must land before the first layer runs
    if (cudaStreamWaitEvent(Caffe::stream(), nh->input_ready, 0) != cudaSuccess) return MSCNN_ERR_CUDA;
    nh->pending_input = false;
  }
  if (!nh->copy_stream) {  // asynchronous uploads never used on this net: nothing to order
    net->ForwardFromTo(from, to);
    return MSCNN_OK;
  }
  if (nh->graph_mode && from == 0 && to == (int)net->layers().size() - 1) {
    // graph replay: one launch for the whole forward; the input blob is free again when it has finished
    net->ForwardFromTo(from, to);
    if (cudaEventRecord(nh->inputs_consumed, Caffe::stream()) != cudaSuccess) return MSCNN_ERR_CUDA;
    nh->consumed_valid = true;
    return MSCNN_OK;
  }
  // Every forward records the point after which the input blob may be overwritten by the next asynchronous upload:
  // right behind the last layer that reads it.
  int c = nh->pending_consumer;
  if (c >= 0) c = net->fused_group_end(net->fused_producer(c));  // never split a fused group
  if (c >= from && c < to) {
    net->ForwardFromTo(from, c);
    if (cudaEventRecord(nh->inputs_consumed, Caffe::stream()) != cudaSuccess) return MSCNN_ERR_CUDA;
    net->ForwardFromTo(c + 1, to);
  } else {
    net->ForwardFromTo(from, to);
    if (cudaEventRecord(nh->inputs_consumed, Caffe::stream()) != cudaSuccess) return MSCNN_ERR_CUDA;
  }
  nh->consumed_valid = true;
  return MSCNN_OK;
}
// host -> blob on a separate copy stream: returns immediately; the copy starts as soon as the layers of the
// forward in flight that read this blob have run, and the next mscnn_net_forward waits for it on the device.
// `host` must stay valid (and should be pinned) until that forward has been issued.
int mscnn_net_set_blob_async(void* h, const char* name, const float* host, long count) {
  H(h)->net->ResolveRowsFor(name);
  NetHandle* nh = H(h);
  Net<float>* net = nh->net.get();
  if (!net->has_blob(name)) return MSCNN_ERR_INVALID;
  Blob<float>* b = net->blob_by_name(name).get();
  if (b->count() != count || released(nh, "mscnn_net_set_blob_async", name)) return MSCNN_ERR_INVALID;
  int rc = async_begin(nh);
  if (rc) return rc;
  float* dst = b->mutable_gpu_data();
  if (cudaMemcpyAsync(dst, host, sizeof(float) * count, cudaMemcpyHostToDevice, nh->copy_stream) != cudaSuccess)
    return MSCNN_ERR_CUDA;
  return async_end(nh, name);
}
// CUDA-graph replay of whole forwards (Net::set_graph_mode): off by default
int mscnn_net_set_graph(void* h, int on) {
  H(h)->graph_mode = on != 0;
  H(h)->net->set_graph_mode(on != 0);
  return MSCNN_OK;
}
int mscnn_net_set_activation_reuse(void* h, int on, const char* const* names, int n) {
  if (!h || n < 0 || (n > 0 && !names)) return MSCNN_ERR_INVALID;
  std::vector<std::string> keep;
  for (int k = 0; k < n; ++k) {
    if (!names[k]) return MSCNN_ERR_INVALID;
    keep.push_back(names[k]);
  }
  if (refuse(H(h), "mscnn_net_set_activation_reuse", H(h)->net->ActivationKeepError(keep))) return MSCNN_ERR_INVALID;
  H(h)->net->set_activation_reuse(on != 0, keep);
  return MSCNN_OK;
}
int mscnn_net_activation_bytes(void* h, size_t* arena, size_t* unplanned) {
  if (!h || !arena || !unplanned) return MSCNN_ERR_INVALID;
  const Net<float>::ActivationPlan& p = H(h)->net->activation_plan();
  *arena = p.arena_bytes;
  *unplanned = p.planned_bytes;
  return MSCNN_OK;
}
int mscnn_net_activation_plan_describe(void* h, char* buf, int cap) {
  if (!h || !buf) return MSCNN_ERR_INVALID;
  const std::string s = H(h)->net->activation_plan_describe();
  if ((int)s.size() + 1 > cap) return MSCNN_ERR_INVALID;
  memcpy(buf, s.c_str(), s.size() + 1);
  return MSCNN_OK;
}
unsigned long long mscnn_net_activation_misses(void* h) { return H(h)->net->activation_misses(); }
const char* mscnn_net_last_error(void* h) { return H(h)->last_error.c_str(); }
int mscnn_net_graph_replayed(void* h) { return H(h)->net->graph_replayed_last_forward() ? 1 : 0; }
// wait for the data-dependent row count of the last forward and trim the blob shapes (every accessor does this)
int mscnn_net_resolve_rows(void* h) {
  H(h)->net->ResolveRows();
  return MSCNN_OK;
}
// the layer that does layer i's work (itself unless the fusion pass folded it away); Net::fused_producer
int mscnn_net_fused_producer(void* h, int layer) {
  if (layer < 0 || layer >= (int)H(h)->net->layers().size()) return MSCNN_ERR_INVALID;
  return H(h)->net->fused_producer(layer);
}
int mscnn_net_set_layer_timing(void* h, int on) {
  H(h)->net->set_layer_timing(on != 0);
  return MSCNN_OK;
}
int mscnn_net_layer_times(void* h, float* ms) {
  const std::vector<float>& t = H(h)->net->layer_times_ms();
  memcpy(ms, t.data(), sizeof(float) * t.size());
  return MSCNN_OK;
}
// proposals of the last forward: total and per image (host values read back by BoxOutput)
int mscnn_net_num_proposals(void* h, int image) {
  H(h)->net->ResolveRows();
  if (!H(h)->box) return MSCNN_ERR_INVALID;
  return image < 0 ? H(h)->box->num_proposals() : H(h)->box->image_proposals(image);
}
// Final detections of the last forward (device outputs): runs mscnn_detect_postprocess on the
// net's proposals_score / cls_pred / bbox_pred blobs.
int mscnn_net_detect(void* hv, const mscnn_detect_cfg* cfg, float* dets_dev, int* det_counts_dev) {
  NetHandle* h = H(hv);
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, nullptr, "proposals_score", "cls_pred", "bbox_pred", &in);
  if (rc) return rc;
  return mscnn::detect_postprocess(false, cfg, nullptr, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(), h->det_ws,
                                   h->det_ws_bytes, in.geom, mscnn::DetectOut::padded(dets_dev, det_counts_dev),
                                   Caffe::stream());
}
// Final detections of this rank's images, packed (header + compacted rows), then ONE all-gather on the communicator's
// stream.  The producer stream first waits for the previous gather (it still reads / writes payload_all).
int mscnn_net_detect_gather(void* hv, const mscnn_detect_cfg* cfg, void* comm, float* payload_all) {
  NetHandle* h = H(hv);
  if (!comm || !payload_all) return MSCNN_ERR_INVALID;
  DetectInputs in;
  int rc = detect_inputs(h, cfg, nullptr, "proposals_score", "cls_pred", "bbox_pred", &in);
  if (rc) return rc;
  int nranks = 0, rank = 0;
  rc = mscnn_comm_info(comm, &nranks, &rank, nullptr);
  if (rc) return rc;
  const size_t per = mscnn_detect_payload_floats(in.N, cfg->max_rois_per_image);
  rc = mscnn_comm_stream_wait(comm, Caffe::stream());
  if (rc) return rc;
  rc = mscnn::detect_postprocess(false, cfg, nullptr, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(), h->det_ws,
                                 h->det_ws_bytes, in.geom, mscnn::DetectOut::packed(payload_all + (size_t)rank * per),
                                 Caffe::stream());
  if (rc) return rc;
  return mscnn_comm_all_gather(comm, payload_all, per, Caffe::stream());
}
// Final detections of this rank packed AND pushed into every rank's gather buffer by the post-process kernel itself
// (peer-memory exchange, xchg.cu): no collective, nothing else to launch.
int mscnn_net_detect_push(void* hv, const mscnn_detect_cfg* cfg, void* xchg) {
  NetHandle* h = H(hv);
  if (!xchg) return MSCNN_ERR_INVALID;
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, nullptr, "proposals_score", "cls_pred", "bbox_pred", &in);
  if (rc) return rc;
  return mscnn::xchg_detect_push(cfg, nullptr, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(), h->det_ws,
                                 h->det_ws_bytes, xchg, in.geom, Caffe::stream());
}
int mscnn_net_detect_cascade(void* hv, const mscnn_detect_cfg* cfg, const char* proposals_blob,
                             const char* cls_prob_blob, const char* output_bbox_blob, float* dets_dev,
                             int* det_counts_dev) {
  NetHandle* h = H(hv);
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, nullptr, proposals_blob, cls_prob_blob, output_bbox_blob, &in);
  if (rc) return rc;
  if (h->net->blob_by_name(cls_prob_blob)->channels() != cfg->num_cls) return MSCNN_ERR_INVALID;
  return mscnn::detect_postprocess(true, cfg, nullptr, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(), h->det_ws,
                                   h->det_ws_bytes, in.geom, mscnn::DetectOut::padded(dets_dev, det_counts_dev),
                                   Caffe::stream());
}
// Several classes of the last forward in one post-process: N x num_ids slots, image-major.  The class set is checked
// before the net is touched.
int mscnn_net_detect_classes(void* hv, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                             float* dets_dev, int* det_counts_dev) {
  size_t unused = 0;
  if (!classes || mscnn_detect_classes_workspace_bytes(cfg, 1, classes, &unused) != MSCNN_OK) return MSCNN_ERR_INVALID;
  NetHandle* h = H(hv);
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, classes, "proposals_score", "cls_pred", "bbox_pred", &in);
  if (rc) return rc;
  return mscnn::detect_postprocess(false, cfg, classes, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(),
                                   h->det_ws, h->det_ws_bytes, in.geom,
                                   mscnn::DetectOut::padded(dets_dev, det_counts_dev), Caffe::stream());
}
int mscnn_net_detect_cascade_classes(void* hv, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                     const char* proposals_blob, const char* cls_prob_blob,
                                     const char* output_bbox_blob, float* dets_dev, int* det_counts_dev) {
  size_t unused = 0;
  if (!classes || mscnn_detect_classes_workspace_bytes(cfg, 1, classes, &unused) != MSCNN_OK) return MSCNN_ERR_INVALID;
  NetHandle* h = H(hv);
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, classes, proposals_blob, cls_prob_blob, output_bbox_blob, &in);
  if (rc) return rc;
  if (h->net->blob_by_name(cls_prob_blob)->channels() != cfg->num_cls) return MSCNN_ERR_INVALID;
  return mscnn::detect_postprocess(true, cfg, classes, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(),
                                   h->det_ws, h->det_ws_bytes, in.geom,
                                   mscnn::DetectOut::padded(dets_dev, det_counts_dev), Caffe::stream());
}
int mscnn_net_detect_push_classes(void* hv, const mscnn_detect_cfg* cfg, const mscnn_detect_classes* classes,
                                  void* xchg) {
  size_t unused = 0;
  if (!classes || !xchg || mscnn_detect_classes_workspace_bytes(cfg, 1, classes, &unused) != MSCNN_OK)
    return MSCNN_ERR_INVALID;
  NetHandle* h = H(hv);
  DetectInputs in;
  const int rc = detect_inputs(h, cfg, classes, "proposals_score", "cls_pred", "bbox_pred", &in);
  if (rc) return rc;
  return mscnn::xchg_detect_push(cfg, classes, in.N, in.prop, in.cls, in.bbox, h->box->num_out_device(), h->det_ws,
                                 h->det_ws_bytes, xchg, in.geom, Caffe::stream());
}
// The proposal list of the last forward.  The original sizes come back from its geometry: org_* there is the
// (float) of the int size, exact for any image size.
int mscnn_net_proposals(void* hv, const mscnn_detect_cfg* cfg, double* props_dev, int* counts_dev) {
  NetHandle* h = H(hv);
  if (!h || !h->box || !cfg || !props_dev || !counts_dev || !h->net->has_blob("proposals_score"))
    return MSCNN_ERR_INVALID;
  // the drivers keep every proposal of an image: a cap below what BoxOutput can emit is refused, as in detect_inputs
  if (cfg->max_rois_per_image < h->box->max_rows_per_image()) {
    refuse(h, "mscnn_net_proposals",
           "max_rois_per_image = " + std::to_string(cfg->max_rois_per_image) + " < " +
               std::to_string(h->box->max_rows_per_image()) +
               " proposals an image can carry (BoxOutput max_nms_num / max_post_nms_num)");
    return MSCNN_ERR_INVALID;
  }
  if (released(h, "mscnn_net_proposals", "proposals_score")) return MSCNN_ERR_INVALID;
  const Blob<float>* in = h->net->input_blobs()[0];
  const int N = in->num();
  if (!h->geom.empty() && h->geom.size() != (size_t)4 * N) return MSCNN_ERR_INVALID;
  std::vector<int> org_hw;
  for (int n = 0; n < (int)h->geom.size() / 4; ++n) {
    org_hw.push_back((int)h->geom[4 * n + 2]);
    org_hw.push_back((int)h->geom[4 * n + 3]);
  }
  return mscnn_proposals_postprocess(cfg, N, h->net->blob_by_name("proposals_score")->gpu_data(),
                                     h->box->num_out_device(), in->height(), in->width(),
                                     org_hw.empty() ? nullptr : org_hw.data(), props_dev, counts_dev, Caffe::stream());
}
}
