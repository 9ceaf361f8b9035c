// caffe::Net<Dtype> -- the slice of /root/reference/include/caffe/net.hpp:23-330 that inference
// drivers use (matcaffe caffe_.cpp, pycaffe _caffe.cpp, tools/caffe.cpp `time`): construct from
// a deploy .prototxt, copy trained parameters, reshape, Forward / ForwardFromTo, look blobs and
// layers up by name.  Init follows net.cpp:49-284: legacy-input upgrade, InsertSplits (same
// split layer / blob names as util/insert_splits.cpp), layer creation through LayerRegistry,
// in-place top handling, outputs = unconsumed tops in name order (net.cpp:268-274).
//
// mscnn_b200 additions (all optional, default on): a fusion pass that folds in-place ReLU into
// the producing Convolution / InnerProduct, 2x2 MAX Pooling into the convolution before it, and
// Concat into its ROIPooling producers (set MSCNN_NO_FUSION=1 to disable).  It fixes every fused
// group when the net is built; no layer changes another layer's state during a forward.  Also
// per-layer device timing for `caffe time`-style reports.
#pragma once
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "caffe/blob.hpp"
#include "caffe/common.hpp"
#include "caffe/layer.hpp"
#include "caffe/proto/caffe.pb.h"

namespace caffe {

CAFFE_API void InsertSplits(const NetParameter& param, NetParameter* param_split);
// text-format NetParameter from a string (throws std::runtime_error on syntax errors)
CAFFE_API void proto_text_read_string(const char* text, NetParameter* param);

template <typename Dtype>
class CAFFE_API Net {
 public:
  explicit Net(const NetParameter& param);
  explicit Net(const string& param_file, Phase phase);
  virtual ~Net() {}

  void Init(const NetParameter& param);

  const vector<Blob<Dtype>*>& Forward(Dtype* loss = NULL);
  const vector<Blob<Dtype>*>& ForwardPrefilled(Dtype* loss = NULL) { return Forward(loss); }
  Dtype ForwardFromTo(int start, int end);
  Dtype ForwardFrom(int start) { return ForwardFromTo(start, (int)layers_.size() - 1); }
  Dtype ForwardTo(int end) { return ForwardFromTo(0, end); }
  void Reshape();

  // Trained parameters by layer name (net.cpp:750-785); source = another NetParameter.
  void CopyTrainedLayersFrom(const NetParameter& param);
  // Binary .caffemodel (NetParameter wire format, net.cpp:787-803).
  void CopyTrainedLayersFrom(const string trained_filename);
  // Share other's trained parameters by layer name (net.cpp:682-712): each parameter blob of a layer other also has
  // ShareData's other's blob; layers this net lacks are ignored.  Blob counts and shapes must match.  The storage
  // carries the version and the packed weight images (blob.hpp), so both nets see every write and pack each image
  // once.  Both nets must live on one device (mscnn_b200: the reference has no multi-device case).
  void ShareTrainedLayersWith(const Net* other);
  // mscnn_b200 extension: the message ShareTrainedLayersWith(other) would abort with, or "" when it would succeed.
  string ShareTrainedLayersError(const Net* other) const;
  // mscnn_b200 extension: the device current when the net was built (-1: none), where its storage lives
  int device() const { return device_; }

  inline const string& name() const { return name_; }
  inline const vector<string>& layer_names() const { return layer_names_; }
  inline const vector<string>& blob_names() const { return blob_names_; }
  inline const vector<shared_ptr<Blob<Dtype> > >& blobs() const { return blobs_; }
  inline const vector<shared_ptr<Layer<Dtype> > >& layers() const { return layers_; }
  inline Phase phase() const { return phase_; }
  inline const vector<vector<Blob<Dtype>*> >& bottom_vecs() const { return bottom_vecs_; }
  inline const vector<vector<Blob<Dtype>*> >& top_vecs() const { return top_vecs_; }
  // the blob indices layer i writes / reads (net.hpp:154-165 of the reference)
  inline const vector<int>& top_ids(int i) const {
    CHECK_GE(i, 0) << "Invalid layer id";
    CHECK_LT(i, (int)top_id_vecs_.size()) << "Invalid layer id";
    return top_id_vecs_[i];
  }
  inline const vector<int>& bottom_ids(int i) const {
    CHECK_GE(i, 0) << "Invalid layer id";
    CHECK_LT(i, (int)bottom_id_vecs_.size()) << "Invalid layer id";
    return bottom_id_vecs_[i];
  }
  inline int num_inputs() const { return (int)net_input_blobs_.size(); }
  inline int num_outputs() const { return (int)net_output_blobs_.size(); }
  inline const vector<Blob<Dtype>*>& input_blobs() const { return net_input_blobs_; }
  inline const vector<Blob<Dtype>*>& output_blobs() const { return net_output_blobs_; }
  inline const vector<int>& input_blob_indices() const { return net_input_blob_indices_; }
  inline const vector<int>& output_blob_indices() const { return net_output_blob_indices_; }
  bool has_blob(const string& blob_name) const;
  const shared_ptr<Blob<Dtype> > blob_by_name(const string& blob_name) const;
  bool has_layer(const string& layer_name) const;
  const shared_ptr<Layer<Dtype> > layer_by_name(const string& layer_name) const;

  // mscnn_b200 extension: device time of each layer in the last Forward (ms), measured with
  // CUDA events when enabled -- the `caffe time` protocol (tools/caffe.cpp:380-389) on the device.
  void set_layer_timing(bool on) { time_layers_ = on; }
  const vector<float>& layer_times_ms() const { return layer_ms_; }

  // mscnn_b200 extension: fused groups, fixed by Init.  fused_producer(i) = the layer that does layer i's work when the
  // fusion pass folded i into it (Pooling -> its convolution, ROIPooling -> the leader of its Concat group), else i.
  // A folded Pooling still runs itself in a forward whose extents its convolution cannot pool (epilogue_pools).
  // ForwardFromTo widens `start` back to that producer, so a range may start anywhere without running a consumer on a
  // blob its producer never wrote; fused_group_end(i) = the last layer whose work layer i does.
  int fused_producer(int layer) const { return fused_producer_.empty() ? layer : fused_producer_[layer]; }
  int fused_group_end(int layer) const;
  // mscnn_b200 extension: the last layer that reads blob_name's storage, directly or through a top on it (-1: none)
  int last_reader(const string& blob_name) const;
  // mscnn_b200 extension: data-dependent rows (layer.hpp DynRows).  No layer waits for the device in the middle of a
  // forward: the blobs behind BoxOutput keep cap rows while the kernels read the true count on the device.
  // ResolveRows() waits for the count (a 12-byte copy issued right behind BoxOutput) and trims those blobs' shapes to
  // what the reference reports (box_output_layer.cpp:201).  ForwardFromTo() calls it before returning unless
  // set_lazy_rows(true): then the forward returns with everything merely queued and the host calls ResolveRows()
  // when it next needs a shape (the C facade does so in every accessor).
  void set_lazy_rows(bool on) { lazy_rows_ = on; }
  void ResolveRows();
  void ResolveRowsFor(const string& blob_name);  // only if that blob's shape depends on the pending count
  // Capture the layers of ForwardFromTo(0, last) into a CUDA graph after one eager forward and replay it while
  // nothing it depends on changed (blob shapes, parameter versions, precision, config epoch); off by default.
  void set_graph_mode(bool on) { graph_mode_ = on; }
  bool graph_replayed_last_forward() const { return graph_replayed_; }

  // mscnn_b200 extension: activation reuse (off by default; DESIGN.md "Activation memory plan").  With it on, the
  // storages (storage_blob_) whose lifetimes do not overlap share one device arena, and
  // after a forward a blob whose bytes a later blob took is released: its shape stays readable, its data accessors
  // abort with a message naming it.  Net inputs, outputs and the blobs named in `keep` are never in the arena, so they
  // stay readable.  Every keep name must be a blob of the net.
  void set_activation_reuse(bool on, const vector<string>& keep = vector<string>());
  // the message set_activation_reuse(true, keep) would abort with, or ""
  string ActivationKeepError(const vector<string>& keep) const;
  bool activation_reuse() const { return reuse_; }
  struct ActivationStorage {
    int blob;             // the blob that owns the storage (the others alias it)
    size_t bytes;         // planes hi (+ lo) and NCHW fp32, each rounded up to 256 B
    size_t plane_bytes;   // bytes of one plane (0: no planes)
    bool lo;              // fp32-faithful: a lo plane as well
    int nchw_count;       // fp32 values of the NCHW side (0: none)
    int first, last;      // layers (execution order) of its first write and last read
    long long offset;     // in the arena; -1 = not planned
    string outside;       // why not: "input", "output" or "kept"
    vector<int> members;  // every blob on this storage
    vector<int> touched;  // the layers that read or write it
  };
  struct ActivationPlan {
    vector<ActivationStorage> storages;  // by first write, then blob index
    size_t arena_bytes = 0;     // the arena the planned storages share
    size_t planned_bytes = 0;   // what the planned storages take without reuse
    size_t unplanned_bytes = 0; // the storages outside the arena
  };
  // The plan for the current input shapes and this thread's precision (host only: nothing is allocated); empty with
  // reuse off.
  const ActivationPlan& activation_plan();
  // one line per storage: blob, bytes, first and last layer, offset (or why it is outside the arena)
  string activation_plan_describe();
  // Planned storages an eager forward found off their arena slot, or holding a device buffer of their own the plan
  // did not give them (each is also logged).  A plane request beyond its
  // slot aborts in PlaneStore::reserve instead, before it could allocate.
  unsigned long long activation_misses() const { return activation_misses_; }
  // The message a data accessor of blob_name would abort with, or "" (readable, or no such blob).
  string released_message(const string& blob_name) const;
  // The message ForwardFromTo(start, end) would abort with, or "".  With reuse on, a range that starts after layer 0
  // is refused when it reads a planned storage written before it, unless it continues the forward that just ran up to
  // start - 1 (the C facade splits one forward there to record where the input blob is free).
  string ForwardRangeError(int start, int end);

 protected:
  void AppendTop(const NetParameter& param, const int layer_id, const int top_id,
                 set<string>* available_blobs, map<string, int>* blob_name_to_idx);
  int AppendBottom(const NetParameter& param, const int layer_id, const int bottom_id,
                   set<string>* available_blobs, map<string, int>* blob_name_to_idx);
  void FuseLayers();
  void FusePooling();
  void MarkDynamicRows();
  bool GraphForward(int start, int end);
  string ActivationSignature() const;
  void ComputeActivationPlan(ActivationPlan* plan) const;
  void BeginActivations(int start, int end);
  void EndActivations(int start, int end, bool replayed);
  void DetachActivations();

  string name_;
  Phase phase_;
  vector<shared_ptr<Layer<Dtype> > > layers_;
  vector<string> layer_names_;
  map<string, int> layer_names_index_;
  vector<shared_ptr<Blob<Dtype> > > blobs_;
  vector<string> blob_names_;
  map<string, int> blob_names_index_;
  vector<vector<Blob<Dtype>*> > bottom_vecs_;
  vector<vector<int> > bottom_id_vecs_;
  vector<vector<Blob<Dtype>*> > top_vecs_;
  vector<vector<int> > top_id_vecs_;
  vector<int> net_input_blob_indices_;
  vector<int> net_output_blob_indices_;
  vector<Blob<Dtype>*> net_input_blobs_;
  vector<Blob<Dtype>*> net_output_blobs_;
  bool time_layers_;
  vector<float> layer_ms_;
  vector<int> storage_blob_;    // per blob: the blob whose bytes it is on (itself unless Layer::TopsShareBottom)
  vector<vector<int> > writers_, readers_;  // per blob: the layers with it among their tops / bottoms, in order
  vector<int> fused_producer_;  // per layer: who does its work (itself unless fused away)
  int dyn_box_ = -1;            // index of the BoxOutput layer whose rows are deferred (-1: none / several)
  vector<int> dyn_layers_;      // layers whose row count derives from it, in execution order
  set<string> dyn_blob_names_;  // blobs whose row count derives from it
  bool lazy_rows_ = false;
  int device_ = -1;
  bool graph_mode_ = false, graph_replayed_ = false;
  struct GraphState;
  shared_ptr<GraphState> graph_;
  // activation reuse (set_activation_reuse)
  bool reuse_ = false;
  vector<string> keep_;
  ActivationPlan plan_;
  string plan_signature_;           // what plan_ was made for ("" = nothing)
  string applied_signature_;        // what the blobs' arena storage was set up for
  unsigned long long plan_epoch_ = 0;  // changes whenever blob addresses may have changed (part of the graph signature)
  shared_ptr<void> arena_;          // device memory, grow-only
  size_t arena_capacity_ = 0;
  vector<int> on_arena_;            // blobs given arena storage
  int chain_end_ = -1;              // last layer of the forward in progress (-1: none to continue)
  unsigned long long activation_misses_ = 0;
};

}  // namespace caffe
