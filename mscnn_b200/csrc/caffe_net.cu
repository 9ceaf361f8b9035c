// caffe::Net for the forward path: graph construction (net.cpp:49-284), split insertion
// (util/insert_splits.cpp:13-138), execution (net.cpp:544-555), weight loading by layer name
// (net.cpp:750-803 incl. a protobuf wire-format reader for .caffemodel files).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>

#include "caffe/layers/mscnn_layers.hpp"
#include "caffe/net.hpp"
#include "config.h"
#include "launch_count.h"
#include "proto_text.hpp"

namespace caffe {

// ------------------------------------------------------------------------- InsertSplits
static string SplitLayerName(const string& layer_name, const string& blob_name, const int blob_idx) {
  std::ostringstream s;
  s << blob_name << "_" << layer_name << "_" << blob_idx << "_split";
  return s.str();
}
static string SplitBlobName(const string& layer_name, const string& blob_name, const int blob_idx,
                            const int split_idx) {
  std::ostringstream s;
  s << blob_name << "_" << layer_name << "_" << blob_idx << "_split_" << split_idx;
  return s.str();
}

// Every top that feeds more than one bottom gets a Split layer right after its LAST writer
// (in-place layers count as writers, which is why conv4_3's split is named after relu4_3).
void InsertSplits(const NetParameter& param, NetParameter* out) {
  out->CopyFrom(param);
  out->clear_layer();
  typedef pair<int, int> Idx;  // (layer, top/bottom index)
  map<string, Idx> last_writer;
  map<Idx, Idx> source_of_bottom;
  map<Idx, int> consumers;
  map<Idx, int> next_split;
  for (int i = 0; i < param.layer_size(); ++i) {
    const LayerParameter& lp = param.layer(i);
    for (int j = 0; j < lp.bottom_size(); ++j) {
      map<string, Idx>::iterator it = last_writer.find(lp.bottom(j));
      if (it == last_writer.end())
        LOG(FATAL) << "Unknown bottom blob '" << lp.bottom(j) << "' (layer '" << lp.name() << "', bottom index "
                   << j << ")";
      source_of_bottom[Idx(i, j)] = it->second;
      ++consumers[it->second];
    }
    for (int j = 0; j < lp.top_size(); ++j) last_writer[lp.top(j)] = Idx(i, j);
  }
  for (int i = 0; i < param.layer_size(); ++i) {
    LayerParameter* lp = out->add_layer();
    const int my_idx = out->layer_size() - 1;
    lp->CopyFrom(param.layer(i));
    for (int j = 0; j < lp->bottom_size(); ++j) {
      const Idx src = source_of_bottom[Idx(i, j)];
      if (consumers[src] > 1)
        lp->set_bottom(j, SplitBlobName(param.layer(src.first).name(), lp->bottom(j), src.second, next_split[src]++));
    }
    for (int j = 0; j < lp->top_size(); ++j) {
      const int count = consumers[Idx(i, j)];
      if (count > 1) {
        const string layer_name = lp->name(), blob_name = lp->top(j);
        LayerParameter* sp = out->add_layer();
        sp->Clear();
        sp->add_bottom(blob_name);
        sp->set_name(SplitLayerName(layer_name, blob_name, j));
        sp->set_type("Split");
        for (int k = 0; k < count; ++k) sp->add_top(SplitBlobName(layer_name, blob_name, j, k));
        lp = out->mutable_layer(my_idx);  // add_layer may have reallocated the vector
      }
    }
  }
}

void proto_text_read_string(const char* text, NetParameter* param) {
  proto_text::ReadNetParamsFromString(text, param);
}

// ---------------------------------------------------------------------------------- Net
template <typename Dtype>
Net<Dtype>::Net(const NetParameter& param) : time_layers_(false) {
  Init(param);
}

template <typename Dtype>
Net<Dtype>::Net(const string& param_file, Phase phase) : time_layers_(false) {
  NetParameter param;
  try {
    proto_text::ReadNetParamsFromTextFile(param_file, &param);  // ReadNetParamsFromTextFileOrDie
  } catch (const std::exception& e) {
    LOG(FATAL) << "Failed to parse NetParameter file: " << param_file << ": " << e.what();
  }
  param.mutable_state()->set_phase(phase);
  Init(param);
}

template <typename Dtype>
void Net<Dtype>::Init(const NetParameter& in_param) {
  phase_ = in_param.state().phase();
  if (cudaGetDevice(&device_) != cudaSuccess) {  // no device: host-only inspection (caffe_api.cu SyncedMemory)
    cudaGetLastError();
    device_ = -1;
  }
  NetParameter upgraded;
  upgraded.CopyFrom(in_param);
  proto_text::UpgradeNetInput(&upgraded);  // UpgradeNetAsNeeded: legacy input fields only
  NetParameter param;
  InsertSplits(upgraded, &param);
  name_ = param.name();
  map<string, int> blob_name_to_idx;
  set<string> available_blobs;
  map<string, shared_ptr<Blob<Dtype> > > shared_params;
  const int L = param.layer_size();
  bottom_vecs_.resize(L);
  top_vecs_.resize(L);
  bottom_id_vecs_.resize(L);
  top_id_vecs_.resize(L);
  for (int layer_id = 0; layer_id < L; ++layer_id) {
    // inherit the net phase (net.cpp:87-90)
    if (!param.layer(layer_id).has_phase()) param.mutable_layer(layer_id)->set_phase(phase_);
    const LayerParameter& layer_param = param.layer(layer_id);
    layers_.push_back(LayerRegistry<Dtype>::CreateLayer(layer_param));
    layer_names_.push_back(layer_param.name());
    for (int b = 0; b < layer_param.bottom_size(); ++b)
      AppendBottom(param, layer_id, b, &available_blobs, &blob_name_to_idx);
    for (int t = 0; t < layer_param.top_size(); ++t) {
      AppendTop(param, layer_id, t, &available_blobs, &blob_name_to_idx);
      if (layer_param.type() == "Input") {  // net.cpp:116-120
        const int blob_id = (int)blobs_.size() - 1;
        net_input_blob_indices_.push_back(blob_id);
        net_input_blobs_.push_back(blobs_[blob_id].get());
      }
    }
    layers_[layer_id]->SetUp(bottom_vecs_[layer_id], top_vecs_[layer_id]);
    // Net::AppendParam (net.cpp:448-538): layers whose ParamSpec carries the same non-empty name share
    // one parameter blob (the cascade nets' third-stage ensemble heads, e.g. "roi_c1_w").  The reference
    // makes the later blob ShareData() with the owner's; here the later layer simply holds the owner's
    // Blob, so its version counter (used to re-pack weights lazily) is shared too.  Shapes must match
    // (share_mode STRICT, the default, net.cpp:497-509).
    vector<shared_ptr<Blob<Dtype> > >& layer_blobs = layers_[layer_id]->blobs();
    for (int j = 0; j < (int)layer_blobs.size() && j < layer_param.param_size(); ++j) {
      const string& pname = layer_param.param(j).name();
      if (pname.empty()) continue;
      typename map<string, shared_ptr<Blob<Dtype> > >::iterator owner = shared_params.find(pname);
      if (owner == shared_params.end()) {
        shared_params[pname] = layer_blobs[j];
      } else {
        CHECK(layer_blobs[j]->shape() == owner->second->shape())
            << "Cannot share param '" << pname << "' with layer '" << layer_param.name()
            << "': shape mismatch (" << owner->second->shape_string() << " vs " << layer_blobs[j]->shape_string() << ")";
        layer_blobs[j] = owner->second;
      }
    }
  }
  // remaining available blobs are the outputs, in name order (std::set walk, net.cpp:268-274)
  for (set<string>::iterator it = available_blobs.begin(); it != available_blobs.end(); ++it) {
    net_output_blobs_.push_back(blobs_[blob_name_to_idx[*it]].get());
    net_output_blob_indices_.push_back(blob_name_to_idx[*it]);
  }
  for (size_t i = 0; i < blob_names_.size(); ++i) blob_names_index_[blob_names_[i]] = (int)i;
  for (size_t i = 0; i < layer_names_.size(); ++i) layer_names_index_[layer_names_[i]] = (int)i;
  layer_ms_.assign(layers_.size(), 0.f);
  storage_blob_.resize(blobs_.size());
  writers_.resize(blobs_.size());
  readers_.resize(blobs_.size());
  for (size_t b = 0; b < blobs_.size(); ++b) storage_blob_[b] = (int)b;
  for (int i = 0; i < L; ++i) {
    for (size_t k = 0; k < bottom_id_vecs_[i].size(); ++k) readers_[bottom_id_vecs_[i][k]].push_back(i);
    for (size_t k = 0; k < top_id_vecs_[i].size(); ++k) {
      writers_[top_id_vecs_[i][k]].push_back(i);
      if (layers_[i]->TopsShareBottom(bottom_vecs_[i]))
        storage_blob_[top_id_vecs_[i][k]] = storage_blob_[bottom_id_vecs_[i][0]];
    }
  }
  fused_producer_.resize(layers_.size());
  for (size_t i = 0; i < layers_.size(); ++i) fused_producer_[i] = (int)i;
  if (!std::getenv("MSCNN_NO_FUSION")) {
    FuseLayers();
    if (!std::getenv("MSCNN_NO_POOL_FUSION")) FusePooling();
  }
  if (!std::getenv("MSCNN_SYNC_ROWS")) MarkDynamicRows();
}

// Layers whose row count is BoxOutput's data-dependent R (transitively: any layer with a bottom blob in the set puts
// its tops into the set).  With exactly one BoxOutput layer in the net its rows are deferred (layer.hpp DynRows).
template <typename Dtype>
void Net<Dtype>::MarkDynamicRows() {
  const int L = (int)layers_.size();
  int box = -1, boxes = 0;
  for (int i = 0; i < L; ++i)
    if (dynamic_cast<BoxOutputLayer<Dtype>*>(layers_[i].get())) { box = i; ++boxes; }
  if (boxes != 1) return;
  BoxOutputLayer<Dtype>* b = static_cast<BoxOutputLayer<Dtype>*>(layers_[box].get());
  set<int> dyn_blobs(top_id_vecs_[box].begin(), top_id_vecs_[box].end());
  for (int i = box + 1; i < L; ++i) {
    bool hit = false;
    for (size_t k = 0; k < bottom_id_vecs_[i].size(); ++k) hit |= dyn_blobs.count(bottom_id_vecs_[i][k]) > 0;
    if (!hit) continue;
    dyn_blobs.insert(top_id_vecs_[i].begin(), top_id_vecs_[i].end());
    layers_[i]->set_dyn_rows(b->dyn_rows());
    dyn_layers_.push_back(i);
  }
  b->set_defer_rows(true);
  dyn_box_ = box;
  for (set<int>::iterator it = dyn_blobs.begin(); it != dyn_blobs.end(); ++it) dyn_blob_names_.insert(blob_names_[*it]);
}

template <typename Dtype>
void Net<Dtype>::ResolveRowsFor(const string& blob_name) {
  if (dyn_box_ >= 0 && dyn_blob_names_.count(blob_name)) ResolveRows();
}

template <typename Dtype>
void Net<Dtype>::ResolveRows() {
  if (dyn_box_ < 0) return;
  BoxOutputLayer<Dtype>* b = static_cast<BoxOutputLayer<Dtype>*>(layers_[dyn_box_].get());
  if (!b->rows_pending()) return;
  b->ResolveRows(top_vecs_[dyn_box_]);
  for (size_t k = 0; k < dyn_layers_.size(); ++k) {
    const int i = dyn_layers_[k];
    layers_[i]->Reshape(bottom_vecs_[i], top_vecs_[i]);  // shrinking never reallocates (blob.cpp:40-44)
  }
}

template <typename Dtype>
void Net<Dtype>::AppendTop(const NetParameter& param, const int layer_id, const int top_id,
                           set<string>* available_blobs, map<string, int>* blob_name_to_idx) {
  const LayerParameter& layer_param = param.layer(layer_id);
  const string& blob_name = layer_param.top(top_id);
  if (layer_param.bottom_size() > top_id && blob_name == layer_param.bottom(top_id)) {
    // in-place computation (net.cpp:391-398)
    top_vecs_[layer_id].push_back(blobs_[(*blob_name_to_idx)[blob_name]].get());
    top_id_vecs_[layer_id].push_back((*blob_name_to_idx)[blob_name]);
  } else if (blob_name_to_idx->find(blob_name) != blob_name_to_idx->end()) {
    LOG(FATAL) << "Top blob '" << blob_name << "' produced by multiple sources.";
  } else {
    shared_ptr<Blob<Dtype> > blob_pointer(new Blob<Dtype>());
    const int blob_id = (int)blobs_.size();
    blobs_.push_back(blob_pointer);
    blob_names_.push_back(blob_name);
    (*blob_name_to_idx)[blob_name] = blob_id;
    top_id_vecs_[layer_id].push_back(blob_id);
    top_vecs_[layer_id].push_back(blob_pointer.get());
  }
  available_blobs->insert(blob_name);
}

template <typename Dtype>
int Net<Dtype>::AppendBottom(const NetParameter& param, const int layer_id, const int bottom_id,
                             set<string>* available_blobs, map<string, int>* blob_name_to_idx) {
  const LayerParameter& layer_param = param.layer(layer_id);
  const string& blob_name = layer_param.bottom(bottom_id);
  if (available_blobs->find(blob_name) == available_blobs->end())
    LOG(FATAL) << "Unknown bottom blob '" << blob_name << "' (layer '" << layer_param.name()
               << "', bottom index " << bottom_id << ")";
  const int blob_id = (*blob_name_to_idx)[blob_name];
  bottom_vecs_[layer_id].push_back(blobs_[blob_id].get());
  bottom_id_vecs_[layer_id].push_back(blob_id);
  available_blobs->erase(blob_name);
  return blob_id;
}

// Fold (a) in-place ReLU into the Convolution / InnerProduct that wrote the blob, when nothing
// reads the blob in between, and (b) a Concat whose bottoms are all produced by ROIPooling
// layers (and consumed only by the Concat) into those producers.
template <typename Dtype>
void Net<Dtype>::FuseLayers() {
  const int L = (int)layers_.size();
  for (int i = 0; i < L; ++i) {
    ReLULayer<Dtype>* relu = dynamic_cast<ReLULayer<Dtype>*>(layers_[i].get());
    if (!relu || bottom_vecs_[i].size() != 1 || top_vecs_[i][0] != bottom_vecs_[i][0]) continue;
    const int blob_id = bottom_id_vecs_[i][0];
    int writer = -1;  // the last layer before the ReLU that writes the blob
    for (int k : writers_[blob_id]) writer = k < i ? k : writer;
    bool clean = true;  // nobody reads the pre-ReLU value
    for (int k : readers_[blob_id]) clean = clean && !(k > writer && k < i);
    if (writer < 0 || !clean) continue;
    if (ConvolutionLayer<Dtype>* conv = dynamic_cast<ConvolutionLayer<Dtype>*>(layers_[writer].get())) {
      conv->set_fuse_relu(true);
      relu->set_fused(true);
    } else if (InnerProductLayer<Dtype>* ip = dynamic_cast<InnerProductLayer<Dtype>*>(layers_[writer].get())) {
      ip->set_fuse_relu(true);
      relu->set_fused(true);
    }
  }
  for (int i = 0; i < L; ++i) {
    ConcatLayer<Dtype>* cat = dynamic_cast<ConcatLayer<Dtype>*>(layers_[i].get());
    if (!cat || bottom_vecs_[i].size() < 2) continue;
    vector<int> offset(L, -1);  // per layer: the channel offset at which a producer writes the Concat top
    bool ok = true;
    int total = 0;
    for (size_t b = 0; b < bottom_id_vecs_[i].size() && ok; ++b) {
      const int blob_id = bottom_id_vecs_[i][b], writer = writers_[blob_id].back();  // every blob has a writer
      const int c = bottom_vecs_[i][b]->channels();
      if (!dynamic_cast<ROIPoolingLayer<Dtype>*>(layers_[writer].get()) || readers_[blob_id].size() != 1 || c % 64 != 0)
        ok = false;
      else
        offset[writer] = total;
      total += c;
    }
    if (!ok) continue;
    // The first producer in execution order leads.  A later one that pools the same feature map with the same ROIs
    // (Split tops share their bottom's storage) and the same geometry joins the leader's launch, up to the kernel's 4
    // variants; any other producer launches its own.
    int leader = -1, variants = 0;
    for (int k = 0; k < L; ++k) {
      if (offset[k] < 0) continue;
      ROIPoolingLayer<Dtype>* rp = static_cast<ROIPoolingLayer<Dtype>*>(layers_[k].get());
      rp->set_concat_target(top_vecs_[i][0], offset[k], total);
      if (leader < 0) {
        leader = k;
        variants = 1;
        continue;
      }
      const ROIPoolingParameter& p = rp->layer_param().roi_pooling_param();
      const ROIPoolingParameter& q = layers_[leader]->layer_param().roi_pooling_param();
      if (variants < 4 && storage_blob_[bottom_id_vecs_[k][0]] == storage_blob_[bottom_id_vecs_[leader][0]] &&
          storage_blob_[bottom_id_vecs_[k][1]] == storage_blob_[bottom_id_vecs_[leader][1]] &&
          p.pooled_h() == q.pooled_h() && p.pooled_w() == q.pooled_w() && p.spatial_scale() == q.spatial_scale()) {
        static_cast<ROIPoolingLayer<Dtype>*>(layers_[leader].get())->add_follower(rp);
        fused_producer_[k] = leader;
        ++variants;
      }
    }
    cat->set_fused(true);
  }
}

// (c) a 2x2 / stride-2 MAX Pooling whose bottom was written by a Convolution (possibly through its
// fused in-place ReLU) is computed in that convolution's epilogue whenever the extents are even
// (epilogue_pools).  If nothing else reads the un-pooled blob it is then not written at all.
template <typename Dtype>
void Net<Dtype>::FusePooling() {
  const int L = (int)layers_.size();
  for (int i = 0; i < L; ++i) {
    PoolingLayer<Dtype>* pool = dynamic_cast<PoolingLayer<Dtype>*>(layers_[i].get());
    if (!pool || !pool->is_max_2x2_s2()) continue;
    const int blob_id = bottom_id_vecs_[i][0];
    // walk back over the writers of the blob: [conv] or [conv, fused in-place relu]
    const vector<int>& w = writers_[blob_id];
    int conv_idx = -1;
    bool ok = true;
    for (int j = (int)w.size() - 1; j >= 0 && conv_idx < 0 && ok; --j) {
      const int k = w[j];
      if (k >= i) continue;
      if (ReLULayer<Dtype>* r = dynamic_cast<ReLULayer<Dtype>*>(layers_[k].get())) {
        if (!r->fused()) ok = false;
        continue;
      }
      if (dynamic_cast<ConvolutionLayer<Dtype>*>(layers_[k].get())) conv_idx = k;
      else ok = false;
    }
    if (!ok || conv_idx < 0) continue;
    ConvolutionLayer<Dtype>* conv = static_cast<ConvolutionLayer<Dtype>*>(layers_[conv_idx].get());
    if (!conv->can_fuse_pool()) continue;
    // other readers of the un-pooled blob (in-place layers, which write it too, excluded)?
    int readers = 0;
    for (int k : readers_[blob_id]) readers += k != i && std::find(w.begin(), w.end(), k) == w.end();
    bool is_net_output = false;
    for (size_t o = 0; o < net_output_blob_indices_.size(); ++o)
      is_net_output = is_net_output || (net_output_blob_indices_[o] == blob_id);
    conv->set_fused_pool(top_vecs_[i][0], readers > 0 || is_net_output);
    pool->set_fused(true);
    fused_producer_[i] = conv_idx;
  }
}

template <typename Dtype>
int Net<Dtype>::last_reader(const string& blob_name) const {
  const int storage = storage_blob_[blob_names_index_.at(blob_name)];
  int last = -1;
  for (size_t b = 0; b < blobs_.size(); ++b)
    if (storage_blob_[b] == storage && !readers_[b].empty()) last = std::max(last, readers_[b].back());
  return last;
}

template <typename Dtype>
int Net<Dtype>::fused_group_end(int layer) const {
  int last = layer;
  for (int k = layer + 1; k < (int)fused_producer_.size(); ++k)
    if (fused_producer_[k] == layer) last = k;
  return last;
}

// ---- CUDA graph replay of the whole forward (set_graph_mode) ----------------------------------------------------
// The forward of a fixed-shape net is the same ~50 launches every time; with deferred rows (layer.hpp DynRows) no layer
// talks to the host in between, so the launches of ForwardFromTo(0, last) are captured once (after one eager forward
// that did every allocation and weight packing) and replayed with a single cudaGraphLaunch.  What a launch depends on
// is folded into a signature: input shapes, parameter versions, precision, stream, config epoch; any change drops the
// graph.  Host-side layer state is identical after every forward of a fixed-shape net, so a replay leaves it alone,
// except BoxOutput's pending row count, which is re-armed.
template <typename Dtype>
struct Net<Dtype>::GraphState {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  std::string signature;
  int warm = 0;
  unsigned long long kernel_nodes = 0;
  ~GraphState() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
  }
};

template <typename Dtype>
bool Net<Dtype>::GraphForward(int start, int end) {
  graph_replayed_ = false;
  cudaStream_t stream = Caffe::stream();
  if (!graph_mode_ || time_layers_ || start != 0 || end != (int)layers_.size() - 1 || stream == nullptr) return false;
  std::ostringstream sig;
  sig << (void*)stream << "|" << (int)Caffe::precision() << "|" << mscnn::config().epoch << "|" << plan_epoch_ << "|";
  for (size_t i = 0; i < net_input_blobs_.size(); ++i) sig << net_input_blobs_[i]->shape_string() << ";";
  unsigned long versions = 0;
  for (size_t i = 0; i < layers_.size(); ++i)
    for (size_t j = 0; j < layers_[i]->blobs().size(); ++j) versions += layers_[i]->blobs()[j]->version() * (unsigned long)(31 * i + j + 1);
  sig << versions;
  if (!graph_ || graph_->signature != sig.str()) {
    graph_.reset(new GraphState());
    graph_->signature = sig.str();
  }
  GraphState& g = *graph_;
  if (g.warm == 0) {  // one eager forward first: allocations and weight packing must not happen under capture
    g.warm = 1;
    return false;
  }
  BoxOutputLayer<Dtype>* box = dyn_box_ >= 0 ? static_cast<BoxOutputLayer<Dtype>*>(layers_[dyn_box_].get()) : nullptr;
  if (!g.exec) {
    if (cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    for (int i = start; i <= end; ++i) layers_[i]->Forward(bottom_vecs_[i], top_vecs_[i]);
    cudaGraph_t graph = nullptr;
    CUDA_CHECK(cudaStreamEndCapture(stream, &graph));
    g.graph = graph;
    CUDA_CHECK(cudaGraphInstantiate(&g.exec, graph, 0));
    size_t n = 0;
    CUDA_CHECK(cudaGraphGetNodes(graph, nullptr, &n));
    std::vector<cudaGraphNode_t> nodes(n);
    if (n) CUDA_CHECK(cudaGraphGetNodes(graph, nodes.data(), &n));
    for (size_t k = 0; k < n; ++k) {
      cudaGraphNodeType t;
      if (cudaGraphNodeGetType(nodes[k], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) ++g.kernel_nodes;
    }
  } else {
    mscnn::g_kernel_launches.fetch_add(g.kernel_nodes, std::memory_order_relaxed);  // the capture counted its own
  }
  CUDA_CHECK(cudaGraphLaunch(g.exec, stream));
  if (box) box->RearmRows();
  graph_replayed_ = true;
  return true;
}

template <typename Dtype>
Dtype Net<Dtype>::ForwardFromTo(int start, int end) {
  CHECK_GE(start, 0);
  CHECK_LT(end, (int)layers_.size());
  start = fused_producer(start);  // a range never starts inside a fused group (net.hpp fused_producer)
  BeginActivations(start, end);
  if (GraphForward(start, end)) {
    EndActivations(start, end, true);
    if (!lazy_rows_) ResolveRows();
    return Dtype(0);
  }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (time_layers_) {
    CUDA_CHECK(cudaEventCreate(&e0));
    CUDA_CHECK(cudaEventCreate(&e1));
  }
  for (int i = start; i <= end; ++i) {
    if (time_layers_) CUDA_CHECK(cudaEventRecord(e0, Caffe::stream()));
    layers_[i]->Forward(bottom_vecs_[i], top_vecs_[i]);
    if (time_layers_) {
      CUDA_CHECK(cudaEventRecord(e1, Caffe::stream()));
      CUDA_CHECK(cudaEventSynchronize(e1));
      CUDA_CHECK(cudaEventElapsedTime(&layer_ms_[i], e0, e1));
    }
  }
  if (time_layers_) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  EndActivations(start, end, false);
  if (!lazy_rows_) ResolveRows();
  return Dtype(0);
}

template <typename Dtype>
const vector<Blob<Dtype>*>& Net<Dtype>::Forward(Dtype* loss) {
  const Dtype l = ForwardFromTo(0, (int)layers_.size() - 1);
  if (loss) *loss = l;
  return net_output_blobs_;
}

template <typename Dtype>
void Net<Dtype>::Reshape() {
  for (size_t i = 0; i < layers_.size(); ++i) layers_[i]->Reshape(bottom_vecs_[i], top_vecs_[i]);
}

template <typename Dtype>
void Net<Dtype>::CopyTrainedLayersFrom(const NetParameter& param) {
  for (int i = 0; i < param.layer_size(); ++i) {
    const LayerParameter& source_layer = param.layer(i);
    const string& source_layer_name = source_layer.name();
    map<string, int>::const_iterator it = layer_names_index_.find(source_layer_name);
    if (it == layer_names_index_.end()) continue;  // "Ignoring source layer"
    vector<shared_ptr<Blob<Dtype> > >& target_blobs = layers_[it->second]->blobs();
    CHECK_EQ((int)target_blobs.size(), source_layer.blobs_size())
        << "Incompatible number of blobs for layer " << source_layer_name;
    for (size_t j = 0; j < target_blobs.size(); ++j) {
      if (!target_blobs[j]->ShapeEquals(source_layer.blobs((int)j))) {
        Blob<Dtype> source_blob;
        source_blob.FromProto(source_layer.blobs((int)j), true);
        LOG(FATAL) << "Cannot copy param " << j << " weights from layer '" << source_layer_name
                   << "'; shape mismatch.  Source param shape is " << source_blob.shape_string()
                   << "; target param shape is " << target_blobs[j]->shape_string();
      }
      target_blobs[j]->FromProto(source_layer.blobs((int)j), false);
    }
  }
}

// A source layer matches the first layer of this net with its name (the reference's linear search).
template <typename Dtype>
string Net<Dtype>::ShareTrainedLayersError(const Net* other) const {
  std::ostringstream msg;
  if (other->device_ != device_) {
    msg << "Cannot share trained layers between nets on different devices (" << other->device_ << " and " << device_
        << ")";
    return msg.str();
  }
  for (size_t i = 0; i < other->layers().size(); ++i) {
    const string& name = other->layer_names()[i];
    const size_t t = std::find(layer_names_.begin(), layer_names_.end(), name) - layer_names_.begin();
    if (t == layer_names_.size()) continue;
    const vector<shared_ptr<Blob<Dtype> > >& source_blobs = other->layers()[i]->blobs();
    const vector<shared_ptr<Blob<Dtype> > >& target_blobs = layers_[t]->blobs();
    if (target_blobs.size() != source_blobs.size()) {
      msg << "Incompatible number of blobs for layer " << name << " (" << target_blobs.size() << " vs. "
          << source_blobs.size() << ")";
      return msg.str();
    }
    for (size_t j = 0; j < target_blobs.size(); ++j)
      if (target_blobs[j]->shape() != source_blobs[j]->shape()) {
        msg << "Cannot share param " << j << " weights from layer '" << name
            << "'; shape mismatch.  Source param shape is " << source_blobs[j]->shape_string()
            << "; target param shape is " << target_blobs[j]->shape_string();
        return msg.str();
      }
  }
  return string();
}

template <typename Dtype>
void Net<Dtype>::ShareTrainedLayersWith(const Net* other) {
  const string err = ShareTrainedLayersError(other);
  if (!err.empty()) LOG(FATAL) << err;
  for (size_t i = 0; i < other->layers().size(); ++i) {
    const string& name = other->layer_names()[i];
    const size_t t = std::find(layer_names_.begin(), layer_names_.end(), name) - layer_names_.begin();
    if (t == layer_names_.size()) continue;  // "Ignoring source layer"
    vector<shared_ptr<Blob<Dtype> > >& target_blobs = layers_[t]->blobs();
    for (size_t j = 0; j < target_blobs.size(); ++j) target_blobs[j]->ShareData(*other->layers()[i]->blobs()[j]);
  }
}

// ---- protobuf wire-format reader for NetParameter.layer[].{name, blobs[]} (caffe.proto:10-22,
// 64-100, 310-330).  Field numbers: NetParameter.layer = 100; LayerParameter.name = 1,
// .blobs = 7; BlobProto.shape = 7 (BlobShape.dim = 1, packed int64), .data = 5 (packed float),
// .num/.channels/.height/.width = 1..4, .double_data = 8.
namespace wire {
struct Reader {
  const unsigned char* p;
  const unsigned char* end;
  bool ok;
  Reader(const void* b, size_t n) : p((const unsigned char*)b), end((const unsigned char*)b + n), ok(true) {}
  bool done() const { return p >= end || !ok; }
  uint64_t varint() {
    uint64_t v = 0;
    int shift = 0;
    while (p < end && shift < 64) {
      const unsigned char c = *p++;
      v |= (uint64_t)(c & 0x7F) << shift;
      if (!(c & 0x80)) return v;
      shift += 7;
    }
    ok = false;
    return 0;
  }
  Reader sub() {
    const uint64_t n = varint();
    if (!ok || n > (uint64_t)(end - p)) { ok = false; return Reader(p, 0); }
    Reader r(p, (size_t)n);
    p += n;
    return r;
  }
  void skip(int wt) {
    if (wt == 0) varint();
    else if (wt == 1) p += 8;
    else if (wt == 2) sub();
    else if (wt == 5) p += 4;
    else ok = false;
    if (p > end) ok = false;
  }
};

static void parse_blob(Reader r, BlobProto* b, bool* ok) {
  while (!r.done()) {
    const uint64_t key = r.varint();
    const int field = (int)(key >> 3), wt = (int)(key & 7);
    if (field == 7 && wt == 2) {  // shape
      Reader s = r.sub();
      while (!s.done()) {
        const uint64_t k2 = s.varint();
        if ((k2 >> 3) == 1 && (k2 & 7) == 2) {
          Reader d = s.sub();
          while (!d.done()) b->mutable_shape()->add_dim((int64_t)d.varint());
        } else if ((k2 >> 3) == 1 && (k2 & 7) == 0) {
          b->mutable_shape()->add_dim((int64_t)s.varint());
        } else {
          s.skip((int)(k2 & 7));
        }
      }
    } else if (field == 5 && wt == 2) {  // packed float data
      Reader d = r.sub();
      const size_t n = (size_t)(d.end - d.p) / 4;
      for (size_t i = 0; i < n; ++i) {
        float v;
        memcpy(&v, d.p + 4 * i, 4);
        b->add_data(v);
      }
    } else if (field == 5 && wt == 5) {  // non-packed float
      if (r.end - r.p < 4) { r.ok = false; return; }
      float v;
      memcpy(&v, r.p, 4);
      r.p += 4;
      b->add_data(v);
    } else if (field == 8 && wt == 2) {  // packed double data
      Reader d = r.sub();
      const size_t n = (size_t)(d.end - d.p) / 8;
      for (size_t i = 0; i < n; ++i) {
        double v;
        memcpy(&v, d.p + 8 * i, 8);
        b->add_double_data(v);
      }
    } else if (field >= 1 && field <= 4 && wt == 0) {
      const int v = (int)r.varint();
      if (field == 1) b->set_num(v);
      else if (field == 2) b->set_channels(v);
      else if (field == 3) b->set_height(v);
      else b->set_width(v);
    } else {
      r.skip(wt);
    }
    if (!r.ok) { *ok = false; return; }
  }
}

// One layer message.  LayerParameter: name = 1, type = 2, blobs = 7 (caffe.proto:310-330); the legacy
// V1LayerParameter (NetParameter.layers = 2): name = 4, blobs = 6 (caffe.proto:1100-1150) -- the reference upgrades
// such files when it loads them (upgrade_proto.cpp:NetNeedsV1ToV2Upgrade); only names and blobs matter here.
static bool parse_layer(Reader l, LayerParameter* lp, int f_name, int f_type, int f_blobs) {
  while (!l.done()) {
    const uint64_t k2 = l.varint();
    const int f2 = (int)(k2 >> 3), w2 = (int)(k2 & 7);
    if (f2 == f_name && w2 == 2) {
      Reader s = l.sub();
      lp->set_name(std::string((const char*)s.p, (size_t)(s.end - s.p)));
    } else if (f2 == f_type && w2 == 2) {
      Reader s = l.sub();
      lp->set_type(std::string((const char*)s.p, (size_t)(s.end - s.p)));
    } else if (f2 == f_blobs && w2 == 2) {
      bool ok = true;
      parse_blob(l.sub(), lp->add_blobs(), &ok);
      if (!ok) return false;
    } else {
      l.skip(w2);
    }
    if (!l.ok) return false;
  }
  return true;
}

static bool parse_net(const std::string& bytes, NetParameter* np) {
  Reader r(bytes.data(), bytes.size());
  while (!r.done()) {
    const uint64_t key = r.varint();
    const int field = (int)(key >> 3), wt = (int)(key & 7);
    if (field == 100 && wt == 2) {
      if (!parse_layer(r.sub(), np->add_layer(), 1, 2, 7)) return false;
    } else if (field == 2 && wt == 2) {  // V1LayerParameter (type is an enum there: not needed for the copy)
      if (!parse_layer(r.sub(), np->add_layer(), 4, -1, 6)) return false;
    } else if (field == 1 && wt == 2) {
      Reader s = r.sub();
      np->set_name(std::string((const char*)s.p, (size_t)(s.end - s.p)));
    } else {
      r.skip(wt);
    }
    if (!r.ok) return false;
  }
  return r.ok;
}
}  // namespace wire

template <typename Dtype>
void Net<Dtype>::CopyTrainedLayersFrom(const string trained_filename) {
  std::ifstream in(trained_filename.c_str(), std::ios::binary);
  CHECK(in.good()) << "cannot open " << trained_filename;
  std::stringstream ss;
  ss << in.rdbuf();
  NetParameter param;
  CHECK(wire::parse_net(ss.str(), &param)) << "malformed caffemodel " << trained_filename;
  int matched = 0;
  for (int i = 0; i < param.layer_size(); ++i) matched += layer_names_index_.count(param.layer(i).name()) ? 1 : 0;
  if (matched == 0)
    LOG(WARNING) << trained_filename << ": none of its " << param.layer_size() << " layers matches a layer of this net "
                 << "by name; the net keeps its current parameters";
  CopyTrainedLayersFrom(param);
}

template <typename Dtype>
bool Net<Dtype>::has_blob(const string& blob_name) const {
  return blob_names_index_.find(blob_name) != blob_names_index_.end();
}
template <typename Dtype>
const shared_ptr<Blob<Dtype> > Net<Dtype>::blob_by_name(const string& blob_name) const {
  shared_ptr<Blob<Dtype> > blob_ptr;
  if (has_blob(blob_name)) blob_ptr = blobs_[blob_names_index_.find(blob_name)->second];
  else LOG(WARNING) << "Unknown blob name " << blob_name;
  return blob_ptr;
}
template <typename Dtype>
bool Net<Dtype>::has_layer(const string& layer_name) const {
  return layer_names_index_.find(layer_name) != layer_names_index_.end();
}
template <typename Dtype>
const shared_ptr<Layer<Dtype> > Net<Dtype>::layer_by_name(const string& layer_name) const {
  shared_ptr<Layer<Dtype> > layer_ptr;
  if (has_layer(layer_name)) layer_ptr = layers_[layer_names_index_.find(layer_name)->second];
  else LOG(WARNING) << "Unknown layer name " << layer_name;
  return layer_ptr;
}

INSTANTIATE_CLASS(Net);

}  // namespace caffe
