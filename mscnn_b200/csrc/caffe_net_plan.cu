// Activation reuse for caffe::Net (net.hpp set_activation_reuse; DESIGN.md "Activation memory plan").
//
// The unit is a storage: a blob together with the tops on its bytes (Net::storage_blob_).  The plan is made on the host
// from the net's static structure and the shapes of the forward it is for: every layer's Reshape runs, in order, on
// shadow blobs (Layer::ReshapeAsForward: BoxOutput's tops at their cap rows), and each layer states which
// representation of which blob its forward reads and writes (Layer::Accesses).  A storage is live from its first
// access to its last; storages whose intervals do not intersect may share bytes of the arena.
#include <algorithm>
#include <climits>
#include <map>
#include <set>
#include <sstream>

#include "caffe/net.hpp"

namespace caffe {

namespace {
inline size_t round256(size_t b) { return (b + 255) / 256 * 256; }
}  // namespace

template <typename Dtype>
string Net<Dtype>::ActivationKeepError(const vector<string>& keep) const {
  for (size_t k = 0; k < keep.size(); ++k)
    if (!has_blob(keep[k]))
      return "Cannot keep '" + keep[k] + "' readable under activation reuse: net '" + name_ +
             "' has no blob of that name";
  return string();
}

template <typename Dtype>
void Net<Dtype>::set_activation_reuse(bool on, const vector<string>& keep) {
  const string err = ActivationKeepError(keep);
  if (!err.empty()) LOG(FATAL) << err;
  DetachActivations();
  reuse_ = on;
  keep_ = on ? keep : vector<string>();
  plan_ = ActivationPlan();
  plan_signature_.clear();
}

template <typename Dtype>
void Net<Dtype>::DetachActivations() {
  for (size_t k = 0; k < on_arena_.size(); ++k) blobs_[on_arena_[k]]->LeaveArena();
  on_arena_.clear();
  for (size_t b = 0; b < blobs_.size(); ++b) blobs_[b]->set_released("");
  arena_.reset();
  arena_capacity_ = 0;
  applied_signature_.clear();
  chain_end_ = -1;
  ++plan_epoch_;
}

template <typename Dtype>
string Net<Dtype>::ActivationSignature() const {
  std::ostringstream s;
  s << (int)Caffe::precision() << "|";
  for (size_t i = 0; i < net_input_blobs_.size(); ++i) s << net_input_blobs_[i]->shape_string() << ";";
  s << "|";
  for (size_t k = 0; k < keep_.size(); ++k) s << keep_[k] << ",";
  return s.str();
}

template <typename Dtype>
const typename Net<Dtype>::ActivationPlan& Net<Dtype>::activation_plan() {
  if (!reuse_) {
    plan_ = ActivationPlan();
    plan_signature_.clear();
    return plan_;
  }
  const string sig = ActivationSignature();
  if (sig != plan_signature_) {
    ActivationPlan p;
    ComputeActivationPlan(&p);
    plan_ = p;
    plan_signature_ = sig;
  }
  return plan_;
}

template <typename Dtype>
void Net<Dtype>::ComputeActivationPlan(ActivationPlan* plan) const {
  const int B = (int)blobs_.size(), L = (int)layers_.size();
  const bool split = Caffe::split();
  // 1. the shapes of the forward
  vector<shared_ptr<Blob<Dtype> > > shadow(B);
  for (int b = 0; b < B; ++b) shadow[b].reset(new Blob<Dtype>());
  for (size_t k = 0; k < net_input_blob_indices_.size(); ++k)
    shadow[net_input_blob_indices_[k]]->Reshape(net_input_blobs_[k]->shape());
  vector<vector<Blob<Dtype>*> > sb(L), st(L);
  for (int i = 0; i < L; ++i) {
    for (size_t k = 0; k < bottom_id_vecs_[i].size(); ++k) sb[i].push_back(shadow[bottom_id_vecs_[i][k]].get());
    for (size_t k = 0; k < top_id_vecs_[i].size(); ++k) st[i].push_back(shadow[top_id_vecs_[i][k]].get());
    layers_[i]->ReshapeAsForward(sb[i], st[i]);
  }
  // 2. who reads and writes what, where, as each layer states it; a fused target (a pooled or Concat top) is named
  // by its real blob, every other blob by its shadow
  std::map<const Blob<Dtype>*, int> id_of;
  for (int b = 0; b < B; ++b) id_of[blobs_[b].get()] = id_of[shadow[b].get()] = b;
  struct Use {
    int first = INT_MAX, last = -1;
    bool planes = false, nchw = false;
    vector<int> at;
  };
  vector<Use> use(B);
  for (int i = 0; i < L; ++i) {
    BlobAccesses<Dtype> acc;
    if (!layers_[i]->Accesses(sb[i], st[i], &acc))
      LOG(FATAL) << "activation reuse has no plan for layer type " << layers_[i]->type() << " (layer "
                 << layer_names_[i] << ")";
    for (size_t k = 0; k < acc.size(); ++k) {
      Use& u = use[storage_blob_[id_of.at(acc[k].first)]];
      u.first = std::min(u.first, i);
      u.last = std::max(u.last, i);
      u.planes = u.planes || acc[k].second == PLANES;
      u.nchw = u.nchw || acc[k].second == NCHW;
      if (u.at.empty() || u.at.back() != i) u.at.push_back(i);
    }
  }
  // 3. bytes, and what stays outside the arena
  std::set<int> inputs(net_input_blob_indices_.begin(), net_input_blob_indices_.end());
  std::set<int> outputs(net_output_blob_indices_.begin(), net_output_blob_indices_.end());
  std::set<int> kept;
  for (size_t k = 0; k < keep_.size(); ++k) kept.insert(blob_names_index_.at(keep_[k]));
  std::map<int, vector<int> > members;
  for (int b = 0; b < B; ++b) members[storage_blob_[b]].push_back(b);
  for (std::map<int, vector<int> >::iterator it = members.begin(); it != members.end(); ++it) {
    const Use& u = use[it->first];
    if (u.last < 0 || !(u.planes || u.nchw)) continue;
    ActivationStorage s;
    s.blob = it->first;
    s.members = it->second;
    s.touched = u.at;
    s.first = u.first;
    s.last = u.last;
    s.offset = -1;
    s.plane_bytes = 0;
    s.lo = false;
    s.nchw_count = 0;
    const Blob<Dtype>& sh = *shadow[it->first];
    if (u.planes) {
      const int cpad = (sh.channels() + 63) / 64 * 64;
      s.plane_bytes = std::max<size_t>((size_t)sh.num() * sh.height() * sh.width() * cpad * 2, 2);
      s.lo = split;
    }
    if (u.nchw) s.nchw_count = std::max(sh.count(), 1);
    s.bytes = round256(s.plane_bytes) * (s.lo ? 2 : 1) + round256((size_t)s.nchw_count * sizeof(Dtype));
    for (size_t k = 0; k < s.members.size(); ++k) {
      const int b = s.members[k];
      if (inputs.count(b)) s.outside = "input";
      else if (outputs.count(b) && s.outside != "input") s.outside = "output";
      else if (kept.count(b) && s.outside.empty()) s.outside = "kept";
    }
    plan->storages.push_back(s);
  }
  std::sort(plan->storages.begin(), plan->storages.end(), [](const ActivationStorage& a, const ActivationStorage& b) {
    return a.first != b.first ? a.first < b.first : a.blob < b.blob;
  });
  // 4. offsets: largest first, each into the smallest gap left by the placed storages it is live with
  vector<int> order;
  for (size_t k = 0; k < plan->storages.size(); ++k) {
    if (plan->storages[k].outside.empty()) {
      order.push_back((int)k);
      plan->planned_bytes += plan->storages[k].bytes;
    } else {
      plan->unplanned_bytes += plan->storages[k].bytes;
    }
  }
  vector<ActivationStorage>& S = plan->storages;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return S[a].bytes > S[b].bytes; });
  vector<int> placed;
  for (size_t k = 0; k < order.size(); ++k) {
    ActivationStorage& s = S[order[k]];
    vector<std::pair<size_t, size_t> > busy;
    for (size_t q = 0; q < placed.size(); ++q) {
      const ActivationStorage& t = S[placed[q]];
      if (t.first <= s.last && s.first <= t.last) busy.push_back(std::make_pair((size_t)t.offset, t.offset + t.bytes));
    }
    std::sort(busy.begin(), busy.end());
    size_t at = 0, best = SIZE_MAX, best_gap = SIZE_MAX;
    for (size_t q = 0; q < busy.size(); ++q) {
      if (busy[q].first > at && busy[q].first - at >= s.bytes && busy[q].first - at < best_gap) {
        best_gap = busy[q].first - at;
        best = at;
      }
      at = std::max(at, busy[q].second);
    }
    s.offset = (long long)(best == SIZE_MAX ? at : best);
    plan->arena_bytes = std::max(plan->arena_bytes, (size_t)s.offset + s.bytes);
    placed.push_back(order[k]);
  }
}

template <typename Dtype>
string Net<Dtype>::activation_plan_describe() {
  const ActivationPlan& p = activation_plan();
  std::ostringstream o;
  for (size_t k = 0; k < p.storages.size(); ++k) {
    const ActivationStorage& s = p.storages[k];
    o << blob_names_[s.blob] << " " << s.bytes << " " << s.first << "-" << s.last << " ";
    if (s.offset >= 0) o << "@" << s.offset;
    else o << s.outside;
    o << "\n";
  }
  return o.str();
}

template <typename Dtype>
string Net<Dtype>::ForwardRangeError(int start, int end) {
  if (!reuse_ || start == 0) return string();
  const ActivationPlan& p = activation_plan();
  if (chain_end_ >= 0 && start == chain_end_ + 1 && applied_signature_ == plan_signature_) return string();
  for (size_t k = 0; k < p.storages.size(); ++k) {
    const ActivationStorage& s = p.storages[k];
    if (s.offset < 0 || s.first >= start) continue;
    for (size_t a = 0; a < s.touched.size(); ++a) {
      const int at = s.touched[a];
      if (at < start || at > end) continue;
      std::ostringstream m;
      m << "ForwardFromTo(" << start << ", " << end << ") with activation reuse on: layer '" << layer_names_[at]
        << "' reads blob '" << blob_names_[s.blob] << "', which is written before layer '" << layer_names_[start]
        << "' and whose storage other blobs reuse; keep it (set_activation_reuse(true, keep)) to run this range";
      return m.str();
    }
  }
  return string();
}

template <typename Dtype>
string Net<Dtype>::released_message(const string& blob_name) const {
  std::map<string, int>::const_iterator it = blob_names_index_.find(blob_name);
  return it == blob_names_index_.end() ? string() : blobs_[it->second]->released();
}

// Called by ForwardFromTo before its layers run: (re-)plans for this forward's shapes and precision, gives the planned
// blobs their arena storage when the plan changed, and makes every blob readable again for a forward from layer 0.
template <typename Dtype>
void Net<Dtype>::BeginActivations(int start, int end) {
  if (!reuse_) return;
  const string err = ForwardRangeError(start, end);
  if (!err.empty()) LOG(FATAL) << err;
  const ActivationPlan& p = activation_plan();
  if (applied_signature_ != plan_signature_) {
    // aliases too: a Split top still holds the view it shared in the last forward
    for (size_t k = 0; k < on_arena_.size(); ++k) blobs_[on_arena_[k]]->LeaveArena();
    on_arena_.clear();
    if (p.arena_bytes > arena_capacity_) {
      arena_.reset();  // the arena only grows: free the old one before the new one is allocated
      arena_capacity_ = 0;
      void* ptr = nullptr;
      CUDA_CHECK(cudaMalloc(&ptr, p.arena_bytes));
      arena_.reset(ptr, [](void* q) { cudaFree(q); });
      arena_capacity_ = p.arena_bytes;
    }
    char* base = static_cast<char*>(arena_.get());
    for (size_t k = 0; k < p.storages.size(); ++k) {
      const ActivationStorage& s = p.storages[k];
      if (s.offset < 0) continue;
      for (size_t m = 0; m < s.members.size(); ++m) {
        if (s.members[m] != s.blob) blobs_[s.members[m]]->LeaveArena();
        on_arena_.push_back(s.members[m]);
      }
      char* at = base + s.offset;
      const size_t planes = s.plane_bytes ? round256(s.plane_bytes) * (s.lo ? 2 : 1) : 0;
      blobs_[s.blob]->UseArena(s.plane_bytes ? at : nullptr, s.lo ? at + round256(s.plane_bytes) : nullptr,
                               s.plane_bytes, s.nchw_count ? reinterpret_cast<Dtype*>(at + planes) : nullptr,
                               s.nchw_count);
    }
    applied_signature_ = plan_signature_;
    chain_end_ = -1;
    ++plan_epoch_;
  }
  // The storages this range writes first are written again: readable once more.  A host read since the last forward
  // may have given a planes-only one an NCHW buffer of its own; the forward does not use it, so it goes.
  for (size_t k = 0; k < p.storages.size(); ++k) {
    const ActivationStorage& s = p.storages[k];
    if (s.offset < 0 || s.first < start || s.first > end) continue;
    for (size_t m = 0; m < s.members.size(); ++m) blobs_[s.members[m]]->set_released("");
    if (!s.nchw_count) blobs_[s.blob]->DropDeviceNchw();
  }
}

// Called by ForwardFromTo after its layers ran (or were replayed): counts planned blobs an eager forward found off
// their slot or holding a device buffer of their own the plan did not give them, and releases every planned storage whose bytes a storage written in this range took over.
template <typename Dtype>
void Net<Dtype>::EndActivations(int start, int end, bool replayed) {
  if (!reuse_) return;
  chain_end_ = end == (int)layers_.size() - 1 ? -1 : end;
  const vector<ActivationStorage>& S = plan_.storages;
  for (size_t k = 0; k < S.size(); ++k) {
    const ActivationStorage& s = S[k];
    if (s.offset < 0) continue;
    if (!replayed && s.first <= end && s.last >= start) {
      char* at = static_cast<char*>(arena_.get()) + s.offset;
      const size_t planes = s.plane_bytes ? round256(s.plane_bytes) * (s.lo ? 2 : 1) : 0;
      if (!blobs_[s.blob]->OnArena(s.plane_bytes ? at : nullptr, s.nchw_count ? at + planes : nullptr)) {
        ++activation_misses_;
        LOG(ERROR) << "activation arena miss: blob '" << blob_names_[s.blob] << "' does not hold its arena slot after "
                   << "layers " << start << ".." << end;
      }
    }
    const ActivationStorage* by = nullptr;
    for (size_t q = 0; q < S.size(); ++q) {
      const ActivationStorage& t = S[q];
      if (t.offset < 0 || t.first <= s.last || t.first < start || t.first > end) continue;
      if (t.offset < s.offset + (long long)s.bytes && s.offset < t.offset + (long long)t.bytes &&
          (!by || t.first < by->first))
        by = &t;
    }
    if (!by) continue;
    for (size_t m = 0; m < s.members.size(); ++m) {
      const string& name = blob_names_[s.members[m]];
      std::ostringstream msg;
      msg << "blob '" << name << "' was released by activation reuse: its storage is reused after layer '"
          << layer_names_[s.last] << "' (by '" << blob_names_[by->blob] << "' from layer '" << layer_names_[by->first]
          << "'); keep it readable by naming '" << name << "' in set_activation_reuse(true, keep)";
      blobs_[s.members[m]]->set_released(msg.str());
    }
  }
}

#define INSTANTIATE_PLAN(T)                                                                  \
  template string Net<T>::ActivationKeepError(const vector<string>&) const;                  \
  template void Net<T>::set_activation_reuse(bool, const vector<string>&);                   \
  template void Net<T>::DetachActivations();                                                 \
  template string Net<T>::ActivationSignature() const;                                       \
  template const Net<T>::ActivationPlan& Net<T>::activation_plan();                          \
  template void Net<T>::ComputeActivationPlan(ActivationPlan*) const;                        \
  template string Net<T>::activation_plan_describe();                                        \
  template string Net<T>::ForwardRangeError(int, int);                                       \
  template string Net<T>::released_message(const string&) const;                             \
  template void Net<T>::BeginActivations(int, int);                                          \
  template void Net<T>::EndActivations(int, int, bool);
INSTANTIATE_PLAN(float)

}  // namespace caffe
