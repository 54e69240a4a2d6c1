#include "net.hpp"
#include "hdf5_min.hpp"
#include "../../../include/fn2_flow.h"
#include "../../../include/fn2_frames.h"

#include <cstdlib>
#include <cstring>
#include <set>

namespace caffe {

void RegisterFlowNetLayers();
bool IsReLULayer(Layer<float>* l, float* slope);
void MarkReLUFused(Layer<float>* l);

template <typename Dtype>
Net<Dtype>::Net(const NetParameter& param, Phase phase) : phase_(phase) {
    RegisterFlowNetLayers();
    CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    if (getenv("FN2_NO_GRAPH")) graph_disabled_ = true;
    Init(param);
}

template <typename Dtype>
Net<Dtype>::~Net() {
    if (graph_exec_) cudaGraphExecDestroy(graph_exec_);
    if (graph_) cudaGraphDestroy(graph_);
    layers_.clear();
    blobs_.clear();
    for (cudaEvent_t e : layer_event_) if (e) cudaEventDestroy(e);
    if (fork_event_) cudaEventDestroy(fork_event_);
    if (join_event_) cudaEventDestroy(join_event_);
    if (stream2_) cudaStreamDestroy(stream2_);
    if (stream_) cudaStreamDestroy(stream_);
}

// Net::Init, net.cpp:40-286 (FilterNet by phase; no Split insertion: fan-out needs no copies
// in a forward-only executor, so the reference's "<blob>_<layer>_<idx>_split" blobs do not
// exist here -- results are unaffected).
template <typename Dtype>
void Net<Dtype>::Init(const NetParameter& param) {
    Caffe::stream() = stream_;
    name_ = param.name;
    force_backward_ = param.force_backward;
    std::set<string> available;
    for (const LayerParameter& lp : param.layers) {
        if (!lp.included_in_phase((int)phase_)) continue;
        // deep-copy the message so layers may edit their own parameters (reshape_every_iter)
        LayerParameter own(std::make_shared<Message>(*lp.m));
        shared_ptr<Layer<Dtype> > layer = LayerRegistry<Dtype>::CreateLayer(own);
        layer->set_phase(phase_);
        const int li = (int)layers_.size();
        layers_.push_back(layer);
        layer_names_.push_back(own.name());
        bottom_vecs_.emplace_back(); top_vecs_.emplace_back();
        bottom_id_vecs_.emplace_back(); top_id_vecs_.emplace_back();
        // AppendBottom, net.cpp:423-448
        for (int b = 0; b < own.bottom_size(); b++) {
            const string& bn = own.bottom(b);
            auto it = blob_names_index_.find(bn);
            CHECK(it != blob_names_index_.end())
                << "Unknown bottom blob '" << bn << "' (layer '" << own.name() << "', bottom index " << b << ")";
            bottom_vecs_[li].push_back(blobs_[it->second].get());
            bottom_id_vecs_[li].push_back(it->second);
        }
        // AppendTop, net.cpp:386-420
        for (int t = 0; t < own.top_size(); t++) {
            const string& tn = own.top(t);
            if (t < own.bottom_size() && own.bottom(t) == tn) {               // in-place
                top_vecs_[li].push_back(blobs_[bottom_id_vecs_[li][t]].get());
                top_id_vecs_[li].push_back(bottom_id_vecs_[li][t]);
            } else {
                CHECK(blob_names_index_.find(tn) == blob_names_index_.end())
                    << "Top blob '" << tn << "' produced by multiple sources.";
                shared_ptr<Blob<Dtype> > nb(new Blob<Dtype>());
                nb->set_layout(layer->TopLayout(), -1);
                const int id = (int)blobs_.size();
                blobs_.push_back(nb);
                blob_names_.push_back(tn);
                blob_names_index_[tn] = id;
                top_vecs_[li].push_back(nb.get());
                top_id_vecs_[li].push_back(id);
                if (string(layer->type()) == "Input") net_input_blob_indices_.push_back(id);   // net.cpp:110-114
            }
            available.insert(tn);
        }
        layer->SetUp(bottom_vecs_[li], top_vecs_[li]);
        for (int b = 0; b < own.bottom_size(); b++) {
            // a blob stays a candidate net output until some layer consumes it (net.cpp:270-276);
            // in-place tops re-insert themselves above
            bool is_top_too = false;
            for (int t = 0; t < own.top_size(); t++) if (own.top(t) == own.bottom(b)) is_top_too = true;
            if (!is_top_too) available.erase(own.bottom(b));
        }
        // re-mark bottoms as usable by later layers (fan-out): availability for *consumption* is
        // tracked by name existence, `available` only decides net outputs
    }
    for (size_t i = 0; i < blob_names_.size(); i++)
        if (available.count(blob_names_[i])) net_output_blob_indices_.push_back((int)i);
    FuseReLUs();
    AliasConcats();
    BuildArena();
    PlanStreams();
    FuseWarpBlocks();
}

// Resample(LINEAR, 2 bottoms, up-sampling a 2-channel flow) -> FlowWarp(img1, flow) -> Eltwise(img0, warped; 1, -1) -> ChannelNorm,
// and Eltwise(flow; coeff): FlowNet2's hand-over between stacked networks.  The fused pass has no backward, so a block fuses only
// when none of its five layers needs backward -- always in FlowNet2's graphs, deploy or training, because the Resample layer
// stops the gradient.
template <typename Dtype>
void Net<Dtype>::FuseWarpBlocks() {
    absorbed_.assign(layers_.size(), 0);
    if (getenv("FN2_NO_WARPFUSE")) return;
    const int L = (int)layers_.size();
    vector<char> layer_need, blob_need;
    NeedBackward(&layer_need, &blob_need);
    auto consumers = [&](int blob, int after) {
        vector<int> c;
        for (int j = after + 1; j < L; j++) for (int b : bottom_id_vecs_[j]) if (b == blob) { c.push_back(j); break; }
        return c;
    };
    auto inplace = [&](int j) { for (int t : top_id_vecs_[j]) for (int b : bottom_id_vecs_[j]) if (t == b) return true; return false; };
    for (int r = 0; r < L; r++) {
        if (string(layers_[r]->type()) != "Resample" || bottom_id_vecs_[r].size() != 2 || top_id_vecs_[r].size() != 1) continue;
        const LayerParameter& rl = layers_[r]->layer_param();
        if (rl.resample_param().type() != 2) continue;
        Blob<Dtype>* fin = bottom_vecs_[r][0];
        Blob<Dtype>* ff = top_vecs_[r][0];
        if (fin->channels() != 2 || fin->height() > ff->height() || fin->width() > ff->width()) continue;
        const int ffid = top_id_vecs_[r][0];
        WarpBlock wb; wb.resample = r; wb.warp = wb.sub = wb.norm = wb.scale = -1; wb.coeff = 0; wb.fill_nan = 0;
        for (int j : consumers(ffid, r)) {
            const string ty = layers_[j]->type();
            if (ty == "FlowWarp" && bottom_id_vecs_[j].size() == 2 && bottom_id_vecs_[j][1] == ffid && wb.warp < 0) wb.warp = j;
            else if (ty == "Eltwise" && bottom_id_vecs_[j].size() == 1 && !inplace(j) && wb.scale < 0) {
                EltwiseParameter ep = layers_[j]->layer_param().eltwise_param();
                if (ep.operation() == "SUM" && ep.coeff_size() == 1) { wb.scale = j; wb.coeff = ep.coeff(0); }
            }
        }
        if (wb.warp < 0 || wb.scale < 0 || inplace(wb.warp)) continue;
        wb.fill_nan = layers_[wb.warp]->layer_param().flow_warp_param().fill_nan() ? 1 : 0;
        const int wid = top_id_vecs_[wb.warp][0];
        if (bottom_vecs_[wb.warp][0]->channels() > 4) continue;
        for (int j : consumers(wid, wb.warp)) {
            if (string(layers_[j]->type()) != "Eltwise" || bottom_id_vecs_[j].size() != 2 || bottom_id_vecs_[j][1] != wid || inplace(j)) continue;
            EltwiseParameter ep = layers_[j]->layer_param().eltwise_param();
            if (ep.operation() == "SUM" && ep.coeff_size() == 2 && ep.coeff(0) == 1.f && ep.coeff(1) == -1.f) { wb.sub = j; break; }
        }
        if (wb.sub < 0) continue;
        const int eid = top_id_vecs_[wb.sub][0];
        for (int j : consumers(eid, wb.sub))
            if (string(layers_[j]->type()) == "ChannelNorm" && !inplace(j)) { wb.norm = j; break; }
        if (wb.norm < 0) continue;
        // the second image must exist before the Resample layer runs, and everything has to sit on one stream
        const int members[4] = {wb.warp, wb.sub, wb.norm, wb.scale};
        bool ok = !layer_need[r];
        for (int m : members) if (layer_need[m] || (!layer_stream_.empty() && layer_stream_[m] != layer_stream_[r])) ok = false;
        auto produced_before = [&](int blob) {
            for (int j = r; j < L; j++) for (int t : top_id_vecs_[j]) if (t == blob) return false;
            return true;
        };
        if (!produced_before(bottom_id_vecs_[wb.warp][0]) || !produced_before(bottom_id_vecs_[wb.sub][0])) ok = false;
        // nobody between the Resample layer and a member may touch the member's top early
        for (int m : members)
            for (int j = r + 1; j < m && ok; j++) {
                if (j == wb.warp || j == wb.sub || j == wb.norm || j == wb.scale) continue;
                for (int b : bottom_id_vecs_[j]) if (b == top_id_vecs_[m][0]) ok = false;
            }
        if (!ok) continue;
        if (!layer_wait_.empty()) for (int m : members) layer_wait_[r] = std::max(layer_wait_[r], layer_wait_[m]);
        warp_head_[r] = wb;
        for (int m : members) absorbed_[m] = 1;
    }
}

template <typename Dtype>
void Net<Dtype>::RunLayer(int i) {
    if (absorbed_[i]) return;
    auto it = warp_head_.find(i);
    if (it == warp_head_.end()) { layers_[i]->Forward(bottom_vecs_[i], top_vecs_[i]); return; }
    const WarpBlock& w = it->second;
    fn2_tensor fin = bottom_vecs_[i][0]->tensor(), ff = top_vecs_[i][0]->mutable_tensor();
    fn2_tensor i1 = bottom_vecs_[w.warp][0]->tensor(), wp = top_vecs_[w.warp][0]->mutable_tensor();
    fn2_tensor i0 = bottom_vecs_[w.sub][0]->tensor(), er = top_vecs_[w.sub][0]->mutable_tensor();
    fn2_tensor en = top_vecs_[w.norm][0]->mutable_tensor(), fs = top_vecs_[w.scale][0]->mutable_tensor();
    int rc = fn2_warp_block_forward(&fin, &i0, &i1, &ff, &wp, &er, &en, &fs, w.coeff, w.fill_nan, Caffe::stream());
    CHECK(rc == 0) << "fn2_warp_block_forward: " << fn2_last_error();
}

template <typename Dtype>
shared_ptr<Blob<Dtype> > Net<Dtype>::blob_by_name(const string& name) const {
    auto it = blob_names_index_.find(name);
    CHECK(it != blob_names_index_.end()) << "Unknown blob name " << name;
    return blobs_[it->second];
}

// Conv/Deconv top followed directly (first consumer, in place) by ReLU -> epilogue fusion.
template <typename Dtype>
void Net<Dtype>::FuseReLUs() {
    if (getenv("FN2_NO_FUSE")) return;
    for (size_t li = 0; li < layers_.size(); li++) {
        const string type = layers_[li]->type();
        if (type != "Convolution" && type != "Deconvolution") continue;
        for (size_t t = 0; t < top_id_vecs_[li].size(); t++) {
            const int bid = top_id_vecs_[li][t];
            // first later layer that touches this blob
            for (size_t lj = li + 1; lj < layers_.size(); lj++) {
                bool touches = false;
                for (int b : bottom_id_vecs_[lj]) if (b == bid) touches = true;
                if (!touches) continue;
                float slope = 0;
                if (IsReLULayer(layers_[lj].get(), &slope) && top_id_vecs_[lj].size() == 1 && top_id_vecs_[lj][0] == bid) {
                    if (layers_[li]->FuseReLU((int)t, slope)) MarkReLUFused(layers_[lj].get());
                }
                break;
            }
        }
    }
}

// Zero-copy channel Concat: bottoms become channel-range views of the top's NHWC storage.
template <typename Dtype>
void Net<Dtype>::AliasConcats() {
    if (getenv("FN2_NO_ALIAS")) return;
    std::set<int> inputs(net_input_blob_indices_.begin(), net_input_blob_indices_.end());
    for (size_t li = 0; li < layers_.size(); li++) {
        if (string(layers_[li]->type()) != "Concat" || bottom_id_vecs_[li].size() < 2) continue;
        Blob<Dtype>* top = top_vecs_[li][0];
        if (top->layout() != Blob<Dtype>::NHWC) continue;
        int c0 = 0;
        std::set<int> seen;
        for (size_t b = 0; b < bottom_id_vecs_[li].size(); b++) {
            const int bid = bottom_id_vecs_[li][b];
            Blob<Dtype>* bl = bottom_vecs_[li][b];
            bool ok = !inputs.count(bid) && !bl->is_alias() && bl->layout() == Blob<Dtype>::NHWC && !seen.count(bid) && bl != top;
            // nobody may write the bottom after the concat ran (it would also change the top)
            for (size_t lj = li + 1; lj < layers_.size() && ok; lj++)
                for (int t : top_id_vecs_[lj]) if (t == bid) ok = false;
            // the top must not be an in-place target of a later layer that some other reader of
            // the bottom must not observe
            for (size_t lj = li + 1; lj < layers_.size() && ok; lj++) {
                bool writes_top = false;
                for (int t : top_id_vecs_[lj]) if (t == top_id_vecs_[li][0]) writes_top = true;
                if (writes_top) ok = false;
            }
            // a bottom that also feeds a convolution with few input channels stays dense: the tensor-core engine then
            // fetches whole kernel rows per TMA box (and needs 16-byte aligned pixels), which beats saving this copy
            for (size_t lj = 0; lj < layers_.size() && ok; lj++) {
                if (string(layers_[lj]->type()) != "Convolution" || bl->channels() > 16) continue;
                for (int bb : bottom_id_vecs_[lj]) if (bb == bid) ok = false;
            }
            seen.insert(bid);
            if (ok) bl->AliasInto(top, c0);
            c0 += bl->channels();
        }
    }
}

// Floats a parameter blob takes in the parameter and gradient arenas: every slot starts 256-byte aligned
template <typename Dtype>
static size_t arena_slot(const Blob<Dtype>& b) { return ((size_t)b.count() + 63) / 64 * 64; }

template <typename Dtype>
void Net<Dtype>::BuildArena() {
    size_t total = 0;
    for (auto& l : layers_)
        for (auto& b : l->blobs()) total += arena_slot(*b);
    arena_floats_ = total;
    if (!total) return;
    arena_.reserve(total * sizeof(Dtype), stream_);
    size_t off = 0;
    for (auto& l : layers_)
        for (auto& b : l->blobs()) {
            b->BindExternal(arena_.as<Dtype>() + off);
            off += arena_slot(*b);
        }
}

template <typename Dtype>
void Net<Dtype>::ParamsChanged() {
    Caffe::stream() = stream_;
    // host-side edits (FromProto / fillers) -> arena
    for (auto& l : layers_) for (auto& b : l->blobs()) b->gpu_data();
    for (auto& l : layers_) l->ParamsChanged();
    params_ready_ = true;
    if (graph_exec_) { cudaGraphExecDestroy(graph_exec_); graph_exec_ = nullptr; }
    if (graph_) { cudaGraphDestroy(graph_); graph_ = nullptr; }
}

// The parameter arena was overwritten on the device (ncclBroadcast from rank 0): the device is authoritative, every cached
// host copy (conv weights, and the DataAugmentation iteration counter that HostTick reads on the host) is stale.
template <typename Dtype>
void Net<Dtype>::ArenaWritten() {
    CUDA_CHECK(cudaDeviceSynchronize());
    for (auto& l : layers_) for (auto& b : l->blobs()) b->MarkDeviceNewer();
    ParamsChanged();
}

template <typename Dtype>
void Net<Dtype>::FillParams(uint64_t seed) {
    for (size_t i = 0; i < layers_.size(); i++) layers_[i]->FillParams(seed * 1000003ULL + i);
    ParamsChanged();
}

static vector<int> strip_leading_ones(const vector<int>& s) {
    size_t i = 0;
    while (i + 1 < s.size() && s[i] == 1) i++;
    return vector<int>(s.begin() + i, s.end());
}

// Net::CopyTrainedLayersFrom(const NetParameter&), net.cpp:752-802
// Net::CopyTrainedLayersFromHDF5 (net.cpp:823-870): /data/<layer name>/<blob index>, unknown source layers ignored, a source
// layer may not have more blobs than the target, every target blob must be present; the blob takes the dataset's shape
// (hdf5_load_nd_dataset, util/hdf5.cpp:20-76).  Parsed by the minimal reader of hdf5_min.cpp (no HDF5 library in this image).
template <typename Dtype>
void Net<Dtype>::CopyTrainedLayersFromHDF5(const void* h5, size_t bytes, const string& prefix) {
    Caffe::stream() = stream_;
    H5File f(h5, bytes);
    CHECK(f.has("/data")) << "Error reading weights: the file has no /data group";
    std::map<string, int> index;
    for (size_t i = 0; i < layer_names_.size(); i++) index[layer_names_[i]] = (int)i;
    std::set<int> filled;
    for (const string& src : f.links("/data")) {
        auto it = index.find(prefix + src);
        if (it == index.end()) continue;                               // "Ignoring source layer"
        filled.insert(it->second);
        auto& target = layers_[it->second]->blobs();
        const string base = "/data/" + src;
        const vector<string> links = f.links(base);
        CHECK_LE(links.size(), target.size()) << "Incompatible number of blobs for layer " << src;
        vector<Blob<Dtype>*> staged;
        vector<shared_ptr<Blob<Dtype> > > tmp;
        for (size_t j = 0; j < target.size(); j++) {
            const string ds = base + "/" + std::to_string(j);
            CHECK(f.has(ds)) << "Incompatible number of blobs for layer " << src;
            vector<int> dims;
            vector<float> v = f.read(ds, &dims);
            CHECK_LE(dims.size(), 4u) << "dataset " << ds << " has more than 4 axes";
            if (layers_[it->second]->DoesUseCustomCopyBlobs()) {           // DataAugmentation adjusts sizes itself (net.cpp:769-778)
                shared_ptr<Blob<Dtype> > b(new Blob<Dtype>());
                b->Reshape(dims);
                if (!v.empty()) memcpy(b->mutable_cpu_data(), v.data(), v.size() * sizeof(float));
                tmp.push_back(b); staged.push_back(b.get());
                continue;
            }
            CHECK_EQ((size_t)target[j]->count(), v.size()) << "Cannot copy param " << j << " weights from layer '" << src
                << "'; shape mismatch (" << v.size() << " values in the file)";
            target[j]->Reshape(dims);
            if (!v.empty()) memcpy(target[j]->mutable_cpu_data(), v.data(), v.size() * sizeof(float));
        }
        if (!staged.empty()) layers_[it->second]->CustomCopyBlobs(staged);
    }
    FillTemplateDefined(filled);
    ParamsChanged();
}

// Caffe fills every layer from its prototxt fillers before it copies trained layers; this net does not (its parameters start
// at zero), so a layer whose weights the template alone defines (TemplateDefinedParams: the deploy nets' diagonal
// scale_conv1) is filled here when the source leaves it out, as a training snapshot does.
template <typename Dtype>
void Net<Dtype>::FillTemplateDefined(const std::set<int>& filled) {
    for (size_t i = 0; i < layers_.size(); i++)
        if (!filled.count((int)i) && layers_[i]->TemplateDefinedParams()) layers_[i]->FillParams(0);
}

template <typename Dtype>
void Net<Dtype>::CopyTrainedLayersFrom(const void* caffemodel, size_t bytes, const string& prefix) {
    static const unsigned char h5sig[8] = {0x89, 'H', 'D', 'F', '\r', '\n', 0x1a, '\n'};
    if (bytes >= 8 && !memcmp(caffemodel, h5sig, 8)) { CopyTrainedLayersFromHDF5(caffemodel, bytes, prefix); return; }   // .caffemodel.h5
    Caffe::stream() = stream_;
    vector<LayerBlobs> src = ParseCaffemodel(caffemodel, bytes);
    std::set<int> filled;
    for (const LayerBlobs& sl : src) {
        size_t ti = 0;
        while (ti != layer_names_.size() && layer_names_[ti] != prefix + sl.name) ++ti;
        if (ti == layer_names_.size()) continue;                               // "Ignoring source layer"
        filled.insert((int)ti);
        auto& target = layers_[ti]->blobs();
        if (layers_[ti]->DoesUseCustomCopyBlobs()) {                            // net.cpp:769-780 (fork)
            vector<shared_ptr<Blob<Dtype> > > tmp;
            vector<Blob<Dtype>*> ptrs;
            for (const auto& bp : sl.blobs) {
                tmp.emplace_back(new Blob<Dtype>());
                vector<int> s = bp.shape;
                while (s.size() < 4) s.insert(s.begin(), 1);
                BlobProtoData p4 = bp; p4.shape = s;
                tmp.back()->FromProto(p4, true);
                ptrs.push_back(tmp.back().get());
            }
            layers_[ti]->CustomCopyBlobs(ptrs);
            continue;
        }
        CHECK_EQ(target.size(), sl.blobs.size()) << "Incompatible number of blobs for layer " << sl.name;
        for (size_t j = 0; j < target.size(); ++j) {
            const bool same = strip_leading_ones(target[j]->shape()) == strip_leading_ones(sl.blobs[j].shape);
            CHECK(same) << "Cannot copy param " << j << " weights from layer '" << sl.name
                        << "'; shape mismatch (net.cpp:782-795)";
            target[j]->FromProto(sl.blobs[j], false);
        }
    }
    FillTemplateDefined(filled);
    ParamsChanged();
}

template <typename Dtype>
std::string Net<Dtype>::ToCaffemodel() {
    Caffe::stream() = stream_;
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    vector<LayerBlobs> out;
    for (size_t i = 0; i < layers_.size(); i++) {
        if (layers_[i]->blobs().empty()) continue;
        LayerBlobs lb;
        lb.name = layer_names_[i];
        lb.type = layers_[i]->type();
        for (auto& b : layers_[i]->blobs()) {
            lb.blobs.emplace_back();
            b->ToProto(&lb.blobs.back());
        }
        out.push_back(std::move(lb));
    }
    return SerializeCaffemodel(name_, out);
}

// Two-stream plan.  Dependencies are tracked on storage (an aliased concat bottom counts as its parent): read-after-write,
// write-after-write and write-after-read.  Greedy list scheduling in prototxt order with a crude cost model: a layer goes
// to the second stream only when that lets it start clearly earlier than on the main stream.
template <typename Dtype>
void Net<Dtype>::PlanStreams() {
    const int L = (int)layers_.size();
    layer_stream_.assign(L, 0); layer_wait_.assign(L, -1); layer_record_.assign(L, 0); layer_event_.assign(L, nullptr);
    uses_stream2_ = false;
    if (getenv("FN2_NO_STREAMS") || L == 0) return;
    std::map<const Blob<Dtype>*, int> root_of;
    auto root = [&](const Blob<Dtype>* b) {
        while (b->alias_parent()) b = b->alias_parent();
        auto it = root_of.find(b);
        if (it == root_of.end()) it = root_of.insert({b, (int)root_of.size()}).first;
        return it->second;
    };
    std::map<int, int> last_writer;                       // storage -> layer
    std::map<int, vector<int> > readers;                  // storage -> layers that read it since the last write
    vector<vector<int> > deps(L);
    for (int i = 0; i < L; i++) {
        std::set<int> d;
        for (Blob<Dtype>* b : bottom_vecs_[i]) { const int r = root(b); if (last_writer.count(r)) d.insert(last_writer[r]); }
        for (Blob<Dtype>* t : top_vecs_[i]) {
            const int r = root(t);
            if (last_writer.count(r)) d.insert(last_writer[r]);
            for (int j : readers[r]) d.insert(j);
        }
        d.erase(i);
        deps[i].assign(d.begin(), d.end());
        for (Blob<Dtype>* b : bottom_vecs_[i]) readers[root(b)].push_back(i);
        for (Blob<Dtype>* t : top_vecs_[i]) { const int r = root(t); last_writer[r] = i; readers[r].clear(); }
    }
    vector<double> finish(L, 0.0);
    double busy[2] = {0.0, 0.0};
    for (int i = 0; i < L; i++) {
        double fl = 0, by = 0;
        layers_[i]->WorkEstimate(bottom_vecs_[i], top_vecs_[i], &fl, &by);
        const double cost = std::max(fl / 100e12, by / 1.5e12) + 4e-6;
        double ready = 0;
        for (int j : deps[i]) ready = std::max(ready, finish[j]);
        const double s0 = std::max(ready, busy[0]), s1 = std::max(ready, busy[1]);
        int s = (s1 + 30e-6 < s0) ? 1 : 0;
        // stay with the producer when that costs nothing
        if (s == 0 && s1 <= s0) for (int j : deps[i]) if (finish[j] == ready && layer_stream_[j] == 1 && busy[1] <= ready) s = 1;
        layer_stream_[i] = s;
        finish[i] = (s ? s1 : s0) + cost;
        busy[s] = finish[i];
        if (s) uses_stream2_ = true;
    }
    if (!uses_stream2_) return;
    for (int i = 0; i < L; i++) {
        int w = -1;
        for (int j : deps[i]) if (layer_stream_[j] != layer_stream_[i]) w = std::max(w, j);
        layer_wait_[i] = w;
        if (w >= 0) layer_record_[w] = 1;
    }
    CUDA_CHECK(cudaStreamCreateWithFlags(&stream2_, cudaStreamNonBlocking));
    for (int i = 0; i < L; i++) if (layer_record_[i]) CUDA_CHECK(cudaEventCreateWithFlags(&layer_event_[i], cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&fork_event_, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&join_event_, cudaEventDisableTiming));
    if (getenv("FN2_DEBUG_STREAMS")) {
        int n1 = 0;
        for (int i = 0; i < L; i++) n1 += layer_stream_[i];
        fprintf(stderr, "[fn2] %d of %d layers on the second stream:", n1, L);
        for (int i = 0; i < L; i++) if (layer_stream_[i]) fprintf(stderr, " %s", layer_names_[i].c_str());
        fprintf(stderr, "\n");
    }
}

template <typename Dtype>
void Net<Dtype>::ForwardEager() {
    if (!uses_stream2_) {
        for (size_t i = 0; i < layers_.size(); ++i) RunLayer((int)i);
        return;
    }
    // fork: everything already queued on the main stream (input copies) precedes the second stream's work; under graph
    // capture this is also what pulls the second stream into the capture
    CUDA_CHECK(cudaEventRecord(fork_event_, stream_));
    CUDA_CHECK(cudaStreamWaitEvent(stream2_, fork_event_, 0));
    for (size_t i = 0; i < layers_.size(); ++i) {
        cudaStream_t st = layer_stream_[i] ? stream2_ : stream_;
        if (layer_wait_[i] >= 0) CUDA_CHECK(cudaStreamWaitEvent(st, layer_event_[layer_wait_[i]], 0));
        Caffe::stream() = st;
        RunLayer((int)i);
        if (layer_record_[i]) CUDA_CHECK(cudaEventRecord(layer_event_[i], st));
    }
    Caffe::stream() = stream_;
    CUDA_CHECK(cudaEventRecord(join_event_, stream2_));
    CUDA_CHECK(cudaStreamWaitEvent(stream_, join_event_, 0));
}

// Net::ForwardFromTo(0, L-1), net.cpp:546-557 -- replayed from a CUDA graph once warm.
template <typename Dtype>
void Net<Dtype>::Forward() {
    Caffe::stream() = stream_;
    if (!params_ready_) ParamsChanged();
    bool safe = !graph_disabled_;
    for (auto& l : layers_) l->HostTick(iter_);
    for (auto& l : layers_) if (!l->GraphSafe()) safe = false;
    if (safe && graph_exec_) {
        CUDA_CHECK(cudaGraphLaunch(graph_exec_, stream_));
        MarkActivationsOnDevice();
        return;
    }
    if (safe && launches_per_forward_ > 0) {
        // second safe call: every lazy allocation happened during the first eager pass
        cudaError_t e = cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            bool ok = true;
            std::string why;
            try { ForwardEager(); } catch (const std::exception& ex) { ok = false; why = ex.what(); }
            cudaGraph_t g = nullptr;
            e = cudaStreamEndCapture(stream_, &g);
            if (ok && e == cudaSuccess && g) {
                cudaGraphExec_t ge = nullptr;
                if (cudaGraphInstantiate(&ge, g, 0) == cudaSuccess) {
                    graph_ = g; graph_exec_ = ge;
                    CUDA_CHECK(cudaGraphLaunch(graph_exec_, stream_));
                    MarkActivationsOnDevice();
                    return;
                }
            }
            if (g) cudaGraphDestroy(g);
            cudaGetLastError();
            graph_disabled_ = true;
            CHECK(ok) << "forward failed during graph capture: " << why;
        } else {
            cudaGetLastError();
            graph_disabled_ = true;
        }
    }
    const uint64_t before = fn2_launch_count();
    ForwardEager();
    launches_per_forward_ = (int)(fn2_launch_count() - before);
}

// A graph replay writes every non-input activation without going through Blob::mutable_tensor: cached host copies
// (Blob::cpu_data() after an earlier pass) are stale from here on.
template <typename Dtype>
void Net<Dtype>::MarkActivationsOnDevice() {
    std::set<int> inputs(net_input_blob_indices_.begin(), net_input_blob_indices_.end());
    for (size_t i = 0; i < blobs_.size(); i++) if (!inputs.count((int)i)) blobs_[i]->MarkDeviceNewer();
}

// ---- backward -----------------------------------------------------------------------------------------------------------
template <typename Dtype>
float Net<Dtype>::lr_mult(int layer, int param) const {
    const LayerParameter& lp = layers_[layer]->layer_param();
    return param < lp.m->count("param") ? lp.m->msg("param", param).f("lr_mult", 1.f) : 1.f;      // ParamSpec default 1
}

template <typename Dtype>
float Net<Dtype>::decay_mult(int layer, int param) const {
    const LayerParameter& lp = layers_[layer]->layer_param();
    return param < lp.m->count("param") ? lp.m->msg("param", param).f("decay_mult", 1.f) : 1.f;   // ParamSpec default 1
}

template <typename Dtype>
vector<typename Net<Dtype>::LearnableParam> Net<Dtype>::LearnableParams() {
    vector<LearnableParam> out;
    size_t off = 0;
    for (size_t i = 0; i < layers_.size(); i++)
        for (size_t pi = 0; pi < layers_[i]->blobs().size(); pi++) {
            const Blob<Dtype>& b = *layers_[i]->blobs()[pi];
            out.push_back({(int)i, (int)pi, off, b.count(), b.shape(), lr_mult((int)i, (int)pi), decay_mult((int)i, (int)pi)});
            off += arena_slot(b);
        }
    return out;
}

template <typename Dtype>
void Net<Dtype>::ParamsUpdated(const vector<int>& learnable_ids) {
    vector<Blob<Dtype>*> all;
    vector<int> layer_of;
    for (size_t i = 0; i < layers_.size(); i++)
        for (auto& b : layers_[i]->blobs()) { all.push_back(b.get()); layer_of.push_back((int)i); }
    std::set<int> touched;
    for (int id : learnable_ids) { all[id]->MarkDeviceNewer(); touched.insert(layer_of[id]); }
    Caffe::stream() = stream_;
    for (int i : touched) layers_[i]->ParamsChanged();
}

template <typename Dtype>
Dtype Net<Dtype>::blob_loss_weight(int b) const {
    for (size_t i = 0; i < layers_.size(); i++)
        for (size_t t = 0; t < top_id_vecs_[i].size(); t++)
            if (top_id_vecs_[i][t] == b && layers_[i]->loss_weight((int)t) != 0) return layers_[i]->loss_weight((int)t);
    return 0;
}

// Which layers need backward and which blobs carry a gradient, from the graph alone (net.cpp:120-170, :223-262): a layer needs
// backward if it has a parameter with lr_mult != 0 or a bottom that needs it (every input blob with force_backward), and it
// allows backward.  propagate_down: false then cuts single bottoms in PlanBackward.  The warp-block fusion and the trainable
// span of the gradient arena follow the same rule.
template <typename Dtype>
void Net<Dtype>::NeedBackward(vector<char>* layer_need, vector<char>* blob_need) const {
    const int L = (int)layers_.size();
    layer_need->assign(L, 0);
    blob_need->assign(blobs_.size(), 0);
    if (force_backward_) for (int b : net_input_blob_indices_) (*blob_need)[b] = 1;       // net.cpp:96-100, :262-267
    for (int i = 0; i < L; i++) {
        bool need = false;
        for (size_t pi = 0; pi < layers_[i]->blobs().size(); pi++) if (lr_mult(i, (int)pi) != 0.f) need = true;
        for (int b : bottom_id_vecs_[i]) if ((*blob_need)[b]) need = true;
        if (!layers_[i]->AllowBackward()) need = false;
        (*layer_need)[i] = need;
        for (int t : top_id_vecs_[i]) if (need) (*blob_need)[t] = 1;
    }
}

// Same decisions as Net::Init's backward bookkeeping (net.cpp:120-170 need_backward / blobs_under_loss, :210-262), made once:
//  * a layer needs backward if it has parameters or a bottom that needs it, and AllowBackward();
//  * it runs only if one of its tops lies under a loss (or under a SetDiff seed);
//  * no Split layers exist here, so a blob read by several layers receives several contributions: the first consumer to run
//    overwrites the diff, the later ones add (Layer::set_bottom_accumulate).  Zero-copy concat children share their parent's
//    diff storage; a child written before its parent forces the parent to be cleared first and everybody to add.
template <typename Dtype>
void Net<Dtype>::PlanBackward() {
    if (bw_planned_) return;
    const int L = (int)layers_.size(), B = (int)blobs_.size();
    vector<char> layer_need, blob_need, under_loss(B, 0);
    NeedBackward(&layer_need, &blob_need);
    for (int s : bw_seeds_) under_loss[s] = 1;
    vector<std::pair<int, Dtype> > loss_tops;
    for (int i = 0; i < L; i++)
        for (size_t t = 0; t < top_id_vecs_[i].size(); t++) {
            const Dtype w = layers_[i]->loss_weight((int)t);
            if (w != 0) { under_loss[top_id_vecs_[i][t]] = 1; loss_tops.push_back({top_id_vecs_[i][t], w}); }
        }
    bw_run_.assign(L, 0);
    for (int i = L - 1; i >= 0; i--) {
        bool contributes = false;
        for (int t : top_id_vecs_[i]) if (under_loss[t]) contributes = true;
        if (!contributes) continue;
        for (int b : bottom_id_vecs_[i]) under_loss[b] = 1;
        bw_run_[i] = layer_need[i];
    }
    // write simulation in execution order
    vector<vector<int> > children(B);
    std::map<const Blob<Dtype>*, int> id_of;
    for (int b = 0; b < B; b++) id_of[blobs_[b].get()] = b;
    auto parent_of = [&](int b) { return blobs_[b]->is_alias() ? id_of[blobs_[b]->alias_parent()] : -1; };
    for (int b = 0; b < B; b++) if (parent_of(b) >= 0) children[parent_of(b)].push_back(b);
    vector<char> written(B, 0);
    std::set<int> zero;
    auto clear_root = [&](int root) {
        zero.insert(root);
        written[root] = 1;
        for (int c : children[root]) written[c] = 1;
    };
    for (int s : bw_seeds_) { written[s] = 1; for (int c : children[s]) written[c] = 1; }
    for (auto& lt : loss_tops) written[lt.first] = 1;
    bw_propagate_.assign(L, {});
    bw_accumulate_.assign(L, {});
    for (int i = L - 1; i >= 0; i--) {
        bw_propagate_[i].assign(bottom_id_vecs_[i].size(), false);
        bw_accumulate_[i].assign(bottom_id_vecs_[i].size(), false);
        if (!bw_run_[i]) continue;
        // tops nobody wrote (consumers outside the loss): their gradient is zero
        for (int t : top_id_vecs_[i])
            if (!written[t]) { const int p = parent_of(t); clear_root(p >= 0 ? p : t); }
        const LayerParameter& lp = layers_[i]->layer_param();
        for (size_t b = 0; b < bottom_id_vecs_[i].size(); b++) {
            const int id = bottom_id_vecs_[i][b];
            bool prop = blob_need[id] != 0;
            if (lp.m->count("propagate_down") > (int)b) {                                // LayerParameter.propagate_down, net.cpp:97-104
                const std::string& v = lp.m->str("propagate_down", (int)b);
                if (v == "false" || v == "False" || v == "0") prop = false;
            }
            bw_propagate_[i][b] = prop;
            if (!prop) continue;
            bool inplace = false;
            for (int t : top_id_vecs_[i]) if (t == id) inplace = true;
            if (inplace) continue;
            if (written[id]) { bw_accumulate_[i][b] = true; continue; }
            const int p = parent_of(id);
            if (p >= 0) { clear_root(p); bw_accumulate_[i][b] = true; continue; }     // child first: clear the parent, everybody adds
            written[id] = 1;
            for (int c : children[id]) written[c] = 1;
        }
    }
    bw_zero_.assign(zero.begin(), zero.end());
    BuildDiffArena();
    for (int i = 0; i < L; i++) layers_[i]->set_bottom_accumulate(bw_accumulate_[i]);
    // loss seeds: top diff = loss_weight (scalar tops)
    for (auto& lt : loss_tops) {
        if (bw_seeds_.count(lt.first)) continue;                     // an explicit SetDiff on a loss top wins over its loss_weight
        Blob<Dtype>* bl = blobs_[lt.first].get();
        vector<Dtype> v((size_t)bl->count(), lt.second);
        bl->set_cpu_diff(v.data());
    }
    bw_planned_ = true;
}

template <typename Dtype>
void Net<Dtype>::BuildDiffArena() {
    if (!diff_arena_.empty() || !arena_floats_) return;
    diff_arena_.reserve(arena_floats_ * sizeof(Dtype), stream_);
    size_t off = 0;
    for (auto& l : layers_)
        for (auto& b : l->blobs()) {
            b->BindExternalDiff(diff_arena_.as<Dtype>() + off);
            off += arena_slot(*b);
        }
}

template <typename Dtype>
void Net<Dtype>::ParamDiffArena(void** dev, size_t* bytes) {
    BuildDiffArena();
    *dev = diff_arena_.get(); *bytes = arena_floats_ * sizeof(Dtype);
}

// Parameters the backward pass writes (lr_mult != 0 in a layer that needs backward) as one range of the gradient arena: a
// stage trained on top of frozen predecessors all-reduces this range only, not the predecessors' gradients, which stay zero.
template <typename Dtype>
void Net<Dtype>::TrainableDiffSpan(void** dev, size_t* bytes) {
    BuildDiffArena();
    vector<char> layer_need, blob_need;
    NeedBackward(&layer_need, &blob_need);
    size_t off = 0, lo = arena_floats_, hi = 0;
    for (size_t i = 0; i < layers_.size(); i++)
        for (size_t pi = 0; pi < layers_[i]->blobs().size(); pi++) {
            const size_t padded = arena_slot(*layers_[i]->blobs()[pi]);
            if (layer_need[i] && lr_mult((int)i, (int)pi) != 0.f) { lo = std::min(lo, off); hi = off + padded; }
            off += padded;
        }
    if (hi == 0) lo = 0;
    *dev = diff_arena_.as<Dtype>() + lo; *bytes = (hi - lo) * sizeof(Dtype);
}

template <typename Dtype>
void Net<Dtype>::ClearParamDiffs() {
    BuildDiffArena();
    if (!diff_arena_.empty()) CUDA_CHECK(cudaMemsetAsync(diff_arena_.get(), 0, arena_floats_ * sizeof(Dtype), stream_));
}

template <typename Dtype>
void Net<Dtype>::Backward() {
    Caffe::stream() = stream_;
    if (!params_ready_) ParamsChanged();
    PlanBackward();
    const uint64_t before = fn2_launch_count();
    for (int b : bw_zero_) blobs_[b]->ZeroDiff(stream_);
    static const bool profile = getenv("FN2_BWD_PROFILE") != nullptr;      // per-layer device times of this pass on stderr
    vector<cudaEvent_t> ev;
    if (profile) { ev.resize(layers_.size() + 1); for (auto& e : ev) cudaEventCreate(&e); cudaEventRecord(ev[layers_.size()], stream_); }
    for (int i = (int)layers_.size() - 1; i >= 0; i--) {
        if (bw_run_[i]) layers_[i]->Backward(top_vecs_[i], bw_propagate_[i], bottom_vecs_[i]);
        if (profile) cudaEventRecord(ev[i], stream_);
    }
    launches_per_backward_ = (int)(fn2_launch_count() - before);
    if (profile) {
        CUDA_CHECK(cudaStreamSynchronize(stream_));
        float total = 0;
        for (int i = (int)layers_.size() - 1; i >= 0; i--) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ev[i + 1], ev[i]);
            total += ms;
            if (bw_run_[i]) fprintf(stderr, "[fn2 bwd] %-24s %-16s %8.3f ms\n", layer_names_[i].c_str(), layers_[i]->type(), ms);
        }
        fprintf(stderr, "[fn2 bwd] total %.3f ms, %d launches\n", total, launches_per_backward_);
        for (auto& e : ev) cudaEventDestroy(e);
    }
}

template <typename Dtype>
void Net<Dtype>::SetDiff(const string& blob, const Dtype* host_nchw) {
    Caffe::stream() = stream_;
    auto it = blob_names_index_.find(blob);
    CHECK(it != blob_names_index_.end()) << "Unknown blob name " << blob;
    if (!bw_seeds_.count(it->second)) { bw_seeds_.insert(it->second); bw_planned_ = false; }
    blobs_[it->second]->set_cpu_diff(host_nchw);
}

template <typename Dtype>
void Net<Dtype>::GetDiff(const string& blob, Dtype* host_nchw) {
    Caffe::stream() = stream_;
    Blob<Dtype>* bl = blob_by_name(blob).get();
    const Dtype* d = bl->cpu_diff();
    std::memcpy(host_nchw, d, (size_t)bl->count() * sizeof(Dtype));
}

template <typename Dtype>
void Net<Dtype>::Sync() {
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

template <typename Dtype>
Dtype* Net<Dtype>::staging(const string& blob, size_t floats) {
    DeviceBuffer& s = staging_[blob];
    s.reserve(floats * sizeof(Dtype));
    return s.as<Dtype>();
}

template <typename Dtype>
void Net<Dtype>::SetInputDevice(const string& blob, const Dtype* dev_nchw) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    fn2_tensor src = nchw_view(const_cast<Dtype*>(dev_nchw), b->num(), b->channels(), b->height(), b->width());
    fn2_tensor dst = b->mutable_tensor();
    FN2_CALL(fn2_copy(&src, &dst, stream_));
}

template <typename Dtype>
void Net<Dtype>::SetInput(const string& blob, const Dtype* host_nchw) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    Dtype* st = staging(blob, (size_t)b->count());
    CUDA_CHECK(cudaMemcpyAsync(st, host_nchw, (size_t)b->count() * sizeof(Dtype), cudaMemcpyHostToDevice, stream_));
    SetInputDevice(blob, st);
}

template <typename Dtype>
void Net<Dtype>::GetBlobDevice(const string& blob, Dtype* dev_nchw) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    fn2_tensor src = b->tensor();
    fn2_tensor dst = nchw_view(dev_nchw, b->num(), b->channels(), b->height(), b->width());
    FN2_CALL(fn2_copy(&src, &dst, stream_));
}

template <typename Dtype>
void Net<Dtype>::GetBlob(const string& blob, Dtype* host_nchw) {
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    Dtype* st = staging(blob + "#out", (size_t)b->count());
    GetBlobDevice(blob, st);
    CUDA_CHECK(cudaMemcpyAsync(host_nchw, st, (size_t)b->count() * sizeof(Dtype), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// The input blob frames go to: refuses a channel count other than 1, 3, 4 and a blob that is not (N, 3, H, W).
template <typename Dtype>
static shared_ptr<Blob<Dtype> > frames_blob(const Net<Dtype>& net, const string& blob, int channels) {
    CHECK(channels == 1 || channels == 3 || channels == 4) << "set_input_frames: channels must be 1, 3 or 4 (gray, RGB, RGBA), got "
                                                           << channels;
    shared_ptr<Blob<Dtype> > b = net.blob_by_name(blob);
    CHECK(b->num_axes() == 4 && b->channels() == 3) << "set_input_frames: blob " << blob << " must have shape (N, 3, H, W), has "
                                                    << b->num_axes() << " axes and " << b->channels() << " channels";
    return b;
}

template <typename Dtype>
void Net<Dtype>::SetInputFramesDevice(const string& blob, const void* dev_frames, int channels) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = frames_blob(*this, blob, channels);
    fn2_tensor dst = b->mutable_tensor();
    FN2_CALL(fn2_frames_to_tensor(dev_frames, channels, &dst, stream_));
}

template <typename Dtype>
void Net<Dtype>::SetInputFrames(const string& blob, const void* host_frames, int channels) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = frames_blob(*this, blob, channels);
    const size_t bytes = (size_t)b->num() * b->height() * b->width() * channels;
    Dtype* st = staging(blob, (bytes + sizeof(Dtype) - 1) / sizeof(Dtype));        // the buffer SetInput stages the blob in
    CUDA_CHECK(cudaMemcpyAsync(st, host_frames, bytes, cudaMemcpyHostToDevice, stream_));
    SetInputFramesDevice(blob, st, channels);
}

// The input blob a flow goes to: refuses a blob that is not (N, 2, H, W).
template <typename Dtype>
static shared_ptr<Blob<Dtype> > flow_blob(const Net<Dtype>& net, const string& blob) {
    shared_ptr<Blob<Dtype> > b = net.blob_by_name(blob);
    CHECK(b->num_axes() == 4 && b->channels() == 2) << "set_input_flow: blob " << blob << " must have shape (N, 2, H, W), has "
                                                    << b->num_axes() << " axes and " << b->channels() << " channels";
    return b;
}

template <typename Dtype>
void Net<Dtype>::SetInputFlowDevice(const string& blob, const void* dev, int format, int flags) {
    Caffe::stream() = stream_;
    fn2_tensor dst = flow_blob(*this, blob)->mutable_tensor();
    FN2_CALL(fn2_flow_to_tensor(dev, format, flags, &dst, stream_));
}

template <typename Dtype>
void Net<Dtype>::GetBlobNHWCDevice(const string& blob, Dtype* dev_nhwc) {
    Caffe::stream() = stream_;
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    fn2_tensor src = b->tensor();
    fn2_tensor dst = nhwc_view(dev_nhwc, b->num(), b->channels(), b->height(), b->width());
    FN2_CALL(fn2_copy(&src, &dst, stream_));
}

template <typename Dtype>
void Net<Dtype>::GetBlobNHWC(const string& blob, Dtype* host_nhwc) {
    shared_ptr<Blob<Dtype> > b = blob_by_name(blob);
    Dtype* st = staging(blob + "#out", (size_t)b->count());
    GetBlobNHWCDevice(blob, st);
    CUDA_CHECK(cudaMemcpyAsync(host_nhwc, st, (size_t)b->count() * sizeof(Dtype), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// Per-layer timing in the style of `caffe time` (tools/caffe.cpp:346-385): CUDA events around
// each layer's Forward on the net's stream.
template <typename Dtype>
void Net<Dtype>::TimeLayers(float* ms) {
    Caffe::stream() = stream_;
    if (!params_ready_) ParamsChanged();
    for (auto& l : layers_) l->HostTick(iter_);
    vector<cudaEvent_t> ev(layers_.size() + 1);
    for (auto& e : ev) CUDA_CHECK(cudaEventCreate(&e));
    CUDA_CHECK(cudaEventRecord(ev[0], stream_));
    for (size_t i = 0; i < layers_.size(); ++i) {
        RunLayer((int)i);
        CUDA_CHECK(cudaEventRecord(ev[i + 1], stream_));
    }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    for (size_t i = 0; i < layers_.size(); ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
    for (auto& e : ev) cudaEventDestroy(e);
}

template class Net<float>;

}  // namespace caffe
