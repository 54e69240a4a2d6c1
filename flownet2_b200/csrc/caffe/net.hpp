// Net: in-order graph executor over the Layer surface (reference: include/caffe/net.hpp,
// src/caffe/net.cpp Init :40-286, AppendTop/AppendBottom :386-448, ForwardFromTo :546-557,
// CopyTrainedLayersFrom :752-802).  New underneath: one stream, fused conv+ReLU, zero-copy
// channel Concat, one contiguous parameter arena, CUDA-graph replay of the whole forward pass.
#pragma once
#include <map>
#include <set>

#include "layer.hpp"

namespace caffe {

template <typename Dtype>
class Net {
 public:
    Net(const NetParameter& param, Phase phase);
    ~Net();

    void Forward();                                    // async on stream()
    // Net::Backward (net.cpp:640-655 BackwardFromTo(L-1, 0)).  Gradients start at the loss tops (loss_weight, layer.hpp:455-478)
    // and at every blob whose diff was given through SetDiff.  Parameter diffs ACCUMULATE like the reference's
    // (ClearParamDiffs = net.cpp:935-955, what Solver::Step calls first).
    void Backward();
    void ClearParamDiffs();
    void SetDiff(const string& blob, const Dtype* host_nchw);
    void GetDiff(const string& blob, Dtype* host_nchw);
    void ParamDiffArena(void** dev, size_t* bytes);
    void TrainableDiffSpan(void** dev, size_t* bytes);
    int launches_per_backward() const { return launches_per_backward_; }
    const vector<char>& layer_need_backward() { PlanBackward(); return bw_run_; }
    void Sync();
    // Net::set_iter / iter (net.hpp:230-231): the iteration the layers see in HostTick (LpqLoss's p/q schedule).  The Solver
    // sets it at the start of every iteration (solver.cpp:202); a net no solver drives stays at 0.
    void set_iter(int iter) { iter_ = iter; }
    int iter() const { return iter_; }
    cudaStream_t stream() const { return stream_; }

    // net.cpp:752-802 (binary proto) / :823-870 (HDF5, by signature).  Source layer X fills target layer prefix + X (a stage's
    // trained sub-network inside the next stage's graph: conv1 -> net1_conv1); source layers with no target are ignored.
    void CopyTrainedLayersFrom(const void* caffemodel, size_t bytes, const string& prefix = "");
    void CopyTrainedLayersFromHDF5(const void* h5, size_t bytes, const string& prefix = "");
    void FillTemplateDefined(const std::set<int>& filled);
    std::string ToCaffemodel();
    void FillParams(uint64_t seed);
    void ParamsChanged();
    void ArenaWritten();                               // device arena overwritten externally (broadcast)
    void ParamArena(void** dev, size_t* bytes) { *dev = arena_.get(); *bytes = arena_floats_ * sizeof(Dtype); }

    // Net::learnable_params (net.cpp:440-490): every layer's parameter blobs in layer order x parameter index, where each one
    // lies in the parameter and gradient arenas, and its ParamSpec multipliers (lr_mult, decay_mult; default 1).
    struct LearnableParam { int layer, index; size_t offset; int count; vector<int> shape; float lr_mult, decay_mult; };
    vector<LearnableParam> LearnableParams();
    float lr_mult(int layer, int param) const;
    float decay_mult(int layer, int param) const;
    // Net::Update (net.cpp:957-964) ran on the device for the given learnable parameters: their device copies are newer, and
    // their layers re-derive what they keep from them (packed convolution weights) on the net's stream.  No host sync.
    void ParamsUpdated(const vector<int>& learnable_ids);
    // loss weight of blob b as a loss layer top (Net::blob_loss_weights, net.cpp:189-196), 0 for other blobs
    Dtype blob_loss_weight(int b) const;

    const vector<string>& layer_names() const { return layer_names_; }
    const vector<shared_ptr<Layer<Dtype> > >& layers() const { return layers_; }
    const vector<string>& blob_names() const { return blob_names_; }
    const vector<shared_ptr<Blob<Dtype> > >& blobs() const { return blobs_; }
    const vector<int>& input_blob_indices() const { return net_input_blob_indices_; }
    const vector<int>& output_blob_indices() const { return net_output_blob_indices_; }
    bool has_blob(const string& name) const { return blob_names_index_.count(name) > 0; }
    shared_ptr<Blob<Dtype> > blob_by_name(const string& name) const;

    // NCHW host/device buffers <-> blob (layout conversion on the net's stream)
    void SetInput(const string& blob, const Dtype* host_nchw);
    void SetInputDevice(const string& blob, const Dtype* dev_nchw);
    void GetBlob(const string& blob, Dtype* host_nchw);
    void GetBlobDevice(const string& blob, Dtype* dev_nchw);
    // 8-bit frames [N][H][W][channels] (1, 3 or 4) -> an (N, 3, H, W) input blob as BGR floats (fn2_frames_to_tensor), and a
    // blob read back as dense NHWC (include/fn2_frames.h)
    void SetInputFrames(const string& blob, const void* host_frames, int channels);
    void SetInputFramesDevice(const string& blob, const void* dev_frames, int channels);
    // flow file payloads on the device -> an (N, 2, H, W) input blob (fn2_flow_to_tensor)
    void SetInputFlowDevice(const string& blob, const void* dev, int format, int flags);
    void GetBlobNHWC(const string& blob, Dtype* host_nhwc);
    void GetBlobNHWCDevice(const string& blob, Dtype* dev_nhwc);

    void TimeLayers(float* ms);
    void LayerWork(int i, double* flops, double* bytes) const { layers_[i]->WorkEstimate(bottom_vecs_[i], top_vecs_[i], flops, bytes); }
    int launches_per_forward() const { return launches_per_forward_; }
    bool graph_active() const { return graph_exec_ != nullptr; }

 private:
    void Init(const NetParameter& param);
    void FuseReLUs();
    void AliasConcats();
    void BuildArena();
    void ForwardEager();
    void MarkActivationsOnDevice();
    void PlanStreams();
    Dtype* staging(const string& blob, size_t floats);
    void FuseWarpBlocks();
    void RunLayer(int i);
    // warp block between stacked networks run as one kernel at the Resample layer's position (fn2_warp_block_forward); the
    // other four layers of the chain become no-ops
    struct WarpBlock { int resample, warp, sub, norm, scale; float coeff; int fill_nan; };
    std::map<int, WarpBlock> warp_head_;        // by the Resample layer's index
    vector<char> absorbed_;
    void NeedBackward(vector<char>* layer_need, vector<char>* blob_need) const;
    void PlanBackward();
    void BuildDiffArena();
    // backward plan (static per graph + seed set): which layers run, per bottom whether the gradient is wanted and whether it is
    // added to a diff an earlier-run consumer already wrote; blobs cleared before the sweep
    bool force_backward_ = false;
    bool bw_planned_ = false;
    vector<char> bw_run_;
    vector<vector<bool> > bw_propagate_, bw_accumulate_;
    vector<int> bw_zero_;
    std::set<int> bw_seeds_;
    DeviceBuffer diff_arena_;
    int launches_per_backward_ = 0;

    Phase phase_;
    int iter_ = 0;
    string name_;
    vector<shared_ptr<Layer<Dtype> > > layers_;
    vector<string> layer_names_;
    vector<vector<Blob<Dtype>*> > bottom_vecs_, top_vecs_;
    vector<vector<int> > bottom_id_vecs_, top_id_vecs_;
    vector<shared_ptr<Blob<Dtype> > > blobs_;
    vector<string> blob_names_;
    std::map<string, int> blob_names_index_;
    vector<int> net_input_blob_indices_, net_output_blob_indices_;
    DeviceBuffer arena_;
    size_t arena_floats_ = 0;
    cudaStream_t stream_ = nullptr;
    // second stream for layers off the critical path (FlowNet2: the FlowNet-SD branch next to the C-S-S chain), so that
    // their tiles fill the idle SMs at the tail of the other branch's kernels
    cudaStream_t stream2_ = nullptr;
    vector<int> layer_stream_;                  // 0 / 1 per layer (PlanStreams)
    vector<int> layer_wait_;                    // last layer on the OTHER stream this layer depends on, or -1
    vector<char> layer_record_;                 // an event is recorded after this layer
    vector<cudaEvent_t> layer_event_;
    cudaEvent_t fork_event_ = nullptr, join_event_ = nullptr;
    bool uses_stream2_ = false;
    cudaGraph_t graph_ = nullptr;
    cudaGraphExec_t graph_exec_ = nullptr;
    bool graph_disabled_ = false;
    bool params_ready_ = false;
    int launches_per_forward_ = 0;
    std::map<string, DeviceBuffer> staging_;
};

}  // namespace caffe
