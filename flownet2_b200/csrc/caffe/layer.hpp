// Layer plugin API and registry -- the drop-in boundary of the reference
// (include/caffe/layer.hpp:34-478, include/caffe/layer_factory.hpp:56-137): same virtuals, same
// REGISTER_LAYER_CLASS type-string registry, so an unchanged prototxt `type:` resolves.  Bodies are
// new: Forward_gpu enqueues fn2_* C-ABI calls on the Net's stream; there is no CPU fallback
// (Forward_cpu throws, like the reference's own Correlation/Resample/DataAugmentation).
#pragma once
#include <map>

#include "blob.hpp"

namespace caffe {

template <typename Dtype>
class Layer {
 public:
    explicit Layer(const LayerParameter& param) : layer_param_(param), phase_(TEST) {}
    virtual ~Layer() {}

    // layer.hpp:67-76
    void SetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
        CheckBlobCounts(bottom, top);
        LayerSetUp(bottom, top);
        Reshape(bottom, top);
    }
    virtual void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {}
    virtual void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;

    // layer.hpp:484-521 (GPU mode only; loss weights are not used on the inference path)
    inline Dtype Forward(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
        Forward_gpu(bottom, top);
        return 0;
    }

    // layer.hpp:523-535: gradients w.r.t. the bottoms flagged in propagate_down (and the layer's parameters) from the top diffs.
    // This engine inserts no Split layers (net.cpp Init): a bottom blob with several consumers receives one contribution per
    // consumer, so Net::Backward tells every layer per bottom whether to OVERWRITE (first contribution) or ADD to the diff.
    inline void Backward(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) {
        if (bottom_accumulate_.size() != bottom.size()) bottom_accumulate_.assign(bottom.size(), false);
        Backward_gpu(top, propagate_down, bottom);
    }
    void set_bottom_accumulate(const vector<bool>& a) { bottom_accumulate_ = a; }
    // loss weight of top i (LayerParameter.loss_weight, layer.hpp:455-478 SetLossWeights; loss layers default to 1 for top 0)
    virtual Dtype loss_weight(int top_index) const {
        const Message* m = layer_param_.m.get();
        if (m->count("loss_weight") > top_index) return (Dtype)m->f("loss_weight", 0, top_index);
        return (Dtype)(IsLossLayer() && top_index == 0 ? 1 : 0);
    }
    virtual bool IsLossLayer() const { return false; }

    vector<shared_ptr<Blob<Dtype> > >& blobs() { return blobs_; }
    const LayerParameter& layer_param() const { return layer_param_; }
    void set_phase(Phase p) { phase_ = p; }
    virtual inline const char* type() const { return ""; }
    virtual inline int ExactNumBottomBlobs() const { return -1; }
    virtual inline int MinBottomBlobs() const { return -1; }
    virtual inline int MaxBottomBlobs() const { return -1; }
    virtual inline int ExactNumTopBlobs() const { return -1; }
    virtual inline int MinTopBlobs() const { return -1; }
    virtual inline int MaxTopBlobs() const { return -1; }
    virtual inline bool EqualNumBottomTopBlobs() const { return false; }
    virtual inline bool AllowBackward() const { return true; }                 // layer.hpp:322 (fork)
    virtual inline bool DoesUseCustomCopyBlobs() const { return false; }       // layer.hpp:130 (fork)
    virtual void CustomCopyBlobs(const vector<Blob<Dtype>*>& blobs) {}          // layer.hpp:136

    // ---- engine hooks (not in the reference) ------------------------------------------------
    // Called once per Net::Forward on the host, with the net's iteration (Net::iter), before any kernel is enqueued (e.g. the
    // DataAugmentation iteration counter, data_augmentation_layer.cu:353-354; LpqLoss's p/q schedule step).
    virtual void HostTick(int iter) {}
    // false while the layer's launch sequence depends on host state (no CUDA-graph replay).
    virtual bool GraphSafe() const { return true; }
    // Parameters were (re)loaded: derive packed device copies.
    virtual void ParamsChanged() {}
    // Fill parameters from the prototxt fillers (Net::FillParams); default: nothing to fill.
    virtual void FillParams(uint64_t seed) {}
    // true when the prototxt alone defines the parameters (a seed-free filler such as "diagonal", so FillParams ignores the
    // seed): Net::CopyTrainedLayersFrom fills them when the source does not name the layer, as Caffe's fillers have by then.
    virtual bool TemplateDefinedParams() const { return false; }
    // Conv/Deconv: fuse an in-place ReLU that directly follows top[i].
    virtual bool FuseReLU(int top_index, float negative_slope) { return false; }
    // Algorithmic work of one Forward (for roofline reporting): flops and bytes moved if every
    // bottom were read once and every top written once.
    virtual void WorkEstimate(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top,
                              double* flops, double* bytes) const {
        double b = 0;
        for (auto* x : bottom) b += 4.0 * x->count();
        for (auto* x : top) b += 4.0 * x->count();
        *flops = 0; *bytes = b;
    }
    // Preferred device layout of tops created by this layer.
    virtual typename Blob<Dtype>::Layout TopLayout() const { return Blob<Dtype>::NHWC; }

 protected:
    virtual void Forward_cpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
        CHECK(false) << type() << ": Forward_cpu is not implemented; the product path is GPU only "
                     << "(the CPU oracle under oracle/ is test infrastructure)";
    }
    virtual void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) = 0;
    virtual void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) {
        for (size_t i = 0; i < propagate_down.size(); i++)
            CHECK(!propagate_down[i]) << type() << " layer cannot do backward (bottom " << i << ")";
    }

    // layer.hpp:417-453
    virtual void CheckBlobCounts(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) {
        if (ExactNumBottomBlobs() >= 0) CHECK_EQ(ExactNumBottomBlobs(), (int)bottom.size()) << type() << " Layer takes " << ExactNumBottomBlobs() << " bottom blob(s) as input.";
        if (MinBottomBlobs() >= 0) CHECK_LE(MinBottomBlobs(), (int)bottom.size()) << type() << " Layer takes at least " << MinBottomBlobs() << " bottom blob(s) as input.";
        if (MaxBottomBlobs() >= 0) CHECK_GE(MaxBottomBlobs(), (int)bottom.size()) << type() << " Layer takes at most " << MaxBottomBlobs() << " bottom blob(s) as input.";
        if (ExactNumTopBlobs() >= 0) CHECK_EQ(ExactNumTopBlobs(), (int)top.size()) << type() << " Layer produces " << ExactNumTopBlobs() << " top blob(s) as output.";
        if (MinTopBlobs() >= 0) CHECK_LE(MinTopBlobs(), (int)top.size()) << type() << " Layer produces at least " << MinTopBlobs() << " top blob(s) as output.";
        if (MaxTopBlobs() >= 0) CHECK_GE(MaxTopBlobs(), (int)top.size()) << type() << " Layer produces at most " << MaxTopBlobs() << " top blob(s) as output.";
        if (EqualNumBottomTopBlobs()) CHECK_EQ(bottom.size(), top.size()) << type() << " Layer produces one top blob as output for each bottom blob input.";
    }

    LayerParameter layer_param_;
    Phase phase_;
    vector<shared_ptr<Blob<Dtype> > > blobs_;
    vector<bool> bottom_accumulate_;              // per bottom: add to the existing diff instead of overwriting it
};

// layer_factory.hpp:56-137
template <typename Dtype>
class LayerRegistry {
 public:
    typedef shared_ptr<Layer<Dtype> > (*Creator)(const LayerParameter&);
    typedef std::map<string, Creator> CreatorRegistry;
    static CreatorRegistry& Registry() {
        static CreatorRegistry* g_registry_ = new CreatorRegistry();
        return *g_registry_;
    }
    static void AddCreator(const string& type, Creator creator) {
        CreatorRegistry& registry = Registry();
        CHECK(registry.count(type) == 0) << "Layer type " << type << " already registered.";
        registry[type] = creator;
    }
    static shared_ptr<Layer<Dtype> > CreateLayer(const LayerParameter& param) {
        const string& type = param.type();
        CreatorRegistry& registry = Registry();
        CHECK(registry.count(type) == 1) << "Unknown layer type: " << type << " (known types: " << LayerTypeListString() << ")";
        return registry[type](param);
    }
    static vector<string> LayerTypeList() {
        vector<string> v;
        for (auto& kv : Registry()) v.push_back(kv.first);
        return v;
    }
 private:
    LayerRegistry() {}
    static string LayerTypeListString() {
        string s;
        for (auto& t : LayerTypeList()) { if (!s.empty()) s += ", "; s += t; }
        return s;
    }
};

template <typename Dtype>
class LayerRegisterer {
 public:
    LayerRegisterer(const string& type, shared_ptr<Layer<Dtype> > (*creator)(const LayerParameter&)) {
        LayerRegistry<Dtype>::AddCreator(type, creator);
    }
};

// The reference instantiates float and double (common.hpp:41); this engine is fp32 only.
#define REGISTER_LAYER_CREATOR(type, creator) \
    static LayerRegisterer<float> g_creator_f_##type(#type, creator<float>)

#define REGISTER_LAYER_CLASS(type)                                                       \
    template <typename Dtype>                                                            \
    shared_ptr<Layer<Dtype> > Creator_##type##Layer(const LayerParameter& param) {       \
        return shared_ptr<Layer<Dtype> >(new type##Layer<Dtype>(param));                 \
    }                                                                                    \
    REGISTER_LAYER_CREATOR(type, Creator_##type##Layer)

}  // namespace caffe
