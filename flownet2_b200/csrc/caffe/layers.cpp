// Layer classes on the FlowNet2 deploy graph.  Each mirrors the reference class of the same
// name (type string, parameter handling, shape rules, error messages) and forwards the device
// work to the fn2_* C-ABI.  Reference files are cited per class.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <set>
#include <sstream>

#include "../../../include/fn2_lpq.h"
#include "layer.hpp"

namespace caffe {

typedef Blob<float> BlobF;

static cudaStream_t S() { return Caffe::stream(); }

// A kernel that overwrites its output cannot write into a bottom diff that already holds another consumer's contribution
// (Net::PlanBackward's accumulate flag): such a bottom gets a scratch diff blob, which is then added in.
template <typename Dtype>
class ScratchDiff {
 public:
    // The blob whose diff the kernel writes: `bottom`, or with `use_scratch` a blob of bottom's layout with `channels` channels
    Blob<Dtype>* target(Blob<Dtype>* bottom, bool use_scratch, int channels) {
        if (!use_scratch) return bottom;
        if (!blob_) blob_.reset(new Blob<Dtype>());
        blob_->set_layout(bottom->layout(), -1);
        blob_->Reshape(bottom->num(), channels, bottom->height(), bottom->width());
        return blob_.get();
    }
    // After the kernel: a scratch target's first bottom->channels() channels go to the bottom's diff, added when it accumulates
    void finish(Blob<Dtype>* target, Blob<Dtype>* bottom, bool accumulate, cudaStream_t st) {
        if (target == bottom) return;
        fn2_tensor s = target->diff_tensor(0, bottom->channels()), d = bottom->diff_tensor();
        FN2_CALL(fn2_axpby(&s, 1.f, &d, accumulate ? 1.f : 0.f, st));
    }
 private:
    shared_ptr<Blob<Dtype> > blob_;
};

// ---------------------------------------------------------------------------------------------
// Fillers (include/caffe/filler.hpp).  Deterministic host RNG (the reference draws from boost
// mt19937, util/rng.hpp:16-20; bit-matching boost is out of scope -- weights come from a
// .caffemodel in real use and from this generator for synthetic benchmarks).
// ---------------------------------------------------------------------------------------------
struct HostRng {
    std::mt19937_64 gen;
    explicit HostRng(uint64_t seed) : gen(seed) {}
    double uniform() { return (double)(gen() >> 11) * (1.0 / 9007199254740992.0); }
    bool has_spare = false;
    double spare = 0;
    double gaussian() {
        if (has_spare) { has_spare = false; return spare; }
        double u, v, s;
        do {
            u = uniform() * 2 - 1; v = uniform() * 2 - 1; s = u * u + v * v;
        } while (s >= 1 || s == 0);
        double m = std::sqrt(-2.0 * std::log(s) / s);
        spare = v * m; has_spare = true;
        return u * m;
    }
};

static void FillBlob(const FillerParameter& fp, BlobF* blob, uint64_t seed) {
    CHECK(blob->count()) << "filler: empty blob";
    float* d = blob->mutable_cpu_data();
    const int count = blob->count();
    const string type = fp.type();
    HostRng rng(seed);
    if (type == "constant") {                                     // filler.hpp:45-60
        for (int i = 0; i < count; i++) d[i] = fp.value();
    } else if (type == "uniform") {                               // :63-76
        for (int i = 0; i < count; i++) d[i] = (float)(fp.min() + (fp.max() - fp.min()) * rng.uniform());
    } else if (type == "gaussian") {                              // :79-113 (no sparsity)
        for (int i = 0; i < count; i++) d[i] = (float)(fp.mean() + fp.std() * rng.gaussian());
    } else if (type == "xavier" || type == "msra") {              // :145-208
        const int fan_in = count / blob->num();
        const int fan_out = count / blob->channels();
        double n = fan_in;
        const string vn = fp.variance_norm();
        if (vn == "AVERAGE" || vn == "2") n = (fan_in + fan_out) / 2.0;
        else if (vn == "FAN_OUT" || vn == "1") n = fan_out;
        if (type == "xavier") {
            const double scale = std::sqrt(3.0 / n);
            for (int i = 0; i < count; i++) d[i] = (float)(-scale + 2 * scale * rng.uniform());
        } else {
            const double sd = std::sqrt(2.0 / n);
            for (int i = 0; i < count; i++) d[i] = (float)(sd * rng.gaussian());
        }
    } else if (type == "diagonal") {                              // filler.hpp:265-290 (fork)
        for (int i = 0; i < count; i++) d[i] = 0.f;
        const int kernel_area = blob->height() * blob->width();
        const int channels = blob->channels(), num = blob->num();
        for (int n = 0; n < num && n < channels; ++n) {
            float v = fp.diag_val_size() > n ? fp.diag_val(n) : 1.f;
            v /= (float)kernel_area;
            for (int k = 0; k < kernel_area; k++) d[kernel_area * (channels * n + n) + k] = v;
        }
    } else {
        CHECK(false) << "Unknown filler name: " << type;          // filler.hpp:318
    }
}

// ---------------------------------------------------------------------------------------------
// Input (input_layer.cpp:8-22), Split / Silence pass-throughs.
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class InputLayer : public Layer<Dtype> {
 public:
    explicit InputLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Input"; }
    int ExactNumBottomBlobs() const override { return 0; }
    int MinTopBlobs() const override { return 1; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const Message& ip = this->layer_param_.m->msg("input_param");
        const int num_top = (int)top.size(), num_shape = ip.count("shape");
        CHECK(num_shape == 0 || num_shape == 1 || num_shape == num_top)
            << "Must specify 'shape' once, once per top blob, or not at all: " << num_top << " tops vs. "
            << num_shape << " shapes.";
        for (int i = 0; i < num_top && num_shape > 0; ++i) {
            const Message& sh = ip.msg("shape", num_shape == 1 ? 0 : i);
            vector<int> dims;
            for (int j = 0; j < sh.count("dim"); j++) dims.push_back(sh.i("dim", 1, j));
            CHECK_EQ(dims.size(), 4u) << "Input blobs on the FlowNet2 path are 4-D (N,C,H,W)";
            top[i]->Reshape(dims);
        }
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {}
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {}
};
REGISTER_LAYER_CLASS(Input);

template <typename Dtype>
class SilenceLayer : public Layer<Dtype> {                         // silence_layer.cpp
 public:
    explicit SilenceLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Silence"; }
    int MinBottomBlobs() const override { return 1; }
    int ExactNumTopBlobs() const override { return 0; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {}
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {}
};
REGISTER_LAYER_CLASS(Silence);

// ---------------------------------------------------------------------------------------------
// ReLU (relu_layer.cpp / relu_layer.cu:9-14).  Usually fused into the producing conv by
// Net::Init; this standalone kernel remains for non-fusable placements.
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class ReLULayer : public Layer<Dtype> {
 public:
    explicit ReLULayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "ReLU"; }
    int ExactNumBottomBlobs() const override { return 1; }
    int ExactNumTopBlobs() const override { return 1; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        top[0]->ReshapeLike(*bottom[0]);
    }
    float negative_slope() const { return this->layer_param_.relu_negative_slope(); }
    void set_fused(bool f) { fused_ = f; }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        if (fused_) return;     // applied in the producer's epilogue
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_relu_forward(&b, &t, negative_slope(), S()));
    }
    // relu_layer.cu:29-55.  Fused into the producer: the producing convolution applies the derivative to its top diff itself.
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        if (fused_ || !propagate_down[0]) return;
        fn2_tensor td = top[0]->tensor(), dy = top[0]->diff_tensor(), dx = bottom[0]->diff_tensor();
        // in place (top == bottom): dx and dy are the same storage, never an accumulation
        FN2_CALL(fn2_relu_backward(&td, &dy, &dx, negative_slope(), top[0] == bottom[0] ? 0 : (this->bottom_accumulate_[0] ? 1 : 0), S()));
    }
    bool fused_ = false;
};
REGISTER_LAYER_CLASS(ReLU);

// ---------------------------------------------------------------------------------------------
// Eltwise (eltwise_layer.cpp:10-65): SUM with coefficients is what the deploy nets use
// (input scaling by 1/255, flow * 20, img0 - warped).
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class EltwiseLayer : public Layer<Dtype> {
 public:
    explicit EltwiseLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Eltwise"; }
    int MinBottomBlobs() const override { return 1; }
    int ExactNumTopBlobs() const override { return 1; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        EltwiseParameter ep = this->layer_param_.eltwise_param();
        CHECK(ep.coeff_size() == 0 || ep.coeff_size() == (int)bottom.size())
            << "Eltwise Layer takes one coefficient per bottom blob.";
        const string op = ep.operation();
        CHECK(op == "SUM" || op == "1") << "Eltwise: only operation SUM is implemented on this path (got " << op << ")";
        CHECK_LE(bottom.size(), 4u) << "Eltwise: at most 4 bottoms";
        coeffs_.assign(bottom.size(), 1.f);
        for (int i = 0; i < ep.coeff_size(); i++) coeffs_[i] = ep.coeff(i);
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        for (size_t i = 1; i < bottom.size(); ++i) CHECK(bottom[i]->shape() == bottom[0]->shape());
        top[0]->ReshapeLike(*bottom[0]);
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor bs[4];
        const fn2_tensor* bp[4];
        for (size_t i = 0; i < bottom.size(); i++) { bs[i] = bottom[i]->tensor(); bp[i] = &bs[i]; }
        fn2_tensor t = top[0]->mutable_tensor();
        FN2_CALL(fn2_eltwise_sum(bp, coeffs_.data(), (int)bottom.size(), &t, S()));
    }
    // eltwise_layer.cu:87-131 (SUM): bottom_diff_i = coeff_i * top_diff
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        fn2_tensor dy = top[0]->diff_tensor();
        for (size_t i = 0; i < bottom.size(); i++) {
            if (!propagate_down[i]) continue;
            fn2_tensor dx = bottom[i]->diff_tensor();
            FN2_CALL(fn2_axpby(&dy, coeffs_[i], &dx, this->bottom_accumulate_[i] ? 1.f : 0.f, S()));
        }
    }
    vector<float> coeffs_;
};
REGISTER_LAYER_CLASS(Eltwise);

// ---------------------------------------------------------------------------------------------
// Concat along channels (concat_layer.cpp:14-75).  When Net::Init could alias the bottoms into
// the top's storage (zero-copy), Forward is a no-op for those bottoms.
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class ConcatLayer : public Layer<Dtype> {
 public:
    explicit ConcatLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Concat"; }
    int MinBottomBlobs() const override { return 1; }
    int ExactNumTopBlobs() const override { return 1; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const int axis = this->layer_param_.concat_axis();
        CHECK_EQ(axis, 1) << "Concat: only the channel axis is used on the FlowNet2 path";
        vector<int> ts = bottom[0]->shape();
        for (size_t i = 1; i < bottom.size(); ++i) {
            CHECK_EQ(bottom[0]->num_axes(), bottom[i]->num_axes()) << "All inputs must have the same #axes.";
            for (int j = 0; j < 4; j++)
                if (j != 1) CHECK_EQ(ts[j], bottom[i]->shape(j)) << "All inputs must have the same shape, except at concat_axis.";
            ts[1] += bottom[i]->shape(1);
        }
        top[0]->Reshape(ts);
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        int c0 = 0;
        for (size_t i = 0; i < bottom.size(); i++) {
            const int c = bottom[i]->channels();
            if (!(bottom[i]->alias_parent() == top[0] && bottom[i]->alias_offset() == c0)) {
                fn2_tensor s = bottom[i]->tensor(), d = top[0]->mutable_tensor(c0, c);
                FN2_CALL(fn2_copy(&s, &d, S()));
            }
            c0 += c;
        }
    }
    // concat_layer.cu:52-75: slices of the top diff.  A zero-copy child's diff IS the slice (Blob::diff_tensor): nothing to do.
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        int c0 = 0;
        for (size_t i = 0; i < bottom.size(); i++) {
            const int c = bottom[i]->channels();
            if (propagate_down[i] && !(bottom[i]->alias_parent() == top[0] && bottom[i]->alias_offset() == c0)) {
                fn2_tensor dy = top[0]->diff_tensor(c0, c), dx = bottom[i]->diff_tensor();
                FN2_CALL(fn2_axpby(&dy, 1.f, &dx, this->bottom_accumulate_[i] ? 1.f : 0.f, S()));
            }
            c0 += c;
        }
    }
};
REGISTER_LAYER_CLASS(Concat);

// Slice along channels (slice_layer.cpp), used by some FlowNet variants to split stacked inputs.
template <typename Dtype>
class SliceLayer : public Layer<Dtype> {
 public:
    explicit SliceLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Slice"; }
    int ExactNumBottomBlobs() const override { return 1; }
    int MinTopBlobs() const override { return 1; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const Message& sp = this->layer_param_.m->msg("slice_param");
        const int axis = sp.has("slice_dim") ? sp.i("slice_dim", 1) : sp.i("axis", 1);
        CHECK_EQ(axis, 1) << "Slice: only the channel axis is supported";
        const int C = bottom[0]->channels(), nt = (int)top.size();
        points_.clear();
        if (sp.count("slice_point")) {
            CHECK_EQ(sp.count("slice_point"), nt - 1);
            int prev = 0;
            for (int i = 0; i < nt - 1; i++) { int pt = sp.i("slice_point", 0, i); CHECK_GT(pt, prev); points_.push_back(pt); prev = pt; }
        } else {
            CHECK_EQ(C % nt, 0) << "Number of top blobs (" << nt << ") should evenly divide input slice axis (" << C << ")";
            for (int i = 1; i < nt; i++) points_.push_back(i * (C / nt));
        }
        int prev = 0;
        for (int i = 0; i < nt; i++) {
            int end = i < nt - 1 ? points_[i] : C;
            top[i]->Reshape(bottom[0]->num(), end - prev, bottom[0]->height(), bottom[0]->width());
            prev = end;
        }
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        int prev = 0;
        for (size_t i = 0; i < top.size(); i++) {
            const int c = top[i]->channels();
            fn2_tensor s = bottom[0]->tensor(prev, c), d = top[i]->mutable_tensor();
            FN2_CALL(fn2_copy(&s, &d, S()));
            prev += c;
        }
    }
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        if (!propagate_down[0]) return;
        int prev = 0;
        for (size_t i = 0; i < top.size(); i++) {
            const int c = top[i]->channels();
            fn2_tensor dy = top[i]->diff_tensor(), dx = bottom[0]->diff_tensor(prev, c);
            FN2_CALL(fn2_axpby(&dy, 1.f, &dx, this->bottom_accumulate_[0] ? 1.f : 0.f, S()));
            prev += c;
        }
    }
    vector<int> points_;
};
REGISTER_LAYER_CLASS(Slice);

// ---------------------------------------------------------------------------------------------
// ChannelNorm (channel_norm_layer.cpp:21-36, .cu:17-30)
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class ChannelNormLayer : public Layer<Dtype> {
 public:
    explicit ChannelNormLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "ChannelNorm"; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom.size(), 1u) << "ChannelNormLayer takes one input blob.";
        CHECK_EQ(top.size(), 1u) << "ChannelNormLayer outputs one blob.";
        top[0]->Reshape(bottom[0]->num(), 1, bottom[0]->height(), bottom[0]->width());
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_channel_norm_forward(&b, &t, S()));
    }
};
REGISTER_LAYER_CLASS(ChannelNorm);

// ---------------------------------------------------------------------------------------------
// FlowWarp (flow_warp_layer.cpp:29-52 shapes; forward .cpp:57-117 / .cu:357-458)
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class FlowWarpLayer : public Layer<Dtype> {
 public:
    explicit FlowWarpLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "FlowWarp"; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom.size(), 2u) << "FlowWarpLayer takes two input blobs: image and flow.";
        CHECK_EQ(top.size(), 1u) << "FlowWarpLayer outputs one blob.";
        CHECK_EQ(bottom[0]->num(), bottom[1]->num()) << "Num of the inputs should be the same";
        CHECK_EQ(2, bottom[1]->channels()) << "Flow should have 2 channels: x-flow and y-flow";
        CHECK_EQ(bottom[0]->width(), bottom[1]->width()) << "Width of the inputs should be the same";
        CHECK_EQ(bottom[0]->height(), bottom[1]->height()) << "Height of the inputs should be the same";
        top[0]->ReshapeLike(*bottom[0]);
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor img = bottom[0]->tensor(), fl = bottom[1]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_flow_warp_forward(&img, &fl, &t, this->layer_param_.flow_warp_param().fill_nan() ? 1 : 0, S()));
    }
    // flow_warp_layer.cu:461-514: scatter-add into the image diff, gather for the flow diff (the kernel overwrites both)
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        if (!propagate_down[0] && !propagate_down[1]) return;
        CHECK(!this->bottom_accumulate_[0] && !this->bottom_accumulate_[1]) << "FlowWarp backward into a shared bottom is not supported";
        fn2_tensor img = bottom[0]->tensor(), fl = bottom[1]->tensor(), dy = top[0]->diff_tensor();
        fn2_tensor di = bottom[0]->diff_tensor(), df = bottom[1]->diff_tensor();
        FN2_CALL(fn2_flow_warp_backward(&img, &fl, &dy, &di, &df, S()));
    }
};
REGISTER_LAYER_CLASS(FlowWarp);

// ---------------------------------------------------------------------------------------------
// Resample (resample_layer.cpp:11-55, .cu:128-206)
// ---------------------------------------------------------------------------------------------
template <typename Dtype>
class ResampleLayer : public Layer<Dtype> {
 public:
    explicit ResampleLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Resample"; }
    bool AllowBackward() const override { return false; }           // resample_layer.hpp:25
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const int t = this->layer_param_.resample_param().type();
        CHECK(t == 1 || t == 2 || t == 3) << "ResampleLayer: only CUBIC, LINEAR and NEAREST interpolation is supported for now";
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        this->layer_param_.m->set("reshape_every_iter", "false");   // resample_layer.cpp:27
        CHECK_GE(bottom.size(), 1u);
        CHECK_LE(bottom.size(), 2u);
        CHECK_EQ(top.size(), 1u);
        int top_h, top_w;
        if (bottom.size() == 1) {
            top_h = this->layer_param_.resample_param().height();
            top_w = this->layer_param_.resample_param().width();
        } else {
            top_h = bottom[1]->height();
            top_w = bottom[1]->width();
        }
        CHECK_GE(top_h, 1) << "ResampleLayer must have top_height > 0";
        CHECK_GE(top_w, 1) << "ResampleLayer must have top_width > 0";
        top[0]->Reshape(bottom[0]->num(), bottom[0]->channels(), top_h, top_w);
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        ResampleParameter rp = this->layer_param_.resample_param();
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_resample_forward(&b, &t, rp.type(), rp.antialias() ? 1 : 0, S()));
    }
};
REGISTER_LAYER_CLASS(Resample);

// ---------------------------------------------------------------------------------------------
// Correlation (correlation_layer.cpp:13-84, .cu:431-504)
// ---------------------------------------------------------------------------------------------
// correlation_param of Correlation and Correlation1D (correlation_layer.cpp:13-35, correlation_layer1d.cpp:13-37)
struct CorrParams {
    int kernel_size = 0, max_displacement = 0, pad = 0, stride1 = 1, stride2 = 1, corr_type = 0, single_direction = 0;
    static CorrParams Parse(const CorrelationParameter& cp) {
        CorrParams p;
        CHECK(cp.has_kernel_size()) << "Filter kernel_size is not set";
        CHECK(cp.has_max_displacement()) << "Max displacement is required.";
        p.kernel_size = cp.kernel_size();
        CHECK(p.kernel_size % 2 == 1) << "Odd kernel size required";
        p.max_displacement = cp.max_displacement();
        p.pad = cp.pad();
        p.stride1 = cp.stride_1();
        p.stride2 = cp.stride_2();
        p.single_direction = cp.single_direction();             // Correlation1D only
        p.corr_type = cp.correlation_type();                     // do_abs is parsed and unused in the reference too
        return p;
    }
    // SURVEY 8(d): bytes = read both maps once + write top once; flops = 2*D^2*k^2*C per output pixel
    template <typename Dtype>
    void WorkEstimate(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top, double* flops, double* bytes) const {
        *bytes = 4.0 * (bottom[0]->count() + bottom[1]->count() + top[0]->count());
        *flops = 2.0 * top[0]->count() * (double)kernel_size * kernel_size * bottom[0]->channels();
    }
};

template <typename Dtype>
class CorrelationLayer : public Layer<Dtype> {
 public:
    explicit CorrelationLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Correlation"; }
    int ExactNumBottomBlobs() const override { return 2; }
    int ExactNumTopBlobs() const override { return 1; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        p_ = CorrParams::Parse(this->layer_param_.correlation_param());
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom[0]->width(), bottom[1]->width()) << "Both bottom blobs must have same width";
        CHECK_EQ(bottom[0]->height(), bottom[1]->height()) << "Both bottom blobs must have same height";
        CHECK_EQ(bottom[0]->channels(), bottom[1]->channels()) << "Both bottom blobs must have same height";
        int tc, th, tw;
        FN2_CALL(fn2_correlation_shape(bottom[0]->height(), bottom[0]->width(), p_.pad, p_.kernel_size,
                                       p_.max_displacement, p_.stride1, p_.stride2, &tc, &th, &tw));
        top[0]->Reshape(bottom[0]->num(), tc, th, tw);
        size_t need = 0;
        FN2_CALL(fn2_correlation_workspace_bytes(bottom[0]->num(), bottom[0]->channels(), bottom[0]->height(),
                                                 bottom[0]->width(), p_.pad, p_.kernel_size, p_.max_displacement,
                                                 p_.stride1, p_.stride2, p_.corr_type, &need));
        ws_.reserve(need, S());
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b0 = bottom[0]->tensor(), b1 = bottom[1]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_correlation_forward(&b0, &b1, &t, p_.pad, p_.kernel_size, p_.max_displacement, p_.stride1,
                                         p_.stride2, p_.corr_type, ws_.get(), ws_.bytes(), S()));
    }
    // correlation_layer.cu:508-600.  The kernels overwrite both bottom diffs.
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        if (!propagate_down[0] && !propagate_down[1]) return;
        size_t need = 0;
        FN2_CALL(fn2_correlation_backward_workspace_bytes(bottom[0]->num(), bottom[0]->channels(), bottom[0]->height(), bottom[0]->width(),
                                                          p_.pad, p_.kernel_size, p_.max_displacement, p_.stride1, p_.stride2, p_.corr_type, &need));
        bws_.reserve(need);
        Blob<Dtype>* tgt[2];
        for (int i = 0; i < 2; i++) tgt[i] = scratch_[i].target(bottom[i], this->bottom_accumulate_[i], bottom[i]->channels());
        fn2_tensor b0 = bottom[0]->tensor(), b1 = bottom[1]->tensor(), dy = top[0]->diff_tensor();
        fn2_tensor d0 = tgt[0]->diff_tensor(), d1 = tgt[1]->diff_tensor();
        FN2_CALL(fn2_correlation_backward(&b0, &b1, &dy, &d0, &d1, p_.pad, p_.kernel_size, p_.max_displacement, p_.stride1, p_.stride2,
                                          p_.corr_type, bws_.get(), bws_.bytes(), S()));
        for (int i = 0; i < 2; i++) scratch_[i].finish(tgt[i], bottom[i], this->bottom_accumulate_[i], S());
    }
    void WorkEstimate(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top, double* flops,
                      double* bytes) const override {
        p_.WorkEstimate(bottom, top, flops, bytes);
    }
    CorrParams p_;
    DeviceBuffer ws_, bws_;
    ScratchDiff<Dtype> scratch_[2];
};
REGISTER_LAYER_CLASS(Correlation);

// Correlation1D (correlation_layer1d.cpp:13-84, correlation_layer1d.cu): displacement along x only (DispNet-style nets).
template <typename Dtype>
class Correlation1DLayer : public Layer<Dtype> {
 public:
    explicit Correlation1DLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Correlation1D"; }
    int ExactNumBottomBlobs() const override { return 2; }
    int ExactNumTopBlobs() const override { return 1; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        p_ = CorrParams::Parse(this->layer_param_.correlation_param());
        CHECK(p_.single_direction >= -1 && p_.single_direction <= 1) << "single_direction must be -1 (left), 0 (off), or 1 (right)";
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom[0]->width(), bottom[1]->width()) << "Both bottom blobs must have same width";
        CHECK_EQ(bottom[0]->height(), bottom[1]->height()) << "Both bottom blobs must have same height";
        CHECK_EQ(bottom[0]->channels(), bottom[1]->channels()) << "Both bottom blobs must have same number of channels";
        int tc, th, tw;
        FN2_CALL(fn2_correlation1d_shape(bottom[0]->height(), bottom[0]->width(), p_.pad, p_.kernel_size, p_.max_displacement,
                                         p_.stride1, p_.stride2, p_.single_direction, &tc, &th, &tw));
        top[0]->Reshape(bottom[0]->num(), tc, th, tw);
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b0 = bottom[0]->tensor(), b1 = bottom[1]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_correlation1d_forward(&b0, &b1, &t, p_.pad, p_.kernel_size, p_.max_displacement, p_.stride1, p_.stride2,
                                           p_.single_direction, p_.corr_type, S()));
    }
    void WorkEstimate(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top, double* flops,
                      double* bytes) const override {
        p_.WorkEstimate(bottom, top, flops, bytes);
    }
    CorrParams p_;
};
REGISTER_LAYER_CLASS(Correlation1D);

// ---------------------------------------------------------------------------------------------
// Convolution / Deconvolution (base_conv_layer.cpp:12-254, conv_layer.cpp, deconv_layer.cpp).
// group == 1 and dilation == 1 (all FlowNet2 layers); several bottom/top pairs share the weights
// (conv_layer.cpp:28).  Engine selection follows GetConvolutionLayer (layer_factory.cpp:37-71):
// engine CAFFE -> exact FP32 SIMT kernel, DEFAULT/CUDNN -> wgmma tensor-core kernel when the
// shape is eligible.
// ---------------------------------------------------------------------------------------------
struct PackedWeights { DeviceBuffer buf; int gen = -1; };   // fn2_conv_pack_weights output of one ParamsChanged generation

template <typename Dtype>
class BaseConvolutionLayer : public Layer<Dtype> {
 public:
    explicit BaseConvolutionLayer(const LayerParameter& p, bool deconv) : Layer<Dtype>(p), deconv_(deconv) {}
    int MinBottomBlobs() const override { return 1; }
    int MinTopBlobs() const override { return 1; }
    bool EqualNumBottomTopBlobs() const override { return true; }

    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        ConvolutionParameter cp = this->layer_param_.convolution_param();
        memset(&d_, 0, sizeof(d_));
        int kh, kw, sh, sw, ph, pw, dh, dw;
        cp.kernel(&kh, &kw); cp.stride(&sh, &sw); cp.pad(&ph, &pw); cp.dilation(&dh, &dw);
        CHECK(dh == 1 && dw == 1) << "dilated convolution is not used on the FlowNet2 path";
        CHECK_EQ(cp.group(), 1) << "grouped convolution is not used on the FlowNet2 path";
        CHECK_GT(cp.num_output(), 0);
        d_.ci = bottom[0]->channels(); d_.co = cp.num_output();
        d_.kh = kh; d_.kw = kw; d_.stride_h = sh; d_.stride_w = sw; d_.pad_h = ph; d_.pad_w = pw;
        d_.deconv = deconv_ ? 1 : 0;
        d_.has_bias = cp.bias_term() ? 1 : 0;
        const string eng = cp.engine();
        d_.engine = (eng == "CAFFE" || eng == "1") ? 1 : 0;
        if (const char* e = getenv("FN2_CONV_ENGINE")) {
            if (!strcmp(e, "simt")) d_.engine = 1;
            else if (!strcmp(e, "tc")) d_.engine = 0;
        }
        d_.input_guard_bytes = Blob<Dtype>::kGuardFloats * (int)sizeof(Dtype);   // every blob's device storage has it
        relu_.assign(top.size(), 0);
        slope_.assign(top.size(), 0.f);
        if (this->blobs_.size() > 0) {
            CHECK_EQ(1 + d_.has_bias, (int)this->blobs_.size()) << "Incorrect number of weight blobs.";
        } else {
            this->blobs_.resize(1 + d_.has_bias);
            // conv [co][ci][kh][kw]; deconv [ci][co][kh][kw] (base_conv_layer.cpp:125-140)
            if (!deconv_) this->blobs_[0].reset(new Blob<Dtype>(d_.co, d_.ci, kh, kw));
            else          this->blobs_[0].reset(new Blob<Dtype>(d_.ci, d_.co, kh, kw));
            if (d_.has_bias) { this->blobs_[1].reset(new Blob<Dtype>()); this->blobs_[1]->Reshape(vector<int>{d_.co}); }
        }
    }
    // the deploy nets' scale_conv1: a diagonal filler and no bias, so its weights follow from the template variables alone
    bool TemplateDefinedParams() const override {
        return !d_.has_bias && this->layer_param_.convolution_param().weight_filler().type() == "diagonal";
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom[0]->channels(), d_.ci) << "Input size incompatible with convolution kernel.";
        for (size_t i = 1; i < bottom.size(); ++i)
            CHECK(bottom[0]->shape() == bottom[i]->shape()) << "All inputs must have the same shape.";
        int Ho, Wo;
        FN2_CALL(fn2_conv_out_shape(&d_, bottom[0]->height(), bottom[0]->width(), &Ho, &Wo));
        for (size_t i = 0; i < top.size(); ++i) top[i]->Reshape(bottom[0]->num(), d_.co, Ho, Wo);
        bottoms_.assign(bottom.begin(), bottom.end());
        size_t need = 0;
        FN2_CALL(fn2_conv_workspace_bytes(&d_, bottom[0]->num(), bottom[0]->height(), bottom[0]->width(), &need));
        ws_.reserve(need);
    }
    void FillParams(uint64_t seed) override {
        ConvolutionParameter cp = this->layer_param_.convolution_param();
        FillBlob(cp.weight_filler(), this->blobs_[0].get(), seed * 2 + 1);
        if (d_.has_bias) FillBlob(cp.bias_filler(), this->blobs_[1].get(), seed * 2 + 2);
    }
    // The packed layout depends on the bottom's pixel stride (small-Ci packing modes), which zero-copy concat aliasing can
    // change after Reshape and which may differ between the bottoms of one layer: one packed copy per distinct stride.
    void ParamsChanged() override {
        ++params_gen_;
        std::set<int> strides;
        for (const Blob<Dtype>* b : bottoms_) strides.insert(b->channel_stride() > 0 ? b->channel_stride() : d_.ci);
        if (strides.empty()) strides.insert(d_.ci);
        for (int cis : strides) {
            size_t floats = 0;
            FN2_CALL(fn2_conv_packed_floats(&d_, cis, &floats));
            DeviceBuffer& pk = packed_[cis].buf;
            pk.reserve(floats * sizeof(float));
            FN2_CALL(fn2_conv_pack_weights(&d_, cis, this->blobs_[0]->gpu_data(), pk.as<float>(), S()));
        }
    }
    void WorkEstimate(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top, double* flops,
                      double* bytes) const override {
        double f = 0, b = 4.0 * this->blobs_[0]->count();
        for (size_t i = 0; i < bottom.size(); i++) {
            // conv: 2*N*Co*Ho*Wo*Ci*kh*kw ; deconv: 2*N*Ci*H*W*Co*kh*kw (every input pixel x every tap)
            const Blob<Dtype>* px = deconv_ ? bottom[i] : top[i];
            f += 2.0 * px->num() * px->height() * px->width() * (double)d_.ci * d_.co * d_.kh * d_.kw;
            b += 4.0 * (bottom[i]->count() + top[i]->count());
        }
        *flops = f; *bytes = b;
    }
    bool FuseReLU(int top_index, float negative_slope) override {
        if (top_index < 0 || top_index >= (int)relu_.size() || relu_[top_index]) return false;
        relu_[top_index] = 1; slope_[top_index] = negative_slope;
        return true;
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        for (size_t i = 0; i < bottom.size(); ++i) {
            fn2_conv_desc d = d_;
            d.relu = relu_[i]; d.negative_slope = slope_[i];
            fn2_tensor b = bottom[i]->tensor(), t = top[i]->mutable_tensor();
            // input_guard_bytes promises readable slack around the bottom's OWN allocation (Blob::kGuardFloats), which the kernel-row
            // packing of small-Ci layers relies on; a zero-copy concat child has none.  Net::AliasConcats keeps such bottoms dense.
            CHECK(!(!deconv_ && bottom[i]->is_alias() && d_.ci <= 16 && d_.input_guard_bytes > 0))
                << "a zero-copy concat child must not feed a convolution with <= 16 input channels (layer " << this->layer_param_.name() << ")";
            auto it = packed_.find(bottom[i]->channel_stride() > 0 ? bottom[i]->channel_stride() : d_.ci);
            CHECK(it != packed_.end() && !it->second.buf.empty()) << "convolution weights were never packed for this bottom layout";
            const DeviceBuffer& packed = it->second.buf;
            FN2_CALL(fn2_conv_forward(&d, &b, packed.as<float>(), d_.has_bias ? this->blobs_[1]->gpu_data() : nullptr, &t,
                                      ws_.get(), ws_.bytes(), S()));
        }
    }
    // conv_layer.cu:26-58 / deconv_layer.cu:26-55.  Weight and bias gradients: fn2_conv_backward_params (ADDED to the parameter
    // diffs like the reference's gemm with beta = 1; Net::ClearParamDiffs zeroes them).  Data gradient: the adjoint operator
    // run through fn2_conv_forward on the top diff (fn2_conv_backward_data_desc).  A fused ReLU is differentiated first, in place
    // on the top diff (the top blob has no other producer).
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        cudaStream_t st = S();
        size_t need = 0;
        FN2_CALL(fn2_conv_backward_params_workspace_bytes(&d_, bottom[0]->num(), bottom[0]->height(), bottom[0]->width(), &need));
        pws_.reserve(need);
        fn2_tensor wd = this->blobs_[0]->diff_tensor();
        float* bd = d_.has_bias ? this->blobs_[1]->diff_tensor().data : nullptr;
        for (size_t i = 0; i < bottom.size(); ++i) {
            fn2_tensor dy = top[i]->diff_tensor();
            if (relu_[i]) {
                fn2_tensor y = top[i]->tensor();
                FN2_CALL(fn2_relu_backward(&y, &dy, &dy, slope_[i], 0, st));
            }
            fn2_tensor x = bottom[i]->tensor();
            FN2_CALL(fn2_conv_backward_params(&d_, &x, &dy, wd.data, bd, 1, pws_.get(), pws_.bytes(), st));
            if (!propagate_down[i]) continue;
            BackwardData(top[i], bottom[i], this->bottom_accumulate_[i], st);
        }
    }
    void BackwardData(Blob<Dtype>* top, Blob<Dtype>* bottom, bool accumulate, cudaStream_t st) {
        fn2_conv_desc bd;
        int flip = 0;
        FN2_CALL(fn2_conv_backward_data_desc(&d_, bottom->height(), bottom->width(), &bd, &flip));
        fn2_tensor dy = top->diff_tensor();
        // The tensor-core engine wants output channels in multiples of 16; concat-sized bottoms (1026, 770, 386, 473 channels)
        // are not.  Their adjoint convolution runs with zero weight rows appended, into the scratch diff blob.
        const bool pad_co = !bd.deconv && bd.co > 16 && bd.co % 16 != 0;
        if (pad_co) {
            // wide tiles: a multiple of 128 when that costs <= 1/8 more channels, else of 64 (of 16 for narrow outputs)
            const int c128 = (bd.co + 127) / 128 * 128, c64 = (bd.co + 63) / 64 * 64;
            bd.co = bd.co <= 64 ? (bd.co + 15) / 16 * 16 : ((c128 - bd.co) * 8 <= bd.co ? c128 : c64);
        }
        // packed weights of the adjoint operator for this top layout (derived once per ParamsChanged generation)
        const int cis = top->channel_stride() > 0 ? top->channel_stride() : d_.co;
        PackedWeights& pk = bpacked_[cis];
        if (pk.gen != params_gen_) {
            const float* w = this->blobs_[0]->gpu_data();
            if (flip || pad_co) {
                const size_t wn = (size_t)bd.co * bd.ci * bd.kh * bd.kw, wreal = (size_t)this->blobs_[0]->count();
                flipped_.reserve(wn * sizeof(float));
                float* fw = flipped_.as<float>();
                if (flip) FN2_CALL(fn2_conv_flip_transpose_weights(&d_, w, fw, st));
                else CUDA_CHECK(cudaMemcpyAsync(fw, w, wreal * sizeof(float), cudaMemcpyDeviceToDevice, st));
                if (wn > wreal) CUDA_CHECK(cudaMemsetAsync(fw + wreal, 0, (wn - wreal) * sizeof(float), st));
                w = fw;
            }
            size_t floats = 0;
            FN2_CALL(fn2_conv_packed_floats(&bd, cis, &floats));
            pk.buf.reserve(floats * sizeof(float));
            FN2_CALL(fn2_conv_pack_weights(&bd, cis, w, pk.buf.as<float>(), st));
            pk.gen = params_gen_;
        }
        int Hb, Wb;
        FN2_CALL(fn2_conv_out_shape(&bd, top->height(), top->width(), &Hb, &Wb));
        CHECK(Hb == bottom->height() && Wb == bottom->width()) << "conv backward: adjoint output " << Hb << "x" << Wb << " != bottom";
        Blob<Dtype>* tgt = bscratch_.target(bottom, accumulate || pad_co, bd.co);
        fn2_tensor dx = tgt->diff_tensor();
        size_t wsn = 0;
        FN2_CALL(fn2_conv_workspace_bytes(&bd, top->num(), top->height(), top->width(), &wsn));
        bws_.reserve(wsn);
        FN2_CALL(fn2_conv_forward(&bd, &dy, pk.buf.as<float>(), nullptr, &dx, bws_.get(), bws_.bytes(), st));
        bscratch_.finish(tgt, bottom, accumulate, st);
    }
    bool deconv_;
    fn2_conv_desc d_;
    vector<int> relu_;
    vector<float> slope_;
    std::map<int, PackedWeights> packed_;        // by bottom pixel stride
    std::map<int, PackedWeights> bpacked_;       // adjoint operator's packed weights, by top pixel stride
    int params_gen_ = 0;                  // bumped by ParamsChanged
    DeviceBuffer flipped_;                // flipped and / or Co-padded weights the adjoint packs from
    DeviceBuffer ws_, pws_, bws_;         // forward, parameter-gradient and adjoint workspaces
    ScratchDiff<Dtype> bscratch_;
    vector<const Blob<Dtype>*> bottoms_;
};

template <typename Dtype>
class ConvolutionLayer : public BaseConvolutionLayer<Dtype> {
 public:
    explicit ConvolutionLayer(const LayerParameter& p) : BaseConvolutionLayer<Dtype>(p, false) {}
    const char* type() const override { return "Convolution"; }
};
REGISTER_LAYER_CLASS(Convolution);

template <typename Dtype>
class DeconvolutionLayer : public BaseConvolutionLayer<Dtype> {
 public:
    explicit DeconvolutionLayer(const LayerParameter& p) : BaseConvolutionLayer<Dtype>(p, true) {}
    const char* type() const override { return "Deconvolution"; }
};
REGISTER_LAYER_CLASS(Deconvolution);

// ---------------------------------------------------------------------------------------------
// DataAugmentation (data_augmentation_layer.cpp:34-205, .cu:321-637,
// augmentation_layer_base.cpp:15-48).  Deploy use: crop == bottom size, no random generators ->
// default coefficients -> "identity" affine through SpatialAugmentation (with its dim-1.05 clamp)
// followed by mean subtraction.  Random coefficient sampling (training) is not built yet and is
// rejected loudly.
// ---------------------------------------------------------------------------------------------
struct TransMat {   // augmentation_layer_base.cpp:15-48, float arithmetic in the same order
    float t0, t1, t2, t3, t4, t5;
    void toIdentity() { t0 = 1; t2 = 0; t4 = 0; t1 = 0; t3 = 1; t5 = 0; }
    void leftMultiply(float u0, float u1, float u2, float u3, float u4, float u5) {
        float a0 = t0, a2 = t2, a4 = t4, a1 = t1, a3 = t3, a5 = t5;
        t0 = a0 * u0 + a1 * u2; t1 = a0 * u1 + a1 * u3;
        t2 = a2 * u0 + a3 * u2; t3 = a2 * u1 + a3 * u3;
        t4 = a4 * u0 + a5 * u2 + u4; t5 = a4 * u1 + a5 * u3 + u5;
    }
};

// AugmentationCoeff (caffe.proto:436-486) as a flat record: 42 float fields in declaration order (= protobuf descriptor
// order, which coeff_to_array / array_to_coeff and the (N,42,1,1) parameter blob rely on) with presence bits.
struct AugCoeff {
    static constexpr int N = 42;
    enum { MIRROR = 0, DX, DY, ANGLE, ZOOM_X, ZOOM_Y, GAMMA, BRIGHTNESS, CONTRAST, COLOR1, COLOR2, COLOR3,
           POW_NOMEAN0, POW_NOMEAN1, POW_NOMEAN2, ADD_NOMEAN0, ADD_NOMEAN1, ADD_NOMEAN2, MULT_NOMEAN0, MULT_NOMEAN1, MULT_NOMEAN2,
           POW_WITHMEAN0, POW_WITHMEAN1, POW_WITHMEAN2, ADD_WITHMEAN0, ADD_WITHMEAN1, ADD_WITHMEAN2, MULT_WITHMEAN0, MULT_WITHMEAN1,
           MULT_WITHMEAN2, LMULT_POW, LMULT_ADD, LMULT_MULT, COL_ANGLE, FOG_AMOUNT, FOG_SIZE, MOTION_BLUR_ANGLE, MOTION_BLUR_SIZE,
           SHADOW_ANGLE, SHADOW_DISTANCE, SHADOW_STRENGTH, NOISE };
    static float def(int f) {
        static const float d[N] = {0, 0, 0, 0, 1, 1,   1, 0, 1, 1, 1, 1,   1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 0, 1, 0,
                                   0, 0, 0, 0, 0, 0, 0, 0};
        return d[f];
    }
    float v[N];
    bool has[N];
    AugCoeff() { clear_all(); }
    void clear(int f) { v[f] = def(f); has[f] = false; }
    void clear_all() { for (int f = 0; f < N; f++) clear(f); }            // augmentation_layer_base.cpp:186-249
    void set(int f, float x) { v[f] = x; has[f] = true; }
    float get(int f) const { return v[f]; }
    // augmentation_layer_base.cpp:352-365: fields whose default is 0 are stored as is, the others as their logarithm
    void to_array(float* out) const {
        for (int f = 0; f < N; f++) out[f] = (std::fabs(def(f)) < 1e-3) ? v[f] : (float)std::log(v[f]);
    }
    void from_array(const float* in) {                                     // :368-379
        for (int f = 0; f < N; f++) set(f, (std::fabs(def(f)) < 1e-3) ? in[f] : (float)std::exp(in[f]));
    }
    void clear_defaults() {                                                // :339-349
        for (int f = 0; f < N; f++) if (std::fabs(def(f) - v[f]) < 1e-3) clear(f);
    }
};

// tTransMat::fromCoeff (augmentation_layer_base.cpp:38-48): crop (cw x ch) -> bottom (bw x bh) coordinates; each factor is
// applied when its coefficient is set
static TransMat TransMatFromCoeff(const AugCoeff& c, int cw, int ch, int bw, int bh) {
    TransMat t; t.toIdentity();
    if (c.get(AugCoeff::MIRROR)) t.leftMultiply(-1, 0, 0, 1, .5f * (float)cw, -.5f * (float)ch);
    else                         t.leftMultiply(1, 0, 0, 1, -.5f * (float)cw, -.5f * (float)ch);
    if (c.has[AugCoeff::ANGLE]) {
        const float a = c.get(AugCoeff::ANGLE);
        t.leftMultiply(std::cos(a), std::sin(a), -std::sin(a), std::cos(a), 0, 0);
    }
    if (c.has[AugCoeff::DX] || c.has[AugCoeff::DY])
        t.leftMultiply(1, 0, 0, 1, c.get(AugCoeff::DX) * (float)cw, c.get(AugCoeff::DY) * (float)ch);
    if (c.has[AugCoeff::ZOOM_X] || c.has[AugCoeff::ZOOM_Y])
        t.leftMultiply((float)(1.0 / c.get(AugCoeff::ZOOM_X)), 0, 0, (float)(1.0 / c.get(AugCoeff::ZOOM_Y)), 0, 0);
    t.leftMultiply(1, 0, 0, 1, .5f * (float)bw, .5f * (float)bh);
    return t;
}

// Which coefficient groups an augmentation_param samples: decided by the presence of their generators
// (data_augmentation_layer.cu:383-396)
struct AugGroups { bool spatial, chromatic, eigen, effect; };
static AugGroups SampledGroups(const AugmentationParameter& aug) {
    AugGroups g;
    g.spatial = aug.has("mirror") || aug.has("rotate") || aug.has("zoom") || aug.has("translate") || aug.has("squeeze") ||
                aug.has("translate_x") || aug.has("translate_y");
    g.chromatic = aug.has("brightness") || aug.has("gamma") || aug.has("contrast") || aug.has("color");
    g.effect = aug.has("fog_size") || aug.has("fog_amount") || aug.has("motion_blur_angle") || aug.has("motion_blur_size") ||
               aug.has("shadow_angle") || aug.has("shadow_distance") || aug.has("shadow_strength") || aug.has("noise");
    g.eigen = aug.has("lmult_pow") || aug.has("lmult_mult") || aug.has("lmult_add") || aug.has("sat_pow") || aug.has("sat_mult") ||
              aug.has("sat_add") || aug.has("col_pow") || aug.has("col_mult") || aug.has("col_add") || aug.has("ladd_pow") ||
              aug.has("ladd_mult") || aug.has("ladd_add") || aug.has("col_rotate");
    return g;
}

// Seed of a layer's coefficient sampler: FN2_SEED (default 1701, the reference tests' seed, test_gradient_check_util.hpp:25)
// hashed with the layer name
static uint32_t seed_of(const std::string& name) {
    uint32_t h = 1701u;
    if (const char* e = getenv("FN2_SEED")) h = (uint32_t)strtoul(e, nullptr, 10);
    for (char c : name) h = h * 16777619u ^ (unsigned char)c;
    return h;
}

// caffe_rng_generate, util/rng.cpp:8-114.  The reference draws from boost::mt19937 through boost's uniform_real /
// normal_distribution / bernoulli_distribution of an unpinned boost version: the random STREAM is unpinned, the
// distributions are restated (uniform on [mean-spread, mean+spread], N(mean, spread), Bernoulli(prob)).
struct AugRng {
    std::mt19937 gen;
    explicit AugRng(uint32_t seed) : gen(seed) {}
    float unit() { return (float)(gen() >> 8) * (1.0f / 16777216.0f); }                    // [0, 1)
    float uniform(float a, float b) { return a + (b - a) * unit(); }
    float gaussian(float mu, float sigma) {
        const float u1 = ((float)(gen() >> 8) + 1.0f) * (1.0f / 16777216.0f), u2 = unit();
        return mu + sigma * std::sqrt(-2.0f * std::log(u1)) * std::cos(6.28318530718f * u2);
    }
    int bernoulli(float p) { return unit() < p ? 1 : 0; }
    // Randtype float; as_bool reproduces the <Dtype,bool> instantiation used for `mirror`
    float generate(const RandomGeneratorParameter& p, float discount_coeff, float prob0_value, bool as_bool = false) {
        const float spread = p.apply_schedule() ? p.spread() * discount_coeff : p.spread();
        const std::string t = p.rand_type();
        float r;
        if (t == "uniform" || t == "gaussian") {
            float tmp = p.mean();
            if (spread > 0.f) tmp = (t == "uniform") ? uniform(p.mean() - spread, p.mean() + spread) : gaussian(p.mean(), spread);
            if (p.exp()) tmp = std::exp(tmp);
            r = tmp;
        } else if (t == "bernoulli") {
            r = (float)(p.prob() > 0.f ? bernoulli(p.prob()) : 0);
        } else if (t == "uniform_bernoulli" || t == "gaussian_bernoulli") {
            const int on = p.prob() > 0.f ? bernoulli(p.prob()) : 0;
            float tmp;
            if (!on) {
                if (!std::isnan(prob0_value)) return as_bool ? (prob0_value != 0.f ? 1.f : 0.f) : prob0_value;
                tmp = 0;
            } else {
                tmp = p.mean();
                if (spread > 0.f) tmp = (t == "uniform_bernoulli") ? uniform(p.mean() - spread, p.mean() + spread) : gaussian(p.mean(), spread);
            }
            if (p.exp()) tmp = std::exp(tmp);
            r = tmp;
        } else {
            CHECK(false) << "Unknown random type " << t;
            r = NAN;
        }
        if (as_bool) r = (r != 0.f) ? 1.f : 0.f;                              // static_cast<bool>
        if (p.discretize()) r = std::round(r);
        r = p.multiplier() * r;
        if (as_bool) r = (r != 0.f) ? 1.f : 0.f;
        return r;
    }
};

// Coefficient sampling of DataAugmentationLayer::Forward_gpu (data_augmentation_layer.cu:372-449) as a stand-alone object, so
// that it can be exercised without a GPU (fn2_aug_sample).
struct AugSampler {
    AugRng rng;
    explicit AugSampler(uint32_t seed) : rng(seed) {}
    // generate_spatial_coeffs, augmentation_layer_base.cpp:73-99
    void generate_spatial(const AugmentationParameter& aug, AugCoeff& c, float dc) {
        if (aug.has("mirror")) c.set(AugCoeff::MIRROR, rng.generate(aug.gen("mirror"), dc, AugCoeff::def(AugCoeff::MIRROR), true));
        if (aug.has("translate")) {
            c.set(AugCoeff::DX, rng.generate(aug.gen("translate"), dc, 0.f));
            c.set(AugCoeff::DY, rng.generate(aug.gen("translate"), dc, 0.f));
        }
        if (aug.has("translate_x")) c.set(AugCoeff::DX, rng.generate(aug.gen("translate_x"), dc, 0.f));
        if (aug.has("translate_y")) c.set(AugCoeff::DY, rng.generate(aug.gen("translate_y"), dc, 0.f));
        if (aug.has("rotate")) c.set(AugCoeff::ANGLE, rng.generate(aug.gen("rotate"), dc, 0.f));
        if (aug.has("zoom")) {
            c.set(AugCoeff::ZOOM_X, rng.generate(aug.gen("zoom"), dc, 1.f));
            c.set(AugCoeff::ZOOM_Y, c.get(AugCoeff::ZOOM_X));
        }
        if (aug.has("squeeze")) {
            const float sq = rng.generate(aug.gen("squeeze"), dc, 1.f);
            c.set(AugCoeff::ZOOM_X, c.get(AugCoeff::ZOOM_X) * sq);
            c.set(AugCoeff::ZOOM_Y, c.get(AugCoeff::ZOOM_Y) / sq);
        }
    }
    // generate_valid_spatial_coeffs, augmentation_layer_base.cpp:102-169: resample until the 4 corners of the crop land
    // inside the source image
    void generate_valid_spatial(const AugmentationParameter& aug, AugCoeff& coeff, float dc, int width, int height, int cw, int ch,
                                int max_num_tries = 50) {
        float in_params[AugCoeff::N], cur[AugCoeff::N];
        coeff.to_array(in_params);
        int counter = 0, good = 0;
        while (good < 4 && counter < max_num_tries) {
            coeff.clear_all();
            generate_spatial(aug, coeff, dc);
            coeff.to_array(cur);
            for (int f = 0; f < AugCoeff::N; f++) cur[f] += in_params[f];
            coeff.from_array(cur);
            good = 0;
            for (int x = 0; x < cw; x += std::max(1, cw - 1))
                for (int y = 0; y < ch; y += std::max(1, ch - 1)) {
                    float x1, y1, x2, y2;
                    if (coeff.get(AugCoeff::MIRROR)) { x1 = -(float)x + .5f * (float)cw; y1 = (float)y - .5f * (float)ch; }
                    else                            { x1 = (float)x - .5f * (float)cw;  y1 = (float)y - .5f * (float)ch; }
                    const float a = coeff.get(AugCoeff::ANGLE);
                    x2 = std::cos(a) * x1 - std::sin(a) * y1;
                    y2 = std::sin(a) * x1 + std::cos(a) * y1;
                    x2 = x2 + coeff.get(AugCoeff::DX) * (float)cw;
                    y2 = y2 + coeff.get(AugCoeff::DY) * (float)ch;
                    x2 = x2 / coeff.get(AugCoeff::ZOOM_X);
                    y2 = y2 / coeff.get(AugCoeff::ZOOM_Y);
                    x2 = x2 + .5f * (float)width;
                    y2 = y2 + .5f * (float)height;
                    if (!(std::floor(x2) < 0 || std::floor(x2) > (float)(width - 2) || std::floor(y2) < 0 || std::floor(y2) > (float)(height - 2)))
                        good++;
                }
            counter++;
        }
        if (counter >= max_num_tries) coeff.from_array(in_params);       // "Exceeded maximum tries in finding spatial coeffs."
    }
    // generate_chromatic_coeffs / _eigen_coeffs / _effect_coeffs, augmentation_layer_base.cpp:252-336
    void generate_chromatic(const AugmentationParameter& aug, AugCoeff& c, float dc) {
        if (aug.has("gamma")) c.set(AugCoeff::GAMMA, rng.generate(aug.gen("gamma"), dc, NAN));
        if (aug.has("brightness")) c.set(AugCoeff::BRIGHTNESS, rng.generate(aug.gen("brightness"), dc, NAN));
        if (aug.has("contrast")) c.set(AugCoeff::CONTRAST, rng.generate(aug.gen("contrast"), dc, NAN));
        if (aug.has("color")) for (int k = 0; k < 3; k++) c.set(AugCoeff::COLOR1 + k, rng.generate(aug.gen("color"), dc, NAN));
    }
    void generate_chromatic_eigen(const AugmentationParameter& aug, AugCoeff& c, float dc) {
        auto g = [&](const char* n) { return rng.generate(aug.gen(n), dc, NAN); };
        if (aug.has("ladd_pow")) c.set(AugCoeff::POW_NOMEAN0, g("ladd_pow"));
        if (aug.has("col_pow")) { c.set(AugCoeff::POW_NOMEAN1, g("col_pow")); c.set(AugCoeff::POW_NOMEAN2, g("col_pow")); }
        if (aug.has("ladd_add")) c.set(AugCoeff::ADD_NOMEAN0, g("ladd_add"));
        if (aug.has("col_add")) { c.set(AugCoeff::ADD_NOMEAN1, g("col_add")); c.set(AugCoeff::ADD_NOMEAN2, g("col_add")); }
        if (aug.has("ladd_mult")) c.set(AugCoeff::MULT_NOMEAN0, g("ladd_mult"));
        if (aug.has("col_mult")) { c.set(AugCoeff::MULT_NOMEAN1, g("col_mult")); c.set(AugCoeff::MULT_NOMEAN2, g("col_mult")); }
        if (aug.has("sat_pow")) { c.set(AugCoeff::POW_WITHMEAN1, g("sat_pow")); c.set(AugCoeff::POW_WITHMEAN2, c.get(AugCoeff::POW_WITHMEAN1)); }
        if (aug.has("sat_add")) { c.set(AugCoeff::ADD_WITHMEAN1, g("sat_add")); c.set(AugCoeff::ADD_WITHMEAN2, c.get(AugCoeff::ADD_WITHMEAN1)); }
        if (aug.has("sat_mult")) { c.set(AugCoeff::MULT_WITHMEAN1, g("sat_mult")); c.set(AugCoeff::MULT_WITHMEAN2, c.get(AugCoeff::MULT_WITHMEAN1)); }
        if (aug.has("lmult_pow")) c.set(AugCoeff::LMULT_POW, g("lmult_pow"));
        if (aug.has("lmult_mult")) c.set(AugCoeff::LMULT_MULT, g("lmult_mult"));
        if (aug.has("lmult_add")) c.set(AugCoeff::LMULT_ADD, g("lmult_add"));
        if (aug.has("col_rotate")) c.set(AugCoeff::COL_ANGLE, g("col_rotate"));
    }
    void generate_effect(const AugmentationParameter& aug, AugCoeff& c, float dc) {
        if (aug.has("fog_amount") || aug.has("fog_size")) {
            c.set(AugCoeff::FOG_AMOUNT, rng.generate(aug.gen("fog_amount"), dc, 0.f));
            c.set(AugCoeff::FOG_SIZE, rng.generate(aug.gen("fog_size"), dc, 0.f));
        }
        if (aug.has("motion_blur_angle") || aug.has("motion_blur_size")) {
            c.set(AugCoeff::MOTION_BLUR_ANGLE, rng.generate(aug.gen("motion_blur_angle"), dc, 0.f));
            c.set(AugCoeff::MOTION_BLUR_SIZE, rng.generate(aug.gen("motion_blur_size"), dc, 0.f));
        }
        if (aug.has("shadow_angle") || aug.has("shadow_distance") || aug.has("shadow_strength")) {
            c.set(AugCoeff::SHADOW_ANGLE, rng.generate(aug.gen("shadow_angle"), dc, 0.f));
            c.set(AugCoeff::SHADOW_DISTANCE, rng.generate(aug.gen("shadow_distance"), dc, 0.f));
            c.set(AugCoeff::SHADOW_STRENGTH, rng.generate(aug.gen("shadow_strength"), dc, 0.f));
        }
        if (aug.has("noise")) c.set(AugCoeff::NOISE, rng.generate(aug.gen("noise"), dc, NAN));
    }
    // one item
    void sample(const AugmentationParameter& aug, float dc, int width, int height, int cw, int ch, AugCoeff& c) {
        const AugGroups g = SampledGroups(aug);
        c.clear_all();
        if (g.spatial) generate_valid_spatial(aug, c, dc, width, height, cw, ch);
        if (g.chromatic) generate_chromatic(aug, c, dc);
        if (g.eigen) generate_chromatic_eigen(aug, c, dc);
        if (g.effect) generate_effect(aug, c, dc);
    }
    // discount schedule, data_augmentation_layer.cu:372-374
    static float discount(const LayerParameter& lp, float num_iter) {
        const float hl = lp.coeff_schedule_half_life(), c0 = lp.coeff_schedule_initial(), c1 = lp.coeff_schedule_final();
        return c0 + (c1 - c0) * (2.f / (1.f + std::exp(-1.0986f * num_iter / hl)) - 1.f);
    }
};

// C-ABI helper (capi.cpp: fn2_aug_sample): coefficients of `num` items in array form (N x 42)
void SampleAugmentationCoeffs(const LayerParameter& lp, uint32_t seed, int num, int width, int height, float num_iter, float* out) {
    AugmentationParameter aug = lp.augmentation_param();
    const int cw = aug.has_crop_width() ? aug.crop_width() : width, ch = aug.has_crop_height() ? aug.crop_height() : height;
    AugSampler sm(seed);
    const float dc = AugSampler::discount(lp, num_iter);
    for (int n = 0; n < num; n++) {
        AugCoeff c;
        sm.sample(aug, dc, width, height, cw, ch, c);
        c.to_array(out + (size_t)n * AugCoeff::N);
    }
}

template <typename Dtype>
class DataAugmentationLayer : public Layer<Dtype> {
 public:
    explicit DataAugmentationLayer(const LayerParameter& p) : Layer<Dtype>(p), sampler_(seed_of(p.name())) {}
    const char* type() const override { return "DataAugmentation"; }
    bool AllowBackward() const override { return false; }              // data_augmentation_layer.hpp:29
    bool DoesUseCustomCopyBlobs() const override { return true; }      // data_augmentation_layer.hpp:43-46
    void CustomCopyBlobs(const vector<Blob<Dtype>*>& blobs) override { adjust_blobs(blobs); }

    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        this->layer_param_.m->set("reshape_every_iter", "false");      // data_augmentation_layer.cpp:39
        if (this->blobs_.size() == 0) {
            this->blobs_.resize(aug.recompute_mean() ? 3 : 1);
            for (auto& b : this->blobs_) {
                b.reset(new Blob<Dtype>());
                // the iteration counter and the running means are state, not weights: one ParamSpec {lr_mult: 0 decay_mult: 0}
                // per blob keeps a solver off them (data_augmentation_layer.cpp:48-65)
                Field f;
                f.name = "param"; f.is_msg = true; f.msg = std::make_shared<Message>();
                f.msg->add("lr_mult", "0");
                f.msg->add("decay_mult", "0");
                this->layer_param_.m->fields.push_back(f);
            }
            this->blobs_[0]->Reshape(1, 1, 1, 1);
        }
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_GE(bottom.size(), 1u) << "Data augmentation layer takes one or two input blobs.";
        CHECK_LE(bottom.size(), 2u) << "Data augmentation layer takes one or two input blobs.";
        CHECK_GE(top.size(), 1u) << "Data augmentation layer outputs one or two output blobs.";
        CHECK_LE(top.size(), 2u) << "Data augmentation layer outputs one or two output blobs.";
        output_params_ = top.size() > 1;                               // data_augmentation_layer.cpp:83-84
        input_params_ = bottom.size() > 1;
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        const int num = bottom[0]->num(), channels = bottom[0]->channels();
        const int height = bottom[0]->height(), width = bottom[0]->width();
        do_cropping_ = aug.has_crop_width() && aug.has_crop_height();
        if (!do_cropping_) { cropped_width_ = width; cropped_height_ = height; }
        else {
            cropped_width_ = aug.crop_width();   CHECK_GE(width, cropped_width_) << "crop width greater than original";
            cropped_height_ = aug.crop_height(); CHECK_GE(height, cropped_height_) << "crop height greater than original";
        }
        top[0]->Reshape(num, channels, cropped_height_, cropped_width_);
        // coefficient blob: (N, 42, 1, 1), taken from bottom[1] or created here (:103-115)
        if (input_params_) {
            CHECK_EQ(bottom[1]->count(), num * AugCoeff::N) << "augmentation parameter blob must be (N," << AugCoeff::N << ",1,1)";
        }
        all_coeffs_.assign((size_t)num * AugCoeff::N, 0.f);
        if (output_params_) { top[1]->set_layout(Blob<Dtype>::PLAIN); top[1]->Reshape(num, AugCoeff::N, 1, 1); }
        // per-batch coefficient records, one pinned host block + one device block:
        //   [N x 6 matrices][N x 6 chromatic][N x 22 chromatic-eigen][N x 9 effects][9 eigvec][pad][32 eigenspace]
        off_mat_ = 0; off_chroma_ = off_mat_ + 6 * num; off_eigen_ = off_chroma_ + 6 * num; off_effect_ = off_eigen_ + 22 * num;
        off_eigvec_ = off_effect_ + 9 * num; off_space_ = (off_eigvec_ + 9 + 1) / 2 * 2; coef_floats_ = off_space_ + 32;
        coef_dev_.reserve(coef_floats_ * sizeof(float));
        coef_host_.reserve(coef_floats_ * sizeof(float));
        memset(coef_host_.get(), 0, coef_floats_ * sizeof(float));
        for (int i = 0; i < 9 && i < aug.chromatic_eigvec_size(); i++) coef_host_.as<float>()[off_eigvec_ + i] = aug.chromatic_eigvec(i);
        gen_active_ = do_cropping_ && !input_params_ && aug.has_any_generator() && (this->phase_ == TRAIN || aug.augment_during_test());
        // default coefficients -> one matrix per sample (data_augmentation_layer.cu:462-468); constant unless coefficients
        // are generated or received
        prepare_records(width, height);
        CUDA_CHECK(cudaMemcpy(coef_dev_.get(), coef_host_.get(), coef_floats_ * sizeof(float), cudaMemcpyHostToDevice));
        if (aug.recompute_mean()) {
            this->blobs_[1]->Reshape(1, channels, cropped_height_, cropped_width_);
            this->blobs_[2]->Reshape(1, channels, 1, 1);
        } else if (aug.mean_size() == 3 && !aug.mean_per_pixel()) {
            float mv[3] = {aug.mean(0), aug.mean(1), aug.mean(2)};
            fixed_mean_dev_.reserve(sizeof(mv));
            CUDA_CHECK(cudaMemcpy(fixed_mean_dev_.get(), mv, sizeof(mv), cudaMemcpyHostToDevice));
        }
        *(this->blobs_[0]->mutable_cpu_data()) = 0;                    // data_augmentation_layer.cpp:155
    }
    void FillParams(uint64_t seed) override {
        // synthetic "trained" state: iteration counter past recompute_mean, plausible RGB means
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        *(this->blobs_[0]->mutable_cpu_data()) = (float)(aug.recompute_mean() + 1);
        if (aug.recompute_mean()) {
            float* pc = this->blobs_[2]->mutable_cpu_data();
            float* pp = this->blobs_[1]->mutable_cpu_data();
            const int C = this->blobs_[2]->count(), area = this->blobs_[1]->count() / C;
            for (int c = 0; c < C; c++) {
                pc[c] = 0.40f + 0.02f * (float)c;
                for (int i = 0; i < area; i++) pp[(size_t)c * area + i] = pc[c];
            }
        }
        sampler_ = AugSampler((uint32_t)(seed * 2654435761u) ^ seed_of(this->layer_param_.name()));
    }
    void HostTick(int) override {
        float& num_iter = *(this->blobs_[0]->mutable_cpu_data());
        num_iter = (float)((int)num_iter + 1);                         // data_augmentation_layer.cu:353-354
        num_iter_ = num_iter;
    }
    bool GraphSafe() const override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        // while the running mean is still being updated the launch sequence changes per call; sampled or received
        // coefficients change the launch sequence and are uploaded from the host every call
        if (gen_active_ || input_params_ || output_params_) return false;
        return !(aug.recompute_mean() > 0 && num_iter_ <= (float)aug.recompute_mean());
    }

 protected:
    // all_coeffs_ (N x 42 array form) -> matrices / chromatic / eigen / effect records in coef_host_
    // (data_augmentation_layer.cu:452-477; tTransMat::fromCoeff augmentation_layer_base.cpp:38-48)
    void prepare_records(int bottomwidth, int bottomheight) {
        const int num = (int)(all_coeffs_.size() / AugCoeff::N);
        has_chromatic_ = has_eigen_ = has_effect_ = has_noise_ = false;
        for (int n = 0; n < num; n++) {
            AugCoeff c;
            c.from_array(&all_coeffs_[(size_t)n * AugCoeff::N]);
            c.clear_defaults();
            const TransMat t = TransMatFromCoeff(c, cropped_width_, cropped_height_, bottomwidth, bottomheight);
            float* const rec = coef_host_.as<float>();
            float* m = rec + off_mat_ + 6 * n;
            m[0] = t.t0; m[1] = t.t1; m[2] = t.t2; m[3] = t.t3; m[4] = t.t4; m[5] = t.t5;
            float* ch = rec + off_chroma_ + 6 * n;          // tChromaticCoeffs: gamma, brightness, contrast, color[3]
            ch[0] = c.get(AugCoeff::GAMMA); ch[1] = c.get(AugCoeff::BRIGHTNESS); ch[2] = c.get(AugCoeff::CONTRAST);
            for (int k = 0; k < 3; k++) ch[3 + k] = c.get(AugCoeff::COLOR1 + k);
            if (ch[0] != 1 || ch[1] != 0 || ch[2] != 1 || ch[3] != 1 || ch[4] != 1 || ch[5] != 1) has_chromatic_ = true;
            float* eg = rec + off_eigen_ + 22 * n;          // tChromaticEigenCoeffs
            for (int k = 0; k < 22; k++) {
                eg[k] = c.get(AugCoeff::POW_NOMEAN0 + k);
                if (eg[k] != AugCoeff::def(AugCoeff::POW_NOMEAN0 + k)) has_eigen_ = true;
            }
            float* ef = rec + off_effect_ + 9 * n;          // tEffectCoeffs
            ef[0] = c.get(AugCoeff::FOG_AMOUNT); ef[1] = c.get(AugCoeff::FOG_SIZE);
            ef[2] = c.get(AugCoeff::MOTION_BLUR_ANGLE); ef[3] = c.get(AugCoeff::MOTION_BLUR_SIZE);
            ef[4] = std::cos(c.get(AugCoeff::SHADOW_ANGLE)); ef[5] = std::sin(c.get(AugCoeff::SHADOW_ANGLE));
            ef[6] = c.get(AugCoeff::SHADOW_DISTANCE); ef[7] = c.get(AugCoeff::SHADOW_STRENGTH); ef[8] = c.get(AugCoeff::NOISE);
            if ((ef[0] != 0 && ef[1] != 0) || ef[3] > 0 || ef[7] > 0 || ef[8] > 0) has_effect_ = true;
            if (ef[8] > 0) has_noise_ = true;
        }
    }

    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        const int num = bottom[0]->num();
        float* coef = coef_dev_.as<float>();
        if (do_cropping_) {
            if (gen_active_ || input_params_) {
                if (input_params_) {
                    const float* in = bottom[1]->cpu_data();              // "Receiving augmentation params" (:107-109)
                    all_coeffs_.assign(in, in + (size_t)num * AugCoeff::N);
                } else {
                    const float dc = AugSampler::discount(this->layer_param_, num_iter_);
                    for (int n = 0; n < num; n++) {
                        AugCoeff c;
                        sampler_.sample(aug, dc, bottom[0]->width(), bottom[0]->height(), cropped_width_, cropped_height_, c);
                        c.to_array(&all_coeffs_[(size_t)n * AugCoeff::N]);
                    }
                }
                prepare_records(bottom[0]->width(), bottom[0]->height());
                CUDA_CHECK(cudaMemcpyAsync(coef_dev_.get(), coef_host_.get(), (size_t)off_eigvec_ * sizeof(float), cudaMemcpyHostToDevice, S()));
            }
            if (output_params_) memcpy(top[1]->mutable_cpu_data(), all_coeffs_.data(), all_coeffs_.size() * sizeof(float));
            if (has_eigen_) {
                CHECK_EQ(bottom[0]->channels(), 3) << "Chromatic-Eigen augmentations only work with 3-channel input";
                CHECK_EQ(aug.chromatic_eigvec_size(), 9) << "You need to specify chromatic eigenvectors for Chromatic-Eigen augmentation";
                FN2_CALL(fn2_chromatic_eigenspace(&b, coef + off_eigvec_, coef + off_space_, S()));
            }
            FN2_CALL(fn2_spatial_augmentation(&b, &t, coef + off_mat_, S()));
            if (has_eigen_) FN2_CALL(fn2_chromatic_eigen_augmentation(&t, coef + off_eigen_, coef + off_space_, aug.max_multiplier(), S()));
            if (has_chromatic_) {
                CHECK_EQ(bottom[0]->channels(), 3) << "Chromatic augmentations only work with 3-channel input";
                FN2_CALL(fn2_color_contrast_augmentation(&t, coef + off_chroma_, aug.max_multiplier(), S()));
            }
            if (has_effect_) {
                CHECK_EQ(bottom[0]->channels(), 3) << "Effect augmentations only work with 3-channel input";
                FN2_CALL(fn2_apply_effects(&t, coef + off_effect_, aug.max_multiplier(), (unsigned long long)sampler_.rng.gen() << 32 | sampler_.rng.gen(),
                                           has_noise_ ? 1 : 0, S()));
            }
            if (gen_active_ || input_params_) CUDA_CHECK(cudaStreamSynchronize(S()));   // coef_host_ is rewritten next call
        } else {
            FN2_CALL(fn2_copy(&b, &t, S()));                                            // data_augmentation_layer.cu:589
        }
        if (aug.recompute_mean() > 0) {
            fn2_tensor mpp = this->blobs_[1]->mutable_tensor();
            float* mpc = this->blobs_[2]->mutable_gpu_data();
            if (num_iter_ <= (float)aug.recompute_mean()) FN2_CALL(fn2_mean_update(&t, &mpp, mpc, num_iter_, S()));
            FN2_CALL(fn2_mean_subtract(&t, &mpp, mpc, aug.mean_per_pixel() ? 1 : 0, S()));
        } else if (aug.mean_size() == 3 && !aug.mean_per_pixel()) {
            FN2_CALL(fn2_mean_subtract(&t, nullptr, fixed_mean_dev_.as<float>(), 0, S()));
        }
    }

    // data_augmentation_layer.cpp:162-205
    void adjust_blobs(const vector<Blob<Dtype>*>& blobs) {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        if (aug.recompute_mean() > 0 && blobs.size() >= 2) {
            CHECK_GE(blobs.size(), 3u) << "DataAugmentation: source layer must carry 3 blobs";
            CHECK_EQ(this->blobs_[1]->channels(), blobs[1]->shape(1));
            const bool same_size = this->blobs_[1]->width() == blobs[1]->shape(3) && this->blobs_[1]->height() == blobs[1]->shape(2);
            const int channels = this->blobs_[1]->channels();
            const int area = this->blobs_[1]->height() * this->blobs_[1]->width();
            const int source_area = blobs[1]->shape(2) * blobs[1]->shape(3);
            *(this->blobs_[0]->mutable_cpu_data()) = blobs[0]->cpu_data()[0];
            if (!aug.mean_per_pixel()) {
                CHECK_EQ(this->blobs_[2]->count(), blobs[2]->count());
                memcpy(this->blobs_[2]->mutable_cpu_data(), blobs[2]->cpu_data(), sizeof(float) * this->blobs_[2]->count());
            } else {
                const float* src = blobs[1]->cpu_data();
                float* pc = this->blobs_[2]->mutable_cpu_data();
                // per-channel average (caffe_cpu_gemv with ones; CBLAS order unpinned -> double)
                for (int c = 0; c < channels; c++) {
                    double acc = 0;
                    for (int i = 0; i < source_area; i++) acc += src[(size_t)c * source_area + i];
                    pc[c] = (float)((1.0 / source_area) * acc);
                }
                float* pp = this->blobs_[1]->mutable_cpu_data();
                if (same_size) memcpy(pp, src, sizeof(float) * (size_t)channels * area);
                else for (int c = 0; c < channels; c++) for (int i = 0; i < area; i++) pp[(size_t)c * area + i] = pc[c];
            }
        }
    }

    bool do_cropping_ = false, input_params_ = false, output_params_ = false, gen_active_ = false;
    bool has_chromatic_ = false, has_eigen_ = false, has_effect_ = false, has_noise_ = false;
    int cropped_width_ = 0, cropped_height_ = 0;
    float num_iter_ = 0;
    vector<float> all_coeffs_;                   // N x 42, array form (coeff_to_array)
    DeviceBuffer coef_host_{DeviceBuffer::PINNED_HOST};   // uploaded asynchronously
    DeviceBuffer coef_dev_;
    size_t coef_floats_ = 0;
    int off_mat_ = 0, off_chroma_ = 0, off_eigen_ = 0, off_effect_ = 0, off_eigvec_ = 0, off_space_ = 0;
    DeviceBuffer fixed_mean_dev_;
    AugSampler sampler_;
};
REGISTER_LAYER_CLASS(DataAugmentation);

// ---------------------------------------------------------------------------------------------
// Training-side layers next to the FlowNet2-C training step (SURVEY.md 8 "next" row 2)
// ---------------------------------------------------------------------------------------------
// array_to_coeff sets every field (augmentation_layer_base.cpp:368-379), so fromCoeff applies every factor
static TransMat TransMatFromArray(const float* arr, int cw, int ch, int bw, int bh) {
    AugCoeff c;
    c.from_array(arr);
    return TransMatFromCoeff(c, cw, ch, bw, bh);
}
static TransMat TransMatInverse(const TransMat& m) {              // augmentation_layer_base.cpp:51-68
    const float a = m.t0, c = m.t2, e = m.t4, b = m.t1, d = m.t3, f = m.t5;
    const float denom = a * d - b * c;
    TransMat r;
    r.t0 = d / denom; r.t1 = -b / denom; r.t2 = -c / denom; r.t3 = a / denom;
    r.t4 = (c * f - d * e) / denom; r.t5 = (b * e - a * f) / denom;
    return r;
}

// L1Loss (l1_loss_layer.hpp, l1loss_layer.cpp:11-90, l1loss_layer.cu:67-192): NaN-masked L1 / end-point-error loss
template <typename Dtype>
class L1LossLayer : public Layer<Dtype> {
 public:
    explicit L1LossLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "L1Loss"; }
    bool IsLossLayer() const override { return true; }
    typename Blob<Dtype>::Layout TopLayout() const override { return Blob<Dtype>::PLAIN; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK(bottom.size() == 1 || bottom.size() == 2) << "L1LossLayer needs one or two input blobs.";
        const Message& lp = this->layer_param_.m->msg("l1_loss_param");
        d_.l2_per_location = lp.b("l2_per_location", false) ? 1 : 0;
        d_.l2_prescale_by_channels = lp.b("l2_prescale_by_channels", false) ? 1 : 0;
        d_.normalize_by_num_entries = lp.b("normalize_by_num_entries", false) ? 1 : 0;
        d_.epsilon = lp.f("epsilon", 1e-2f);
        d_.plateau = lp.f("plateau", 0.f);
        state_.reserve(4 * sizeof(float), S());
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        if (bottom.size() > 1) CHECK(bottom[0]->shape() == bottom[1]->shape()) << "L1Loss: bottoms must have the same shape";
        top[0]->set_layout(Blob<Dtype>::PLAIN);
        top[0]->Reshape(vector<int>());                               // loss layers output a scalar (l1loss_layer.cpp:69-70)
        size_t need = 0;
        FN2_CALL(fn2_l1loss_workspace_bytes(bottom[0]->num(), bottom[0]->height(), bottom[0]->width(), &need));
        ws_.reserve(need);
    }
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b0 = bottom[0]->tensor(), b1 = b0;
        if (bottom.size() > 1) b1 = bottom[1]->tensor();
        FN2_CALL(fn2_l1loss_forward(&b0, bottom.size() > 1 ? &b1 : nullptr, &d_, state_.as<float>(), top[0]->mutable_gpu_data(), ws_.get(),
                                    ws_.bytes(), S()));
    }
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        const bool p0 = propagate_down[0], p1 = bottom.size() > 1 && propagate_down[1];
        if (!p0 && !p1) return;
        fn2_tensor b0 = bottom[0]->tensor(), b1 = b0, d0 = b0, d1 = b0;
        if (bottom.size() > 1) b1 = bottom[1]->tensor();
        if (p0) d0 = bottom[0]->diff_tensor();
        if (p1) d1 = bottom[1]->diff_tensor();
        fn2_tensor td = top[0]->diff_tensor();
        FN2_CALL(fn2_l1loss_backward(&b0, bottom.size() > 1 ? &b1 : nullptr, &d_, state_.as<float>(), td.data, p0 ? &d0 : nullptr, p1 ? &d1 : nullptr,
                                     this->bottom_accumulate_[0] ? 1 : 0, bottom.size() > 1 && this->bottom_accumulate_[1] ? 1 : 0, S()));
    }
 protected:
    fn2_l1loss_desc d_;
    DeviceBuffer state_, ws_;
};
REGISTER_LAYER_CLASS(L1Loss);

// LpqLoss (lpq_loss_layer.hpp, lpq_loss_layer.cpp:13-138, lpq_loss_layer.cu:96-245): the robust NaN-masked
// sum_locations (sum_c w (|d_c| + p_epsilon)^p + q_epsilon)^q / norm, with p and q following a schedule over the net's iteration
template <typename Dtype>
class LpqLossLayer : public Layer<Dtype> {
 public:
    explicit LpqLossLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "LpqLoss"; }
    bool IsLossLayer() const override { return true; }
    typename Blob<Dtype>::Layout TopLayout() const override { return Blob<Dtype>::PLAIN; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const Message& lp = this->layer_param_.m->msg("lpq_loss_param");
        const int ns = lp.count("pq_episode_starts_at_iter"), np = lp.count("p"), nq = lp.count("q");
        starts_.clear(); p_.clear(); q_.clear();
        // lpq_loss_layer.cpp:19-82: one p and one q without start iterations are constant values; otherwise the three lists
        // have equal, non-zero sizes, strictly increasing start iterations, and the first one is 0
        if (ns == 0 && np == 1 && nq == 1) {
            starts_.push_back(0);
        } else {
            if (ns != np || np != nq) {
                std::ostringstream os;
                os << "Incompatible sizes: (pq_episode_starts_at_iter -> " << ns << ", p -> " << np << ", q -> " << nq << ")";
                throw CaffeError(os.str());
            }
            if (ns < 1) throw CaffeError("Lpq schedule parameters must not be empty");
            for (int i = 0; i < ns; i++) starts_.push_back((unsigned)lp.num("pq_episode_starts_at_iter", 0, i));
            for (int i = 0; i + 1 < ns; i++)
                if (starts_[i] >= starts_[i + 1]) {
                    std::ostringstream os;
                    os << "pq_episode_starts_at_frame is not ordered or contains duplicates:";
                    for (unsigned v : starts_) os << " " << v;
                    throw CaffeError(os.str());
                }
            if (starts_[0] != 0) throw CaffeError("First entry in pq_episode_starts_at_frame is not 0, this is probably a mistake.");
        }
        for (int i = 0; i < np; i++) { p_.push_back(lp.f("p", 0.f, i)); q_.push_back(lp.f("q", 0.f, i)); }
        CHECK(bottom.size() == 1 || bottom.size() == 2) << "LpqLossLayer needs one or two input blobs.";
        d_.p_epsilon = lp.f("p_epsilon", 0.f);
        d_.q_epsilon = lp.f("q_epsilon", 1e-2f);
        d_.l2_prescale_by_channels = lp.b("l2_prescale_by_channels", false) ? 1 : 0;
        d_.normalize_by_num_entries = lp.b("normalize_by_num_entries", false) ? 1 : 0;
        state_.reserve(FN2_LPQLOSS_STATE_FLOATS * sizeof(float), S());
        step_ = -1;
    }
    // The schedule step of iteration `iter`: the last one whose start iteration is <= iter.  The reference pops a queue as the
    // iteration grows (lpq_loss_layer.cu:100-135), which gives the same step whenever the iteration only grows; the lookup also
    // stays right after a Solver restore to an earlier iteration.  A changed (p, q) goes to the device state with one copy on
    // the net's stream: after the previous backward, which still reads the old pair, and before this forward or its graph
    // replay.  The source is pageable, so the copy has taken the values by the time it returns.
    void HostTick(int iter) override {
        int k = 0;
        while (k + 1 < (int)starts_.size() && starts_[k + 1] <= (unsigned)iter) k++;
        if (k == step_) return;
        step_ = k;
        pq_[0] = p_[k]; pq_[1] = q_[k];
        CUDA_CHECK(cudaMemcpyAsync(state_.as<float>() + 4, pq_, sizeof(pq_), cudaMemcpyHostToDevice, S()));
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        if (bottom.size() > 1) CHECK(bottom[0]->shape() == bottom[1]->shape()) << "LpqLoss: bottoms must have the same shape";
        top[0]->set_layout(Blob<Dtype>::PLAIN);
        top[0]->Reshape(vector<int>());                               // loss layers output a scalar (lpq_loss_layer.cpp:144-146)
        size_t need = 0;
        FN2_CALL(fn2_lpqloss_workspace_bytes(bottom[0]->num(), bottom[0]->height(), bottom[0]->width(), &need));
        ws_.reserve(need);
    }
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b0 = bottom[0]->tensor(), b1 = b0;
        if (bottom.size() > 1) b1 = bottom[1]->tensor();
        FN2_CALL(fn2_lpqloss_forward(&b0, bottom.size() > 1 ? &b1 : nullptr, &d_, state_.as<float>(), top[0]->mutable_gpu_data(), ws_.get(),
                                     ws_.bytes(), S()));
    }
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        const bool p0 = propagate_down[0], p1 = bottom.size() > 1 && propagate_down[1];
        if (!p0 && !p1) return;
        fn2_tensor b0 = bottom[0]->tensor(), b1 = b0, d0 = b0, d1 = b0;
        if (bottom.size() > 1) b1 = bottom[1]->tensor();
        if (p0) d0 = bottom[0]->diff_tensor();
        if (p1) d1 = bottom[1]->diff_tensor();
        fn2_tensor td = top[0]->diff_tensor();
        FN2_CALL(fn2_lpqloss_backward(&b0, bottom.size() > 1 ? &b1 : nullptr, &d_, state_.as<float>(), td.data, p0 ? &d0 : nullptr, p1 ? &d1 : nullptr,
                                      this->bottom_accumulate_[0] ? 1 : 0, bottom.size() > 1 && this->bottom_accumulate_[1] ? 1 : 0, S()));
    }
 protected:
    fn2_lpqloss_desc d_;
    vector<unsigned> starts_;
    vector<float> p_, q_;
    float pq_[2] = {0.f, 0.f};
    int step_ = -1;
    DeviceBuffer state_, ws_;
};
REGISTER_LAYER_CLASS(LpqLoss);

// Downsample (downsample_layer.cpp:20-58, downsample_layer.cu:15-80): ground-truth pyramid for the multi-scale losses
template <typename Dtype>
class DownsampleLayer : public Layer<Dtype> {
 public:
    explicit DownsampleLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Downsample"; }
    bool AllowBackward() const override { return false; }             // "DownsamplingLayer cannot do backward." (.cu:131-137)
    typename Blob<Dtype>::Layout TopLayout() const override { return Blob<Dtype>::PLAIN; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK(bottom.size() >= 1 && bottom.size() <= 2 && top.size() == 1) << "Downsample takes one or two bottoms and one top";
        this->layer_param_.m->set("reshape_every_iter", "false");
        int th, tw;
        if (bottom.size() == 1) {
            const Message& dp = this->layer_param_.m->msg("downsample_param");
            th = dp.i("top_height", 0); tw = dp.i("top_width", 0);
        } else { th = bottom[1]->height(); tw = bottom[1]->width(); }
        CHECK_GE(th, 1) << "DownsampleLayer must have top_height > 0";
        CHECK_GE(tw, 1) << "DownsampleLayer must have top_width > 0";
        top[0]->Reshape(bottom[0]->num(), bottom[0]->channels(), th, tw);
    }
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_downsample_forward(&b, &t, S()));
    }
};
REGISTER_LAYER_CLASS(Downsample);

// FlowAugmentation (flow_augmentation_layer.cpp:30-75, .cu:24-166): the ground-truth flow under the two images' spatial
// transforms.  bottoms: flow, coefficient blob of image 1, coefficient blob of image 2 (N x 42 each).
template <typename Dtype>
class FlowAugmentationLayer : public Layer<Dtype> {
 public:
    explicit FlowAugmentationLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "FlowAugmentation"; }
    bool AllowBackward() const override { return false; }             // flow_augmentation_layer.hpp
    bool GraphSafe() const override { return false; }                 // the matrices come from host blobs every pass
    typename Blob<Dtype>::Layout TopLayout() const override { return Blob<Dtype>::PLAIN; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        CHECK_GT(aug.crop_width(), 0) << "Please enter crop width if you want to perform augmentation";
        CHECK_GT(aug.crop_height(), 0) << "Please enter crop height if you want to perform augmentation";
        this->layer_param_.m->set("reshape_every_iter", "false");
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom.size(), 3) << "Flow augmentation layer takes three input blobs: FlowField, Img1TransfParams, Img2TransfParams";
        CHECK_EQ(top.size(), 1) << "Flow augmentation layer outputs one output blob: Augmented Flow";
        CHECK_EQ(bottom[0]->channels(), 2) << "Flow data must have two channels";
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        cw_ = aug.crop_width(); ch_ = aug.crop_height();
        const int num = bottom[0]->num();
        top[0]->Reshape(num, 2, ch_, cw_);
        mats_dev_.reserve((size_t)num * 12 * sizeof(float));
        mats_host_.reserve((size_t)num * 12 * sizeof(float));
    }
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        const int num = bottom[0]->num();
        CHECK_EQ(bottom[1]->count(), num * AugCoeff::N) << "FlowAugmentation: coefficient blob 1 must be N x 42";
        CHECK_EQ(bottom[2]->count(), num * AugCoeff::N) << "FlowAugmentation: coefficient blob 2 must be N x 42";
        const float* p1 = bottom[1]->cpu_data();
        const float* p2 = bottom[2]->cpu_data();
        CUDA_CHECK(cudaStreamSynchronize(S()));                         // the previous pass may still read mats_host_
        for (int n = 0; n < num; n++) {
            const TransMat m1 = TransMatFromArray(p1 + (size_t)n * AugCoeff::N, cw_, ch_, bottom[0]->width(), bottom[0]->height());
            const TransMat m2 = TransMatInverse(TransMatFromArray(p2 + (size_t)n * AugCoeff::N, cw_, ch_, bottom[0]->width(), bottom[0]->height()));
            float* a = mats_host_.as<float>() + 6 * n;
            float* b = mats_host_.as<float>() + 6 * num + 6 * n;
            a[0] = m1.t0; a[1] = m1.t1; a[2] = m1.t2; a[3] = m1.t3; a[4] = m1.t4; a[5] = m1.t5;
            b[0] = m2.t0; b[1] = m2.t1; b[2] = m2.t2; b[3] = m2.t3; b[4] = m2.t4; b[5] = m2.t5;
        }
        CUDA_CHECK(cudaMemcpyAsync(mats_dev_.get(), mats_host_.get(), (size_t)num * 12 * sizeof(float), cudaMemcpyHostToDevice, S()));
        fn2_tensor b = bottom[0]->tensor(), t = top[0]->mutable_tensor();
        FN2_CALL(fn2_flow_augmentation(&b, &t, mats_dev_.as<float>(), mats_dev_.as<float>() + 6 * num, S()));
    }
 protected:
    int cw_ = 0, ch_ = 0;
    DeviceBuffer mats_dev_;
    DeviceBuffer mats_host_{DeviceBuffer::PINNED_HOST};   // uploaded asynchronously
};
REGISTER_LAYER_CLASS(FlowAugmentation);

// GenerateAugmentationParameters (generate_augmentation_parameters_layer.cpp:33-105, .cu:16-117): host-only coefficient
// generator; modes "add" / "replace" / "regenerate" against an incoming coefficient blob.
template <typename Dtype>
class GenerateAugmentationParametersLayer : public Layer<Dtype> {
 public:
    explicit GenerateAugmentationParametersLayer(const LayerParameter& p) : Layer<Dtype>(p), sampler_(seed_of(p.name())) {}
    const char* type() const override { return "GenerateAugmentationParameters"; }
    bool AllowBackward() const override { return false; }
    bool GraphSafe() const override { return false; }
    typename Blob<Dtype>::Layout TopLayout() const override { return Blob<Dtype>::PLAIN; }
    void LayerSetUp(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        this->layer_param_.m->set("reshape_every_iter", "false");
    }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        CHECK(bottom.size() == 1 || bottom.size() == 3) << "Generate augmentation parameters layer takes one (any blob from which it can "
            "take num and potentially original image size) or three (aug params, orig data, augmented data) input blobs.";
        CHECK_EQ(top.size(), 1) << "Generate augmentation parameters layer outputs one output blob.";
        mode_ = aug.m->str_or("mode", "add");
        if (bottom.size() == 1 && (bottom[0]->width() > 1 || bottom[0]->height() > 1)) mode_ = "regenerate";
        num_ = bottom[0]->num();
        if (bottom.size() == 3) {
            cw_ = bottom[2]->width(); ch_ = bottom[2]->height(); bw_ = bottom[1]->width(); bh_ = bottom[1]->height();
        } else {
            CHECK(aug.has_crop_width() && aug.has_crop_height()) << "Need crop_width and crop_height if there is no blob specifying these";
            cw_ = aug.crop_width(); ch_ = aug.crop_height();
            if (bottom[0]->width() > 1 || bottom[0]->height() > 1) { bw_ = bottom[0]->width(); bh_ = bottom[0]->height(); }
            else {
                CHECK(aug.m->has("bottomwidth") && aug.m->has("bottomheight")) << "Need bottomwidth and bottomheight if there is no blob specifying these";
                bw_ = aug.m->i("bottomwidth", 0); bh_ = aug.m->i("bottomheight", 0);
            }
        }
        CHECK_GE(num_, 1) << "Must provide num with a bottom blob or in the prototxt";
        top[0]->set_layout(Blob<Dtype>::PLAIN);
        top[0]->Reshape(num_, AugCoeff::N, 1, 1);
        num_iter_ = 0;
    }
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        AugmentationParameter aug = this->layer_param_.augmentation_param();
        num_iter_++;
        const float dc = AugSampler::discount(this->layer_param_, (float)num_iter_);
        AugGroups g = {false, false, false, false};
        if (this->phase_ == TRAIN || aug.augment_during_test()) g = SampledGroups(aug);
        if (g.spatial) CHECK(cw_ >= 1 && ch_ >= 1 && bw_ >= 1 && bh_ >= 1) << "Must provide crop and bottom sizes to do spatial augmentations";
        const bool use_in = mode_ == "add" || mode_ == "replace";
        const float* in = use_in ? bottom[0]->cpu_data() : nullptr;
        float* out = top[0]->mutable_cpu_data();
        const bool fresh = mode_ == "regenerate" || mode_ == "replace";
        for (int n = 0; n < num_; n++) {
            AugCoeff c;
            if (use_in) c.from_array(in + (size_t)n * AugCoeff::N);
            if (g.spatial) {
                if (mode_ == "replace") for (int f = AugCoeff::MIRROR; f <= AugCoeff::ZOOM_Y; f++) c.clear(f);     // clear_spatial_coeffs
                sampler_.generate_valid_spatial(aug, c, dc, bw_, bh_, cw_, ch_, 50);
            }
            float* o = out + (size_t)n * AugCoeff::N;
            c.to_array(o);
            // the other groups either overwrite fields of the running record ("regenerate" / "replace") or are drawn into a fresh
            // record whose array form is ADDED (add_coeff_to_array, augmentation_layer_base.cpp:172-180)
            auto group = [&](bool on, void (AugSampler::*gen)(const AugmentationParameter&, AugCoeff&, float)) {
                if (!on) return;
                if (fresh) { (sampler_.*gen)(aug, c, dc); c.to_array(o); }
                else {
                    AugCoeff tmp;
                    (sampler_.*gen)(aug, tmp, dc);
                    float arr[AugCoeff::N];
                    tmp.to_array(arr);
                    for (int f = 0; f < AugCoeff::N; f++) o[f] += arr[f];
                }
            };
            group(g.chromatic, &AugSampler::generate_chromatic);
            group(g.eigen, &AugSampler::generate_chromatic_eigen);
            group(g.effect, &AugSampler::generate_effect);
        }
    }
 protected:
    std::string mode_;
    int num_ = 0, cw_ = 0, ch_ = 0, bw_ = 0, bh_ = 0, num_iter_ = 0;
    AugSampler sampler_;
};
REGISTER_LAYER_CLASS(GenerateAugmentationParameters);

// Split (split_layer.cpp:9-52): the layer Net::Init's InsertSplits puts behind every blob with several readers.  This executor
// needs none (fan-out costs nothing in the forward pass, Net::PlanBackward accumulates the gradients), but a prototxt that already
// contains Split layers -- e.g. one written back by the reference's upgrade tools -- must load: tops are copies of the bottom,
// the backward sums the top diffs (split_layer.cpp:38-52).
template <typename Dtype>
class SplitLayer : public Layer<Dtype> {
 public:
    explicit SplitLayer(const LayerParameter& p) : Layer<Dtype>(p) {}
    const char* type() const override { return "Split"; }
    void Reshape(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        CHECK_EQ(bottom.size(), 1u) << "Split takes one bottom";
        for (Blob<Dtype>* t : top) {
            CHECK(t != bottom[0]) << this->type() << " Layer does not allow in-place computation.";       // split_layer.cpp:17-19
            t->ReshapeLike(*bottom[0]);
        }
    }
 protected:
    void Forward_gpu(const vector<Blob<Dtype>*>& bottom, const vector<Blob<Dtype>*>& top) override {
        fn2_tensor s = bottom[0]->tensor();
        for (Blob<Dtype>* t : top) {
            fn2_tensor d = t->mutable_tensor();
            FN2_CALL(fn2_copy(&s, &d, S()));
        }
    }
    void Backward_gpu(const vector<Blob<Dtype>*>& top, const vector<bool>& propagate_down, const vector<Blob<Dtype>*>& bottom) override {
        if (!propagate_down[0]) return;
        fn2_tensor dx = bottom[0]->diff_tensor();
        for (size_t i = 0; i < top.size(); i++) {
            fn2_tensor dy = top[i]->diff_tensor();
            FN2_CALL(fn2_axpby(&dy, 1.f, &dx, (i > 0 || this->bottom_accumulate_[0]) ? 1.f : 0.f, S()));
        }
    }
};
REGISTER_LAYER_CLASS(Split);

// referenced by net.cpp to force this translation unit (and its static registrars) to link
void RegisterFlowNetLayers() {}

// helpers for net.cpp's ReLU fusion
bool IsReLULayer(Layer<float>* l, float* slope) {
    auto* r = dynamic_cast<ReLULayer<float>*>(l);
    if (!r) return false;
    *slope = r->negative_slope();
    return true;
}
void MarkReLUFused(Layer<float>* l) {
    if (auto* r = dynamic_cast<ReLULayer<float>*>(l)) r->set_fused(true);
}

}  // namespace caffe
