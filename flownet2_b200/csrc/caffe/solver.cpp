#include "solver.hpp"

#include <cmath>
#include <cstring>

namespace caffe {

namespace {
// Fields that take effect here, and fields accepted with no effect: the caller builds the TRAIN net itself (net, train_net),
// runs on the GPU it chose (solver_mode GPU, device_id), seeds through FN2_SEED (random_seed), and has no test nets to run or
// log to print (test_compute_loss, test_initialization, display, debug_info).  rms_decay belongs to RMSProp.
const char* const kKnown[] = {
    "type", "base_lr", "lr_policy", "gamma", "power", "stepsize", "stepvalue", "max_iter", "momentum", "momentum2", "delta",
    "weight_decay", "regularization_type", "clip_gradients", "iter_size", "average_loss", "snapshot", "snapshot_prefix",
    "snapshot_after_train", "snapshot_format", "snapshot_diff", "solver_mode", "test_interval",
    "net", "train_net", "display", "debug_info", "device_id", "random_seed", "test_compute_loss", "test_initialization", "rms_decay"};
const char* const kPolicies[] = {"fixed", "step", "exp", "inv", "multistep", "poly", "sigmoid"};

size_t slot(long long count) { return (size_t)(count + 63) / 64 * 64; }
}  // namespace

void Solver::Validate(const SolverParameter& p) {
    const Message& m = *p.m;
    for (const Field& f : m.fields) {
        if (f.name == "test_net" || f.name == "test_net_param" || f.name == "test_iter" || f.name == "test_state")
            throw CaffeError("SolverParameter." + f.name + ": test nets are not supported by this solver; run the TEST net "
                             "separately");
        bool known = false;
        for (const char* k : kKnown) if (f.name == k) known = true;
        if (!known) throw CaffeError("SolverParameter." + f.name + " is not supported by this solver");
    }
    const std::string type = p.type();
    if (type != "SGD" && type != "Adam")
        throw CaffeError("SolverParameter.type: solver type " + type + " is not supported (this solver runs SGD and Adam)");
    if (m.i("test_interval", 0) > 0)
        throw CaffeError("SolverParameter.test_interval: test nets are not supported by this solver; run the TEST net separately");
    const std::string fmt = m.str_or("snapshot_format", "BINARYPROTO");
    if (fmt != "BINARYPROTO" && fmt != "1")
        throw CaffeError("SolverParameter.snapshot_format: " + fmt + " snapshots are not supported (BINARYPROTO)");
    if (m.b("snapshot_diff", false)) throw CaffeError("SolverParameter.snapshot_diff: diff snapshots are not supported");
    const std::string mode = m.str_or("solver_mode", "GPU");
    if (mode != "GPU" && mode != "1") throw CaffeError("SolverParameter.solver_mode: " + mode + " is not supported (GPU)");
    bool policy = false;
    for (const char* k : kPolicies) if (p.lr_policy() == k) policy = true;
    if (!policy) throw CaffeError("Unknown learning rate policy: " + p.lr_policy());        // sgd_solver.cpp:60
    if (p.regularization_type() != "L2" && p.regularization_type() != "L1")
        throw CaffeError("Unknown regularization type: " + p.regularization_type());           // sgd_solver.cpp:170
    if (p.lr_policy() == "step" && p.stepsize() <= 0)
        throw CaffeError("SolverParameter.stepsize must be positive for lr_policy step");
    if (p.iter_size() < 1) throw CaffeError("SolverParameter.iter_size must be at least 1");
    if (p.average_loss() < 1) throw CaffeError("average_loss should be non-negative.");          // solver.cpp:208 CHECK_GE(.., 1)
}

// The reference's types (sgd_solver.cpp:27-63 with <math.h> in scope through mkl_alternate.hpp, so std::pow / std::exp are
// visible unqualified): pow(float, int) promotes to double and is narrowed to Dtype; pow(float, float) and exp(float) are the
// float functions, and everything around them is float arithmetic.
float Solver::LearningRate(const SolverParameter& p, int iter, int* current_step) {
    const std::string& policy = p.lr_policy();
    const float base_lr = p.base_lr(), gamma = p.gamma(), power = p.power();
    if (policy == "fixed") return base_lr;
    if (policy == "step") {
        *current_step = iter / p.stepsize();
        return (float)(base_lr * std::pow((double)gamma, (double)*current_step));
    }
    if (policy == "exp") return (float)(base_lr * std::pow((double)gamma, (double)iter));
    if (policy == "inv") {
        const float x = 1.f + gamma * (float)iter;
        return base_lr * std::pow(x, -power);
    }
    if (policy == "multistep") {
        if (*current_step < p.stepvalue_size() && iter >= p.stepvalue(*current_step)) ++*current_step;
        return (float)(base_lr * std::pow((double)gamma, (double)*current_step));
    }
    if (policy == "poly") {
        const float x = 1.f - (float)iter / (float)p.max_iter();
        return base_lr * std::pow(x, power);
    }
    if (policy == "sigmoid") {
        const float arg = -gamma * ((float)iter - (float)p.stepsize());
        return base_lr * (1.f / (1.f + std::exp(arg)));
    }
    throw CaffeError("Unknown learning rate policy: " + policy);
}

Solver::Solver(const SolverParameter& param, Net<float>* net) : param_(param), net_(net) {
    Validate(param_);
    adam_ = param_.type() == "Adam";
    params_ = net_->LearnableParams();
    vector<fn2::SolverChunk> chunks;
    for (size_t id = 0; id < params_.size(); id++) {
        const auto& lp = params_[id];
        // lr_mult == 0: the reference's update cannot change the data, so the blob is skipped (and keeps a zero history,
        // DESIGN.md section 4)
        if (lp.lr_mult == 0.f || lp.count == 0) continue;
        const int seg = (int)segs_.size();
        segs_.push_back({(long long)lp.offset, (long long)hist_floats_, (long long)lp.count, lp.lr_mult,
                         param_.weight_decay() * lp.decay_mult});
        trainable_.push_back((int)id);
        hist_floats_ += slot(lp.count);
        const long long groups = ((long long)lp.count + 3) / 4;
        for (long long g = 0; g < groups; g += fn2::kChunkGroups) chunks.push_back({seg, (int)g});
    }
    nchunks_ = (int)chunks.size();
    if (nchunks_ == 0) return;
    cudaStream_t st = net_->stream();
    segs_dev_.reserve(segs_.size() * sizeof(fn2::SolverSegment));
    chunks_dev_.reserve(chunks.size() * sizeof(fn2::SolverChunk));
    CUDA_CHECK(cudaMemcpy(segs_dev_.get(), segs_.data(), segs_.size() * sizeof(fn2::SolverSegment), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(chunks_dev_.get(), chunks.data(), chunks.size() * sizeof(fn2::SolverChunk), cudaMemcpyHostToDevice));
    hist0_.reserve(hist_floats_ * sizeof(float), st);
    if (adam_) hist1_.reserve(hist_floats_ * sizeof(float), st);
    if (param_.clip_gradients() >= 0) {
        partial_.reserve((size_t)nchunks_ * sizeof(double));
        scale_.reserve(sizeof(float));
    }
}

void Solver::ApplyUpdate() {
    const float rate = LearningRate(param_, iter_, &current_step_);
    if (nchunks_ > 0) {
        void* data; void* diff;
        size_t bytes;
        net_->ParamArena(&data, &bytes);
        net_->ParamDiffArena(&diff, &bytes);
        cudaStream_t st = net_->stream();
        fn2::SolverUpdateArgs a;
        memset(&a, 0, sizeof(a));
        a.data = (float*)data; a.diff = (float*)diff;
        a.hist0 = hist0_.as<float>(); a.hist1 = hist1_.as<float>();
        a.segs = segs_dev_.as<fn2::SolverSegment>(); a.chunks = chunks_dev_.as<fn2::SolverChunk>();
        if (param_.clip_gradients() >= 0) {
            FN2_CALL(fn2::solver_clip_scale(a.diff, a.segs, a.chunks, nchunks_, partial_.as<double>(), param_.clip_gradients(),
                                            scale_.as<float>(), st));
            a.clip_scale = scale_.as<float>();
        }
        a.rate = rate;
        a.momentum = param_.momentum();
        a.momentum2 = param_.momentum2();
        a.delta = param_.delta();
        if (adam_) {                                                           // adam_solver.cpp:39-41
            const int t = iter_ + 1;
            a.correction = (float)(std::sqrt(1.0 - std::pow((double)a.momentum2, (double)t)) /
                                   (1.0 - std::pow((double)a.momentum, (double)t)));
        }
        a.normalize = param_.iter_size() != 1;
        a.accum_normalization = 1.f / (float)param_.iter_size();
        a.l1 = param_.regularization_type() == "L1";
        FN2_CALL(fn2::solver_update(a, nchunks_, adam_, st));
        net_->ParamsUpdated(trainable_);
    }
    ++iter_;
}

std::string Solver::State(const std::string& learned_net) {
    net_->Sync();
    vector<float> h0(hist_floats_), h1(adam_ ? hist_floats_ : 0);
    if (hist_floats_) {
        CUDA_CHECK(cudaMemcpy(h0.data(), hist0_.get(), hist_floats_ * sizeof(float), cudaMemcpyDeviceToHost));
        if (adam_) CUDA_CHECK(cudaMemcpy(h1.data(), hist1_.get(), hist_floats_ * sizeof(float), cudaMemcpyDeviceToHost));
    }
    SolverStateData s;
    s.iter = iter_;
    s.current_step = current_step_;
    s.learned_net = learned_net;
    for (int which = 0; which < (adam_ ? 2 : 1); which++) {
        const vector<float>& h = which ? h1 : h0;
        size_t k = 0;
        for (size_t id = 0; id < params_.size(); id++) {
            BlobProtoData b;
            b.shape = params_[id].shape;
            b.data.assign((size_t)params_[id].count, 0.f);
            if (k < trainable_.size() && trainable_[k] == (int)id) {
                memcpy(b.data.data(), h.data() + segs_[k].hist_offset, (size_t)params_[id].count * sizeof(float));
                k++;
            }
            s.history.push_back(std::move(b));
        }
    }
    return SerializeSolverState(s);
}

void Solver::Restore(const void* bytes, size_t n) {
    SolverStateData s = ParseSolverState(bytes, n);
    const size_t want = params_.size() * (adam_ ? 2 : 1);
    CHECK_EQ(s.history.size(), want) << "Incorrect length of history blobs.";              // sgd_solver.cpp:316-317
    for (size_t i = 0; i < want; i++) {
        const auto& lp = params_[i % params_.size()];
        CHECK_EQ(s.history[i].data.size(), (size_t)lp.count) << "history blob " << i << " does not match the size of parameter "
                                                             << net_->layer_names()[lp.layer] << "[" << lp.index << "]";
    }
    net_->Sync();
    for (int which = 0; which < (adam_ ? 2 : 1); which++)
        for (size_t k = 0; k < trainable_.size(); k++) {
            const BlobProtoData& b = s.history[which * params_.size() + trainable_[k]];
            float* dst = (which ? hist1_ : hist0_).as<float>() + segs_[k].hist_offset;
            CUDA_CHECK(cudaMemcpy(dst, b.data.data(), b.data.size() * sizeof(float), cudaMemcpyHostToDevice));
        }
    iter_ = s.iter;
    current_step_ = s.current_step;
}

}  // namespace caffe
