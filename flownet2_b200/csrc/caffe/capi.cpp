// extern "C" net-level entry points of include/fn2.h, fn2_frames.h, fn2_flow.h and fn2_lpq.h over caffe::Net<float>, and the solver's of
// include/fn2_solver.h over caffe::Solver.
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "../../../include/fn2_eval.h"
#include "../../../include/fn2_flow.h"
#include "../../../include/fn2_frames.h"
#include "../../../include/fn2_lpq.h"
#include "../../../include/fn2_solver.h"
#include "net.hpp"
#include "hdf5_min.hpp"
#include "solver.hpp"

namespace fn2 { void set_error(const char* fmt, ...); }

struct fn2_net {
    std::unique_ptr<caffe::Net<float> > net;
    std::vector<std::string> input_names, output_names;
    std::string caffemodel_cache;
};

#define FN2_TRY try {
#define FN2_CATCH                                                        \
    } catch (const caffe::ParseError& e) {                               \
        fn2::set_error("%s", e.what());                                  \
        return FN2_ERR_PARSE;                                            \
    } catch (const std::exception& e) {                                  \
        fn2::set_error("%s", e.what());                                  \
        return strstr(e.what(), "Unknown") ? FN2_ERR_NOTFOUND : FN2_ERR_INVALID; \
    }

// A status-returning net entry point: FN2_ERR_INVALID if an argument is null, else f() (FN2_OK if it returns nothing) with
// its exceptions mapped to a status, so none crosses the extern "C" boundary.
template <class F>
static int net_call(const char* what, bool args_ok, F&& f) {
    if (!args_ok) { fn2::set_error("%s: null argument", what); return FN2_ERR_INVALID; }
    FN2_TRY
        if constexpr (std::is_void<decltype(f())>::value) { f(); return FN2_OK; }
        else return f();
    FN2_CATCH
}

// The size-query convention: out == NULL reports the size in *bytes; otherwise out receives the output if *bytes holds it.
// A text output includes its terminating NUL.
static int emit(const char* what, const std::string& s, bool text, void* out, size_t* bytes) {
    if (!bytes) { fn2::set_error("%s: null size pointer", what); return FN2_ERR_INVALID; }
    const size_t n = s.size() + (text ? 1 : 0);
    if (!out) { *bytes = n; return FN2_OK; }
    if (*bytes < n) { fn2::set_error("%s: buffer too small", what); return FN2_ERR_INVALID; }
    memcpy(out, s.c_str(), n);
    *bytes = n;
    return FN2_OK;
}

namespace caffe { void SampleAugmentationCoeffs(const LayerParameter& lp, uint32_t seed, int num, int width, int height, float num_iter, float* out); }

extern "C" {

int fn2_net_create(const char* prototxt_text, int phase, fn2_net** out) {
    return fn2_net_create_batch(prototxt_text, phase, 0, out);
}

int fn2_net_create_batch(const char* prototxt_text, int phase, int batch, fn2_net** out) {
    return net_call("net_create", prototxt_text && out, [&] {
        *out = nullptr;
        caffe::NetParameter np = caffe::NetParameter::FromText(prototxt_text);
        if (batch > 0) {
            for (auto& lp : np.layers) {
                if (lp.type() != "Input") continue;
                caffe::Message* ip = lp.m->mutable_msg("input_param");
                for (auto& f : ip->fields)
                    if (f.name == "shape" && f.is_msg)
                        for (auto& d : f.msg->fields)
                            if (d.name == "dim") { d.scalar = std::to_string(batch); break; }
            }
        }
        std::unique_ptr<fn2_net> h(new fn2_net());
        h->net.reset(new caffe::Net<float>(np, phase == 0 ? caffe::TRAIN : caffe::TEST));
        for (int i : h->net->input_blob_indices()) h->input_names.push_back(h->net->blob_names()[i]);
        for (int i : h->net->output_blob_indices()) h->output_names.push_back(h->net->blob_names()[i]);
        *out = h.release();
    });
}

void fn2_net_destroy(fn2_net* net) { delete net; }

int fn2_net_copy_trained_layers(fn2_net* net, const void* caffemodel, size_t bytes) {
    return net_call("copy_trained_layers", net && caffemodel, [&] { net->net->CopyTrainedLayersFrom(caffemodel, bytes); });
}

int fn2_net_copy_trained_layers_prefixed(fn2_net* net, const void* caffemodel, size_t bytes, const char* prefix) {
    return net_call("copy_trained_layers_prefixed", net && caffemodel && prefix,
                    [&] { net->net->CopyTrainedLayersFrom(caffemodel, bytes, prefix); });
}

int fn2_net_param_layers(fn2_net* net, char* out, size_t* bytes) {
    return net_call("param_layers", net && bytes, [&] {
        caffe::Net<float>& n = *net->net;
        std::string text;
        for (size_t i = 0; i < n.layers().size(); i++) {
            caffe::Layer<float>& l = *n.layers()[i];
            if (l.blobs().empty()) continue;
            std::string shapes, mults;
            for (size_t j = 0; j < l.blobs().size(); j++) {
                if (j) { shapes += ","; mults += ","; }
                const std::vector<int>& s = l.blobs()[j]->shape();
                for (size_t k = 0; k < s.size(); k++) shapes += (k ? "x" : "") + std::to_string(s[k]);
                char m[32];
                snprintf(m, sizeof(m), "%g", n.lr_mult((int)i, (int)j));
                mults += m;
            }
            const char* flags = l.DoesUseCustomCopyBlobs() ? "c" : l.TemplateDefinedParams() ? "t" : "-";
            text += n.layer_names()[i] + "\t" + l.type() + "\t" + flags + "\t" + shapes + "\t" + mults + "\n";
        }
        return emit("param_layers", text, true, out, bytes);
    });
}

int fn2_net_to_caffemodel(fn2_net* net, void* buf, size_t* bytes) {
    return net_call("to_caffemodel", net && bytes, [&] {
        std::string& cache = net->caffemodel_cache;        // serialised once for the query and the fill call
        if (!buf || cache.empty()) cache = net->net->ToCaffemodel();
        const int rc = emit("to_caffemodel", cache, false, buf, bytes);
        if (buf && rc == FN2_OK) { cache.clear(); cache.shrink_to_fit(); }
        return rc;
    });
}

int fn2_net_fill_params(fn2_net* net, uint64_t seed) {
    return net_call("fill_params", net, [&] { net->net->FillParams(seed); });
}

int fn2_net_param_arena(fn2_net* net, void** dev_ptr, size_t* bytes) {
    return net_call("param_arena", net && dev_ptr && bytes, [&] { net->net->ParamArena(dev_ptr, bytes); });
}

int fn2_net_params_changed(fn2_net* net) {
    // the caller wrote the DEVICE arena: host caches of every param blob are stale
    return net_call("params_changed", net, [&] { net->net->ArenaWritten(); });
}

int fn2_net_num_inputs(fn2_net* net) { return net ? (int)net->input_names.size() : 0; }
const char* fn2_net_input_name(fn2_net* net, int i) {
    return (net && i >= 0 && i < (int)net->input_names.size()) ? net->input_names[i].c_str() : nullptr;
}
int fn2_net_num_outputs(fn2_net* net) { return net ? (int)net->output_names.size() : 0; }
const char* fn2_net_output_name(fn2_net* net, int i) {
    return (net && i >= 0 && i < (int)net->output_names.size()) ? net->output_names[i].c_str() : nullptr;
}
int fn2_net_num_blobs(fn2_net* net) { return net ? (int)net->net->blob_names().size() : 0; }
const char* fn2_net_blob_name(fn2_net* net, int i) {
    return (net && i >= 0 && i < (int)net->net->blob_names().size()) ? net->net->blob_names()[i].c_str() : nullptr;
}
int fn2_net_num_layers(fn2_net* net) { return net ? (int)net->net->layer_names().size() : 0; }
const char* fn2_net_layer_name(fn2_net* net, int i) {
    return (net && i >= 0 && i < (int)net->net->layer_names().size()) ? net->net->layer_names()[i].c_str() : nullptr;
}
const char* fn2_net_layer_type(fn2_net* net, int i) {
    return (net && i >= 0 && i < (int)net->net->layers().size()) ? net->net->layers()[i]->type() : nullptr;
}

int fn2_net_blob_shape(fn2_net* net, const char* blob, int shape[4]) {
    return net_call("blob_shape", net && blob && shape, [&] {
        auto b = net->net->blob_by_name(blob);
        for (int i = 0; i < 4; i++) shape[i] = b->shape(i);
    });
}

int fn2_net_set_input(fn2_net* net, const char* blob, const float* host_nchw) {
    return net_call("set_input", net && blob && host_nchw, [&] { net->net->SetInput(blob, host_nchw); });
}
int fn2_net_set_input_device(fn2_net* net, const char* blob, const float* dev_nchw) {
    return net_call("set_input_device", net && blob && dev_nchw, [&] { net->net->SetInputDevice(blob, dev_nchw); });
}
int fn2_net_get_blob(fn2_net* net, const char* blob, float* host_nchw) {
    return net_call("get_blob", net && blob && host_nchw, [&] { net->net->GetBlob(blob, host_nchw); });
}
int fn2_net_get_blob_device(fn2_net* net, const char* blob, float* dev_nchw) {
    return net_call("get_blob_device", net && blob && dev_nchw, [&] { net->net->GetBlobDevice(blob, dev_nchw); });
}

// ---- 8-bit frames in, NHWC out (include/fn2_frames.h) ----
int fn2_net_set_input_frames(fn2_net* net, const char* blob, const void* host_frames, int channels) {
    return net_call("set_input_frames", net && blob && host_frames, [&] { net->net->SetInputFrames(blob, host_frames, channels); });
}
int fn2_net_set_input_frames_device(fn2_net* net, const char* blob, const void* dev_frames, int channels) {
    return net_call("set_input_frames_device", net && blob && dev_frames,
                    [&] { net->net->SetInputFramesDevice(blob, dev_frames, channels); });
}
int fn2_net_set_input_flow_device(fn2_net* net, const char* blob, const void* dev, int format, int flags) {
    return net_call("set_input_flow_device", net && blob && dev, [&] { net->net->SetInputFlowDevice(blob, dev, format, flags); });
}
int fn2_net_get_blob_nhwc(fn2_net* net, const char* blob, float* host) {
    return net_call("get_blob_nhwc", net && blob && host, [&] { net->net->GetBlobNHWC(blob, host); });
}
int fn2_net_get_blob_nhwc_device(fn2_net* net, const char* blob, float* dev) {
    return net_call("get_blob_nhwc_device", net && blob && dev, [&] { net->net->GetBlobNHWCDevice(blob, dev); });
}

int fn2_net_forward(fn2_net* net) { return net_call("forward", net, [&] { net->net->Forward(); }); }
int fn2_net_backward(fn2_net* net) { return net_call("backward", net, [&] { net->net->Backward(); }); }
int fn2_net_clear_param_diffs(fn2_net* net) { return net_call("clear_param_diffs", net, [&] { net->net->ClearParamDiffs(); }); }
int fn2_net_set_diff(fn2_net* net, const char* blob, const float* host_nchw) {
    return net_call("set_diff", net && blob && host_nchw, [&] { net->net->SetDiff(blob, host_nchw); });
}
int fn2_net_get_diff(fn2_net* net, const char* blob, float* host_nchw) {
    return net_call("get_diff", net && blob && host_nchw, [&] { net->net->GetDiff(blob, host_nchw); });
}
int fn2_net_param_diff_arena(fn2_net* net, void** dev_ptr, size_t* bytes) {
    return net_call("param_diff_arena", net && dev_ptr && bytes, [&] { net->net->ParamDiffArena(dev_ptr, bytes); });
}
int fn2_net_trainable_diff_span(fn2_net* net, void** dev_ptr, size_t* bytes) {
    return net_call("trainable_diff_span", net && dev_ptr && bytes, [&] { net->net->TrainableDiffSpan(dev_ptr, bytes); });
}
static caffe::Blob<float>* find_param(fn2_net* net, const char* layer, int index) {
    const auto& names = net->net->layer_names();
    for (size_t i = 0; i < names.size(); i++)
        if (names[i] == layer) {
            auto& bl = net->net->layers()[i]->blobs();
            if (index < 0 || index >= (int)bl.size()) return nullptr;
            return bl[index].get();
        }
    return nullptr;
}
int fn2_net_param_shape(fn2_net* net, const char* layer, int index, int shape[4]) {
    return net_call("param_shape", net && layer && shape, [&] {
        caffe::Blob<float>* b = find_param(net, layer, index);
        if (!b) { fn2::set_error("param_shape: no parameter blob %s[%d]", layer, index); return FN2_ERR_INVALID; }
        for (int i = 0; i < 4; i++) shape[i] = b->shape(i);
        return FN2_OK;
    });
}
int fn2_net_get_param(fn2_net* net, const char* layer, int index, int diff, float* host) {
    return net_call("get_param", net && layer && host, [&] {
        caffe::Blob<float>* b = find_param(net, layer, index);
        if (!b) { fn2::set_error("get_param: no parameter blob %s[%d]", layer, index); return FN2_ERR_INVALID; }
        caffe::Caffe::stream() = net->net->stream();
        net->net->Sync();
        if (diff) { void* a; size_t n; net->net->ParamDiffArena(&a, &n); }
        const float* p = diff ? b->cpu_diff() : b->cpu_data();
        memcpy(host, p, (size_t)b->count() * sizeof(float));
        return FN2_OK;
    });
}
int fn2_net_launches_per_backward(fn2_net* net) { return net ? net->net->launches_per_backward() : 0; }
int fn2_net_layer_need_backward(fn2_net* net, int layer) {
    if (!net || layer < 0 || layer >= (int)net->net->layers().size()) return -1;
    FN2_TRY
        return net->net->layer_need_backward()[layer] ? 1 : 0;
    } catch (...) { return -1; }
}

int fn2_net_set_iter(fn2_net* net, int iter) {
    return net_call("set_iter", net && iter >= 0, [&] { net->net->set_iter(iter); });
}
int fn2_net_iter(fn2_net* net, int* iter) { return net_call("iter", net && iter, [&] { *iter = net->net->iter(); }); }
int fn2_net_sync(fn2_net* net) { return net_call("sync", net, [&] { net->net->Sync(); }); }
void* fn2_net_stream(fn2_net* net) { return net ? (void*)net->net->stream() : nullptr; }

int fn2_net_time_layers(fn2_net* net, float* ms) {
    return net_call("time_layers", net && ms, [&] { net->net->TimeLayers(ms); });
}
int fn2_net_launches_per_forward(fn2_net* net) { return net ? net->net->launches_per_forward() : 0; }
int fn2_net_graph_active(fn2_net* net) { return net && net->net->graph_active() ? 1 : 0; }

int fn2_net_layer_work(fn2_net* net, int layer, double* flops, double* bytes) {
    return net_call("layer_work", net && flops && bytes, [&] {
        if (layer < 0 || layer >= (int)net->net->layers().size()) { fn2::set_error("layer_work: bad argument"); return FN2_ERR_INVALID; }
        net->net->LayerWork(layer, flops, bytes);
        return FN2_OK;
    });
}

int fn2_proto_canonical(const char* prototxt_text, char* out, size_t* bytes) {
    if (!prototxt_text) { fn2::set_error("proto_canonical: null text"); return FN2_ERR_INVALID; }
    FN2_TRY
        caffe::NetParameter np = caffe::NetParameter::FromText(prototxt_text);
        std::string s;
        if (!np.name.empty()) s += "name: \"" + np.name + "\"\n";
        for (const auto& l : np.layers) s += "layer {\n" + caffe::PrintTextFormat(*l.m, 1) + "}\n";
        return emit("proto_canonical", s, true, out, bytes);
    FN2_CATCH
}

int fn2_aug_sample(const char* layer_prototxt, unsigned int seed, int num, int width, int height, float num_iter, float* coeffs_out) {
    if (!layer_prototxt || !coeffs_out || num <= 0) { fn2::set_error("aug_sample: invalid argument"); return FN2_ERR_INVALID; }
    FN2_TRY
        caffe::NetParameter np = caffe::NetParameter::FromText(layer_prototxt);
        const caffe::LayerParameter* lp = nullptr;
        for (const auto& l : np.layers) if (l.type() == "DataAugmentation") { lp = &l; break; }
        if (!lp) { fn2::set_error("aug_sample: no DataAugmentation layer in the text"); return FN2_ERR_INVALID; }
        caffe::SampleAugmentationCoeffs(*lp, seed, num, width, height, num_iter, coeffs_out);
        return FN2_OK;
    FN2_CATCH
}

static std::string caffemodel_to_h5(const void* caffemodel, size_t n) {
    std::vector<caffe::LayerBlobs> ls = caffe::ParseCaffemodel(caffemodel, n);
    std::vector<std::pair<std::string, std::vector<caffe::H5Blob> > > layers;
    for (const auto& l : ls) {
        if (l.blobs.empty()) continue;
        std::vector<caffe::H5Blob> bl;
        for (const auto& b : l.blobs) { caffe::H5Blob hb; hb.dims = b.shape; hb.data = b.data; bl.push_back(std::move(hb)); }
        layers.push_back({l.name, std::move(bl)});
    }
    return caffe::WriteCaffemodelH5(layers);
}

int fn2_caffemodel_to_hdf5(const void* caffemodel, size_t n, void* out, size_t* bytes) {
    if (!caffemodel || !bytes) { fn2::set_error("caffemodel_to_hdf5: null argument"); return FN2_ERR_INVALID; }
    try {
        return emit("caffemodel_to_hdf5", caffemodel_to_h5(caffemodel, n), false, out, bytes);
    } catch (const std::exception& e) {
        fn2::set_error("%s", e.what());
        return FN2_ERR_PARSE;
    }
}

int fn2_net_to_hdf5(fn2_net* net, void* buf, size_t* bytes) {
    return net_call("to_hdf5", net && bytes, [&] {
        const std::string cm = net->net->ToCaffemodel();
        return emit("to_hdf5", caffemodel_to_h5(cm.data(), cm.size()), false, buf, bytes);
    });
}

int fn2_hdf5_summary(const void* h5, size_t n, char* out, size_t* bytes) {
    if (!h5) { fn2::set_error("hdf5_summary: null data"); return FN2_ERR_INVALID; }
    try {
        caffe::H5File f(h5, n);
        std::string s;
        char buf[128];
        for (const auto& kv : f.datasets()) {
            s += kv.first + " f" + std::to_string(kv.second.elem_size * 8) + " [";
            for (size_t i = 0; i < kv.second.dims.size(); i++) { snprintf(buf, sizeof(buf), i ? ",%d" : "%d", kv.second.dims[i]); s += buf; }
            std::vector<float> v = f.read(kv.first);
            double sum = 0;
            for (float x : v) sum += (double)x;
            snprintf(buf, sizeof(buf), "] n=%zu sum=%.9g first=%.9g last=%.9g", v.size(), sum, v.empty() ? 0.0 : (double)v.front(), v.empty() ? 0.0 : (double)v.back());
            s += buf;
            s += "\n";
        }
        return emit("hdf5_summary", s, true, out, bytes);
    } catch (const std::exception& e) {
        fn2::set_error("%s", e.what());
        return FN2_ERR_PARSE;
    }
}

int fn2_caffemodel_summary(const void* caffemodel, size_t n, char* out, size_t* bytes) {
    if (!caffemodel) { fn2::set_error("caffemodel_summary: null data"); return FN2_ERR_INVALID; }
    FN2_TRY
        std::vector<caffe::LayerBlobs> ls = caffe::ParseCaffemodel(caffemodel, n);
        std::string s;
        char buf[128];
        for (const auto& l : ls) {
            s += l.name + " " + l.type;
            for (const auto& b : l.blobs) {
                s += " [";
                for (size_t i = 0; i < b.shape.size(); i++) { snprintf(buf, sizeof(buf), i ? ",%d" : "%d", b.shape[i]); s += buf; }
                double sum = 0;
                for (float v : b.data) sum += (double)v;
                snprintf(buf, sizeof(buf), "] n=%zu sum=%.9g", b.data.size(), sum);
                s += buf;
            }
            s += "\n";
        }
        return emit("caffemodel_summary", s, true, out, bytes);
    FN2_CATCH
}

// ---- solver (include/fn2_solver.h) ----
struct fn2_solver {
    fn2_net* net;
    std::unique_ptr<caffe::Solver> solver;
};

int fn2_solver_create(const char* solver_text, fn2_net* net, fn2_solver** out) {
    return net_call("solver_create", solver_text && net && out, [&] {
        *out = nullptr;
        std::unique_ptr<fn2_solver> h(new fn2_solver());
        h->net = net;
        h->solver.reset(new caffe::Solver(caffe::SolverParameter::FromText(solver_text), net->net.get()));
        *out = h.release();
    });
}

void fn2_solver_destroy(fn2_solver* solver) { delete solver; }

int fn2_solver_apply_update(fn2_solver* solver) {
    return net_call("solver_apply_update", solver, [&] { solver->solver->ApplyUpdate(); });
}

int fn2_solver_iter(fn2_solver* solver, int* iter, int* current_step) {
    return net_call("solver_iter", solver && iter && current_step, [&] {
        *iter = solver->solver->iter();
        *current_step = solver->solver->current_step();
    });
}

int fn2_solver_output_loss_weights(fn2_solver* solver, float* weights, int n) {
    return net_call("solver_output_loss_weights", solver && weights, [&] {
        const auto& outs = solver->net->net->output_blob_indices();
        if (n != (int)outs.size()) { fn2::set_error("solver_output_loss_weights: the net has %d outputs", (int)outs.size()); return FN2_ERR_INVALID; }
        for (int i = 0; i < n; i++) weights[i] = solver->net->net->blob_loss_weight(outs[i]);
        return FN2_OK;
    });
}

int fn2_solver_state(fn2_solver* solver, const char* learned_net, void* out, size_t* bytes) {
    return net_call("solver_state", solver && learned_net && bytes, [&] {
        return emit("solver_state", solver->solver->State(learned_net), false, out, bytes);
    });
}

int fn2_solver_restore(fn2_solver* solver, const void* state, size_t bytes) {
    return net_call("solver_restore", solver && state, [&] { solver->solver->Restore(state, bytes); });
}

int fn2_solverstate_learned_net(const void* state, size_t n, char* out, size_t* bytes) {
    if (!state) { fn2::set_error("solverstate_learned_net: null state"); return FN2_ERR_INVALID; }
    FN2_TRY
        return emit("solverstate_learned_net", caffe::ParseSolverState(state, n).learned_net, true, out, bytes);
    FN2_CATCH
}

int fn2_solver_learning_rate(const char* solver_text, int iter, int* current_step, float* rate) {
    return net_call("solver_learning_rate", solver_text && current_step && rate, [&] {
        const caffe::SolverParameter p = caffe::SolverParameter::FromText(solver_text);
        caffe::Solver::Validate(p);
        *rate = caffe::Solver::LearningRate(p, iter, current_step);
    });
}

int fn2_solver_params(const char* solver_text, char* out, size_t* bytes) {
    if (!solver_text) { fn2::set_error("solver_params: null text"); return FN2_ERR_INVALID; }
    FN2_TRY
        return emit("solver_params", caffe::SolverParameter::FromText(solver_text).Resolved(), true, out, bytes);
    FN2_CATCH
}

}  // extern "C"
