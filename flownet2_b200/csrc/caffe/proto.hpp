// Minimal protobuf support for the Caffe schema subset the FlowNet2 forward path uses
// (reference: src/caffe/proto/caffe.proto).  No libprotobuf: a generic text-format parser
// (the prototxt side, util/io.cpp:34-43 ReadProtoFromTextFile) into a field tree, thin typed
// accessors with the .proto's defaults, and a wire-format reader/writer for the
// NetParameter / LayerParameter / BlobProto part of a .caffemodel (util/io.cpp:53-65).
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace caffe {

struct ParseError : std::runtime_error {
    explicit ParseError(const std::string& m) : std::runtime_error(m) {}
};

struct Message;
struct Field {
    std::string name;
    bool is_msg = false;
    std::string scalar;                // token text (strings unescaped, enums by name)
    std::shared_ptr<Message> msg;
};

// Generic field tree.  Accessors never throw for absent optional fields: they return the default.
struct Message {
    std::vector<Field> fields;

    int count(const std::string& name) const;
    bool has(const std::string& name) const { return count(name) > 0; }
    const std::string& str(const std::string& name, int idx = 0) const;        // "" if absent
    std::string str_or(const std::string& name, const std::string& def) const;
    double num(const std::string& name, double def, int idx = 0) const;
    float f(const std::string& name, float def, int idx = 0) const { return (float)num(name, def, idx); }
    int i(const std::string& name, int def, int idx = 0) const { return (int)num(name, def, idx); }
    bool b(const std::string& name, bool def) const;
    const Message& msg(const std::string& name, int idx = 0) const;             // empty if absent
    Message* mutable_msg(const std::string& name);                              // creates if absent
    void set(const std::string& name, const std::string& value);                // replace or add
    void add(const std::string& name, const std::string& value);
    static const Message& empty();
};

// Text format -> tree.  Throws ParseError with line information.
Message ParseTextFormat(const std::string& text);
// Tree -> text (debugging / round-trip tests).
std::string PrintTextFormat(const Message& m, int indent = 0);

// ---- typed views (names and defaults from caffe.proto; line numbers in comments) ----------
struct FillerParameter {                       // caffe.proto:43-65
    const Message* m;
    std::string type() const { return m->str_or("type", "constant"); }
    float value() const { return m->f("value", 0); }
    float min() const { return m->f("min", 0); }
    float max() const { return m->f("max", 1); }
    float mean() const { return m->f("mean", 0); }
    float std() const { return m->f("std", 1); }
    std::string variance_norm() const { return m->str_or("variance_norm", "FAN_IN"); }
    int diag_val_size() const { return m->count("diag_val"); }
    float diag_val(int i) const { return m->f("diag_val", 1, i); }
};

struct ConvolutionParameter {                  // caffe.proto:847-898
    const Message* m;
    int num_output() const { return m->i("num_output", 0); }
    bool bias_term() const { return m->b("bias_term", true); }
    int group() const { return m->i("group", 1); }
    // resolves the repeated / _h,_w spellings like BaseConvolutionLayer::LayerSetUp
    // (base_conv_layer.cpp:28-103); returns {h, w}
    void kernel(int* h, int* w) const;
    void stride(int* h, int* w) const;
    void pad(int* h, int* w) const;
    void dilation(int* h, int* w) const;
    FillerParameter weight_filler() const { return FillerParameter{&m->msg("weight_filler")}; }
    FillerParameter bias_filler() const { return FillerParameter{&m->msg("bias_filler")}; }
    std::string engine() const { return m->str_or("engine", "DEFAULT"); }   // DEFAULT / CAFFE / CUDNN
};

struct CorrelationParameter {                  // caffe.proto:628-644
    const Message* m;
    int pad() const { return m->i("pad", 0); }
    bool has_kernel_size() const { return m->has("kernel_size"); }
    int kernel_size() const { return m->i("kernel_size", 0); }
    bool has_max_displacement() const { return m->has("max_displacement"); }
    int max_displacement() const { return m->i("max_displacement", 0); }
    int stride_1() const { return m->i("stride_1", 1); }
    int stride_2() const { return m->i("stride_2", 1); }
    bool do_abs() const { return m->b("do_abs", false); }
    int single_direction() const { return m->i("single_direction", 0); }   // Correlation1D: -1 left, 0 both, +1 right
    int correlation_type() const;              // 0 MULTIPLY, 1 SUBTRACT
};

struct FlowWarpParameter {                     // caffe.proto:553-560
    const Message* m;
    bool fill_nan() const;                     // fill_value == NOT_A_NUMBER
};

struct ResampleParameter {                     // caffe.proto:665-677
    const Message* m;
    bool antialias() const { return m->b("antialias", true); }
    bool has_width() const { return m->has("width"); }
    bool has_height() const { return m->has("height"); }
    int width() const { return m->i("width", 0); }
    int height() const { return m->i("height", 0); }
    float factor() const { return m->f("factor", 1.0f); }
    int type() const;                          // 1 NEAREST 2 LINEAR 3 CUBIC 4 AREA
};

struct RandomGeneratorParameter {              // caffe.proto:607-616
    const Message* m;
    std::string rand_type() const { return m->str_or("rand_type", "uniform"); }
    bool exp() const { return m->b("exp", false); }
    float mean() const { return m->f("mean", 0.f); }
    float spread() const { return m->f("spread", 0.f); }
    float prob() const { return m->f("prob", 1.f); }
    bool apply_schedule() const { return m->b("apply_schedule", true); }
    bool discretize() const { return m->b("discretize", false); }
    float multiplier() const { return m->f("multiplier", 1.f); }
};

struct AugmentationParameter {                 // caffe.proto:489-546
    const Message* m;
    bool has_crop_width() const { return m->has("crop_width"); }
    bool has_crop_height() const { return m->has("crop_height"); }
    int crop_width() const { return m->i("crop_width", 0); }
    int crop_height() const { return m->i("crop_height", 0); }
    float max_multiplier() const { return m->f("max_multiplier", 255.f); }
    bool augment_during_test() const { return m->b("augment_during_test", false); }
    int recompute_mean() const { return m->i("recompute_mean", 0); }
    bool mean_per_pixel() const { return m->b("mean_per_pixel", true); }
    int mean_size() const { return m->count("mean"); }
    float mean(int i) const { return m->f("mean", 0, i); }
    // true if any RandomGeneratorParameter (spatial/chromatic/eigen/effect) is present
    bool has_any_generator() const;
    bool has(const char* generator) const { return m->has(generator); }
    RandomGeneratorParameter gen(const char* generator) const { return RandomGeneratorParameter{&m->msg(generator)}; }
    int chromatic_eigvec_size() const { return m->count("chromatic_eigvec"); }
    float chromatic_eigvec(int i) const { return m->f("chromatic_eigvec", 0, i); }
};

struct EltwiseParameter {                      // caffe.proto:1011-1023
    const Message* m;
    std::string operation() const { return m->str_or("operation", "SUM"); }
    int coeff_size() const { return m->count("coeff"); }
    float coeff(int i) const { return m->f("coeff", 1, i); }
};

struct LayerParameter {                        // caffe.proto:312-425
    std::shared_ptr<Message> m;
    LayerParameter() : m(std::make_shared<Message>()) {}
    explicit LayerParameter(std::shared_ptr<Message> mm) : m(std::move(mm)) {}
    const std::string& name() const { return m->str("name"); }
    const std::string& type() const { return m->str("type"); }
    int bottom_size() const { return m->count("bottom"); }
    int top_size() const { return m->count("top"); }
    const std::string& bottom(int i) const { return m->str("bottom", i); }
    const std::string& top(int i) const { return m->str("top", i); }
    bool reshape_every_iter() const { return m->b("reshape_every_iter", true); }   // caffe.proto:424
    ConvolutionParameter convolution_param() const { return ConvolutionParameter{&m->msg("convolution_param")}; }
    CorrelationParameter correlation_param() const { return CorrelationParameter{&m->msg("correlation_param")}; }
    FlowWarpParameter flow_warp_param() const { return FlowWarpParameter{&m->msg("flow_warp_param")}; }
    ResampleParameter resample_param() const { return ResampleParameter{&m->msg("resample_param")}; }
    AugmentationParameter augmentation_param() const { return AugmentationParameter{&m->msg("augmentation_param")}; }
    EltwiseParameter eltwise_param() const { return EltwiseParameter{&m->msg("eltwise_param")}; }
    float relu_negative_slope() const { return m->msg("relu_param").f("negative_slope", 0); }
    // CoeffScheduleParameter, caffe.proto:693-697
    float coeff_schedule_half_life() const { return m->msg("coeff_schedule_param").f("half_life", 1.f); }
    float coeff_schedule_initial() const { return m->msg("coeff_schedule_param").f("initial_coeff", 1.f); }
    float coeff_schedule_final() const { return m->msg("coeff_schedule_param").f("final_coeff", 1.f); }
    int concat_axis() const;                   // ConcatParameter axis / concat_dim (concat_layer.cpp:21-31)
    // phase rules (NetStateRule include/exclude, net.cpp:288-360): true if the layer is kept
    bool included_in_phase(int phase) const;
};

struct NetParameter {
    std::string name;
    bool force_backward = false;               // caffe.proto:88-91: gradients also for blobs no parameter depends on (inputs)
    std::vector<LayerParameter> layers;
    // Builds the layer list from a parsed prototxt, rewriting legacy `input:` +
    // `input_shape{}` / `input_dim:` into one Input layer placed first
    // (util/upgrade_proto.cpp:953-992).
    static NetParameter FromText(const std::string& prototxt);
};

// SolverParameter, caffe.proto:104-244, read from a solver prototxt.  FromText applies UpgradeSolverType
// (upgrade_proto.cpp:1002-1037: the deprecated solver_type enum becomes the type string) and nothing else; which values the
// engine's solver accepts is Solver's business (solver.cpp Validate).
struct SolverParameter {
    std::shared_ptr<Message> m;
    static SolverParameter FromText(const std::string& text);
    std::string type() const { return m->str_or("type", "SGD"); }
    float base_lr() const { return m->f("base_lr", 0); }
    std::string lr_policy() const { return m->str_or("lr_policy", ""); }
    float gamma() const { return m->f("gamma", 0); }
    float power() const { return m->f("power", 0); }
    int stepsize() const { return m->i("stepsize", 0); }
    int stepvalue_size() const { return m->count("stepvalue"); }
    int stepvalue(int i) const { return m->i("stepvalue", 0, i); }
    int max_iter() const { return m->i("max_iter", 0); }
    float momentum() const { return m->f("momentum", 0); }
    float momentum2() const { return m->f("momentum2", 0.999f); }
    float delta() const { return m->f("delta", 1e-8f); }
    float weight_decay() const { return m->f("weight_decay", 0); }
    std::string regularization_type() const { return m->str_or("regularization_type", "L2"); }
    float clip_gradients() const { return m->f("clip_gradients", -1); }
    int iter_size() const { return m->i("iter_size", 1); }
    int average_loss() const { return m->i("average_loss", 1); }
    int snapshot() const { return m->i("snapshot", 0); }
    std::string snapshot_prefix() const { return m->str_or("snapshot_prefix", ""); }
    bool snapshot_after_train() const { return m->b("snapshot_after_train", true); }
    // every field above as `name: value` lines in this order (the resolved view tests compare with caffe_pb2)
    std::string Resolved() const;
};

// ---- binary .caffemodel subset ------------------------------------------------------------
struct BlobProtoData {
    std::vector<int> shape;                    // from shape{dim} or legacy num/channels/height/width
    std::vector<float> data;                   // data (5) or double_data (8) narrowed
};
struct LayerBlobs {
    std::string name, type;
    std::vector<BlobProtoData> blobs;
};
// NetParameter.layer = 100 (and V1 `layers` = 2), LayerParameter.{name=1,type=2,blobs=7},
// BlobProto.{shape=7{dim=1}, data=5, double_data=8, num..width=1..4}   caffe.proto:10-22,94,313-331
std::vector<LayerBlobs> ParseCaffemodel(const void* bytes, size_t n);
std::string SerializeCaffemodel(const std::string& net_name, const std::vector<LayerBlobs>& layers);
// SolverState, caffe.proto:247-252: iter = 1, learned_net = 2, history = 3 (BlobProto), current_step = 4.  To and from bytes
// with the .caffemodel's BlobProto encoding (sgd_solver.cpp:260-322).
struct SolverStateData {
    int iter = 0;
    int current_step = 0;
    std::string learned_net;
    std::vector<BlobProtoData> history;
};
SolverStateData ParseSolverState(const void* bytes, size_t n);
std::string SerializeSolverState(const SolverStateData& s);

}  // namespace caffe
