#include "proto.hpp"

#include <map>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <sstream>

namespace caffe {

// ------------------------------------------------------------------------------------------
// Message accessors
// ------------------------------------------------------------------------------------------
const Message& Message::empty() {
    static const Message e;
    return e;
}
int Message::count(const std::string& name) const {
    int n = 0;
    for (const auto& f : fields) if (f.name == name) n++;
    return n;
}
static const Field* find_field(const Message& m, const std::string& name, int idx) {
    int n = 0;
    for (const auto& f : m.fields)
        if (f.name == name) {
            if (n == idx) return &f;
            n++;
        }
    return nullptr;
}
const std::string& Message::str(const std::string& name, int idx) const {
    static const std::string none;
    const Field* f = find_field(*this, name, idx);
    return (f && !f->is_msg) ? f->scalar : none;
}
std::string Message::str_or(const std::string& name, const std::string& def) const {
    const Field* f = find_field(*this, name, 0);
    return (f && !f->is_msg) ? f->scalar : def;
}
double Message::num(const std::string& name, double def, int idx) const {
    const Field* f = find_field(*this, name, idx);
    if (!f || f->is_msg) return def;
    const std::string& s = f->scalar;
    if (s == "inf" || s == "infinity") return INFINITY;
    if (s == "-inf" || s == "-infinity") return -INFINITY;
    if (s == "nan") return NAN;
    if (s == "true") return 1;
    if (s == "false") return 0;
    char* end = nullptr;
    double v;
    if (s.size() > 2 && s[0] == '0' && (s[1] == 'x' || s[1] == 'X')) v = (double)strtoll(s.c_str(), &end, 16);
    else v = strtod(s.c_str(), &end);
    // protobuf accepts a trailing 'f' on floats
    if (end && (*end == 'f' || *end == 'F')) end++;
    if (!end || *end != 0) throw ParseError("field '" + name + "': '" + s + "' is not a number");
    return v;
}
bool Message::b(const std::string& name, bool def) const {
    const Field* f = find_field(*this, name, 0);
    if (!f || f->is_msg) return def;
    const std::string& s = f->scalar;
    if (s == "true" || s == "True" || s == "t" || s == "1") return true;
    if (s == "false" || s == "False" || s == "f" || s == "0") return false;
    throw ParseError("field '" + name + "': '" + s + "' is not a bool");
}
const Message& Message::msg(const std::string& name, int idx) const {
    const Field* f = find_field(*this, name, idx);
    return (f && f->is_msg && f->msg) ? *f->msg : empty();
}
Message* Message::mutable_msg(const std::string& name) {
    for (auto& f : fields)
        if (f.name == name && f.is_msg) return f.msg.get();
    Field f;
    f.name = name; f.is_msg = true; f.msg = std::make_shared<Message>();
    fields.push_back(f);
    return fields.back().msg.get();
}
void Message::set(const std::string& name, const std::string& value) {
    for (auto& f : fields)
        if (f.name == name && !f.is_msg) { f.scalar = value; return; }
    add(name, value);
}
void Message::add(const std::string& name, const std::string& value) {
    Field f;
    f.name = name; f.scalar = value;
    fields.push_back(f);
}

// ------------------------------------------------------------------------------------------
// Text-format parser
// ------------------------------------------------------------------------------------------
namespace {
struct Lexer {
    const std::string& s;
    size_t pos = 0;
    int line = 1;
    explicit Lexer(const std::string& t) : s(t) {}

    [[noreturn]] void fail(const std::string& what) const {
        std::ostringstream o;
        o << "prototxt:" << line << ": " << what;
        throw ParseError(o.str());
    }
    void skip_ws() {
        while (pos < s.size()) {
            char c = s[pos];
            if (c == '\n') { line++; pos++; }
            else if (c == ' ' || c == '\t' || c == '\r') pos++;
            else if (c == '#') { while (pos < s.size() && s[pos] != '\n') pos++; }
            else break;
        }
    }
    bool eof() { skip_ws(); return pos >= s.size(); }
    char peek() { skip_ws(); return pos < s.size() ? s[pos] : 0; }
    bool accept(char c) { if (peek() == c) { pos++; return true; } return false; }
    static bool ident_char(char c) {
        return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_' || c == '.';
    }
    std::string ident() {
        skip_ws();
        size_t b = pos;
        if (pos < s.size() && s[pos] == '[') {           // extension name "[pkg.ext]" -- kept verbatim
            while (pos < s.size() && s[pos] != ']') pos++;
            if (pos < s.size()) pos++;
            return s.substr(b, pos - b);
        }
        while (pos < s.size() && ident_char(s[pos])) pos++;
        if (b == pos) fail(std::string("expected field name, got '") + (pos < s.size() ? s[pos] : '?') + "'");
        return s.substr(b, pos - b);
    }
    std::string quoted() {
        // one or more adjacent string literals are concatenated
        std::string out;
        while (true) {
            char q = peek();
            if (q != '"' && q != '\'') break;
            pos++;
            while (true) {
                if (pos >= s.size()) fail("unterminated string");
                char c = s[pos++];
                if (c == q) break;
                if (c == '\n') fail("newline in string");
                if (c == '\\') {
                    if (pos >= s.size()) fail("bad escape");
                    char e = s[pos++];
                    switch (e) {
                        case 'n': out += '\n'; break;
                        case 't': out += '\t'; break;
                        case 'r': out += '\r'; break;
                        case '\\': out += '\\'; break;
                        case '"': out += '"'; break;
                        case '\'': out += '\''; break;
                        case 'x': {
                            int v = 0, nd = 0;
                            while (pos < s.size() && nd < 2 && isxdigit((unsigned char)s[pos])) {
                                char h = s[pos++];
                                v = v * 16 + (h <= '9' ? h - '0' : (h | 32) - 'a' + 10);
                                nd++;
                            }
                            out += (char)v;
                            break;
                        }
                        default:
                            if (e >= '0' && e <= '7') {
                                int v = e - '0', nd = 1;
                                while (pos < s.size() && nd < 3 && s[pos] >= '0' && s[pos] <= '7') { v = v * 8 + (s[pos++] - '0'); nd++; }
                                out += (char)v;
                            } else out += e;
                    }
                } else out += c;
            }
        }
        return out;
    }
    std::string scalar() {
        char c = peek();
        if (c == '"' || c == '\'') return quoted();
        size_t b = pos;
        if (pos < s.size() && (s[pos] == '-' || s[pos] == '+')) pos++;
        while (pos < s.size() && (ident_char(s[pos]) || s[pos] == '+' || s[pos] == '-')) {
            // allow exponent signs only directly after e/E
            if ((s[pos] == '+' || s[pos] == '-') && !(pos > b && (s[pos - 1] == 'e' || s[pos - 1] == 'E'))) break;
            pos++;
        }
        if (b == pos) fail(std::string("expected a value, got '") + c + "'");
        return s.substr(b, pos - b);
    }
};

void parse_fields(Lexer& lx, Message& m, char closer) {
    while (true) {
        if (lx.eof()) {
            if (closer) lx.fail("unexpected end of input, missing closing brace");
            return;
        }
        char c = lx.peek();
        if (closer && c == closer) { lx.pos++; return; }
        if (c == '}' || c == '>') lx.fail("unbalanced closing brace");
        std::string name = lx.ident();
        bool colon = lx.accept(':');
        char n = lx.peek();
        if (n == '{' || n == '<') {
            lx.pos++;
            Field f;
            f.name = name; f.is_msg = true; f.msg = std::make_shared<Message>();
            parse_fields(lx, *f.msg, n == '{' ? '}' : '>');
            m.fields.push_back(std::move(f));
        } else {
            if (!colon) lx.fail("expected ':' or '{' after field '" + name + "'");
            if (lx.accept('[')) {
                if (!lx.accept(']')) {
                    while (true) {
                        char e = lx.peek();
                        if (e == '{' || e == '<') {
                            lx.pos++;
                            Field f;
                            f.name = name; f.is_msg = true; f.msg = std::make_shared<Message>();
                            parse_fields(lx, *f.msg, e == '{' ? '}' : '>');
                            m.fields.push_back(std::move(f));
                        } else {
                            m.add(name, lx.scalar());
                        }
                        if (lx.accept(']')) break;
                        if (!lx.accept(',')) lx.fail("expected ',' or ']' in list");
                    }
                }
            } else {
                m.add(name, lx.scalar());
            }
        }
        if (!lx.accept(',')) lx.accept(';');
    }
}
}  // namespace

Message ParseTextFormat(const std::string& text) {
    Lexer lx(text);
    Message m;
    parse_fields(lx, m, 0);
    return m;
}

std::string PrintTextFormat(const Message& m, int indent) {
    std::ostringstream o;
    std::string pad(indent * 2, ' ');
    for (const auto& f : m.fields) {
        if (f.is_msg) {
            o << pad << f.name << " {\n" << PrintTextFormat(*f.msg, indent + 1) << pad << "}\n";
        } else {
            bool bare = !f.scalar.empty();
            for (char c : f.scalar)
                if (!(Lexer::ident_char(c) || c == '-' || c == '+')) bare = false;
            // names that carry string values in caffe.proto are always quoted
            static const char* string_fields[] = {"name", "type", "bottom", "top", "input", "mode",
                                                  "write_augmented", "write_mean", "file", "folder",
                                                  "prefix", "suffix", "source", "mean_file", "rand_type"};
            for (const char* sf : string_fields) if (f.name == sf) bare = false;
            if (bare) o << pad << f.name << ": " << f.scalar << "\n";
            else {
                o << pad << f.name << ": \"";
                for (char c : f.scalar) {
                    if (c == '"' || c == '\\') o << '\\' << c;
                    else if (c == '\n') o << "\\n";
                    else o << c;
                }
                o << "\"\n";
            }
        }
    }
    return o.str();
}

// ------------------------------------------------------------------------------------------
// Typed views
// ------------------------------------------------------------------------------------------
static void resolve_hw(const Message& m, const char* rep, const char* h, const char* w, int def, int* oh, int* ow) {
    if (m.has(h) || m.has(w)) {
        if (m.count(rep)) throw ParseError(std::string("Either ") + rep + " or " + h + "/" + w + " should be specified; not both.");
        *oh = m.i(h, def); *ow = m.i(w, def);
        return;
    }
    int n = m.count(rep);
    if (n == 0) { *oh = *ow = def; }
    else if (n == 1) { *oh = *ow = m.i(rep, def, 0); }
    else { *oh = m.i(rep, def, 0); *ow = m.i(rep, def, 1); }
}
void ConvolutionParameter::kernel(int* h, int* w) const {
    resolve_hw(*m, "kernel_size", "kernel_h", "kernel_w", 0, h, w);
    if (*h <= 0 || *w <= 0) throw ParseError("Filter dimensions must be nonzero (base_conv_layer.cpp:53)");
}
void ConvolutionParameter::stride(int* h, int* w) const { resolve_hw(*m, "stride", "stride_h", "stride_w", 1, h, w); }
void ConvolutionParameter::pad(int* h, int* w) const { resolve_hw(*m, "pad", "pad_h", "pad_w", 0, h, w); }
void ConvolutionParameter::dilation(int* h, int* w) const {
    int n = m->count("dilation");
    if (n == 0) { *h = *w = 1; }
    else if (n == 1) { *h = *w = m->i("dilation", 1, 0); }
    else { *h = m->i("dilation", 1, 0); *w = m->i("dilation", 1, 1); }
}

int CorrelationParameter::correlation_type() const {
    std::string s = m->str_or("correlation_type", "MULTIPLY");
    if (s == "MULTIPLY" || s == "0") return 0;
    if (s == "SUBTRACT" || s == "1") return 1;
    throw ParseError("unknown correlation_type " + s);
}
bool FlowWarpParameter::fill_nan() const {
    std::string s = m->str_or("fill_value", "ZERO");
    if (s == "ZERO" || s == "1") return false;
    if (s == "NOT_A_NUMBER" || s == "2") return true;
    throw ParseError("unknown fill_value " + s);
}
int ResampleParameter::type() const {
    std::string s = m->str_or("type", "LINEAR");
    if (s == "NEAREST" || s == "1") return 1;
    if (s == "LINEAR" || s == "2") return 2;
    if (s == "CUBIC" || s == "3") return 3;
    if (s == "AREA" || s == "4") return 4;
    throw ParseError("unknown resample type " + s);
}
bool AugmentationParameter::has_any_generator() const {
    static const char* gens[] = {"mirror", "translate", "rotate", "zoom", "squeeze", "translate_x", "translate_y",
                                 "gamma", "brightness", "contrast", "color", "lmult_pow", "lmult_mult", "lmult_add",
                                 "sat_pow", "sat_mult", "sat_add", "col_pow", "col_mult", "col_add", "ladd_pow",
                                 "ladd_mult", "ladd_add", "col_rotate", "fog_amount", "fog_size",
                                 "motion_blur_angle", "motion_blur_size", "shadow_angle", "shadow_distance",
                                 "shadow_strength", "noise"};
    for (const char* g : gens) if (m->has(g)) return true;
    return false;
}
int LayerParameter::concat_axis() const {
    const Message& c = m->msg("concat_param");
    if (c.has("concat_dim")) return c.i("concat_dim", 1);
    return c.i("axis", 1);
}
bool LayerParameter::included_in_phase(int phase) const {
    // NetStateRule phase only (net.cpp:288-360 StateMeetsRule); stage/level rules are not used by
    // the FlowNet2 deploy nets.
    auto phase_of = [](const Message& rule, int def) {
        if (!rule.has("phase")) return def;
        std::string s = rule.str("phase");
        return (s == "TRAIN" || s == "0") ? 0 : 1;
    };
    int ninc = m->count("include"), nexc = m->count("exclude");
    if (ninc) {
        for (int i = 0; i < ninc; i++) if (phase_of(m->msg("include", i), phase) == phase) return true;
        return false;
    }
    for (int i = 0; i < nexc; i++) if (phase_of(m->msg("exclude", i), 1 - phase) == phase) return false;
    return true;
}

// UpgradeV1LayerParameter (util/upgrade_proto.cpp:680-862) + UpgradeV1LayerType (:864-949): a V1 `layers { type: CONVOLUTION
// blobs_lr: 1 weight_decay: 1 ... }` entry as a `layer { type: "Convolution" param { lr_mult: 1 decay_mult: 1 } ... }` message.
static std::shared_ptr<Message> UpgradeV1Layer(const Message& v1) {
    static const std::map<std::string, std::string> types = {
        {"NONE", ""}, {"ABSVAL", "AbsVal"}, {"ACCURACY", "Accuracy"}, {"ARGMAX", "ArgMax"}, {"BNLL", "BNLL"}, {"CONCAT", "Concat"},
        {"CONTRASTIVE_LOSS", "ContrastiveLoss"}, {"CONVOLUTION", "Convolution"}, {"DECONVOLUTION", "Deconvolution"}, {"DATA", "Data"},
        {"DROPOUT", "Dropout"}, {"DUMMY_DATA", "DummyData"}, {"EUCLIDEAN_LOSS", "EuclideanLoss"}, {"ELTWISE", "Eltwise"}, {"EXP", "Exp"},
        {"FLATTEN", "Flatten"}, {"HDF5_DATA", "HDF5Data"}, {"HDF5_OUTPUT", "HDF5Output"}, {"HINGE_LOSS", "HingeLoss"}, {"IM2COL", "Im2col"},
        {"IMAGE_DATA", "ImageData"}, {"INFOGAIN_LOSS", "InfogainLoss"}, {"INNER_PRODUCT", "InnerProduct"}, {"LRN", "LRN"},
        {"MEMORY_DATA", "MemoryData"}, {"MULTINOMIAL_LOGISTIC_LOSS", "MultinomialLogisticLoss"}, {"MVN", "MVN"}, {"POOLING", "Pooling"},
        {"POWER", "Power"}, {"RELU", "ReLU"}, {"SIGMOID", "Sigmoid"}, {"SIGMOID_CROSS_ENTROPY_LOSS", "SigmoidCrossEntropyLoss"},
        {"SILENCE", "Silence"}, {"SOFTMAX", "Softmax"}, {"SOFTMAX_LOSS", "SoftmaxWithLoss"}, {"SPLIT", "Split"}, {"SLICE", "Slice"},
        {"TANH", "TanH"}, {"WINDOW_DATA", "WindowData"}, {"THRESHOLD", "Threshold"}};
    auto out = std::make_shared<Message>();
    auto copy_all = [&](const char* name) { for (const auto& f : v1.fields) if (f.name == name) out->fields.push_back(f); };
    copy_all("bottom"); copy_all("top"); copy_all("name"); copy_all("include"); copy_all("exclude");
    if (v1.has("type")) {
        const std::string& t = v1.str("type");
        auto it = types.find(t);
        if (it == types.end()) throw ParseError("Unknown V1LayerParameter layer type: " + t);       // :946-947
        out->add("type", it->second);
    }
    copy_all("blobs");
    // param (shared-weight names), blob_share_mode, blobs_lr, weight_decay -> one ParamSpec per blob (:705-736)
    const int nparam = std::max(std::max(v1.count("param"), v1.count("blob_share_mode")), std::max(v1.count("blobs_lr"), v1.count("weight_decay")));
    for (int i = 0; i < nparam; i++) {
        Field f;
        f.name = "param"; f.is_msg = true; f.msg = std::make_shared<Message>();
        if (i < v1.count("param")) f.msg->add("name", v1.str("param", i));
        if (i < v1.count("blob_share_mode")) f.msg->add("share_mode", v1.str("blob_share_mode", i));
        if (i < v1.count("blobs_lr")) f.msg->add("lr_mult", v1.str("blobs_lr", i));
        if (i < v1.count("weight_decay")) f.msg->add("decay_mult", v1.str("weight_decay", i));
        out->fields.push_back(f);
    }
    copy_all("loss_weight");
    static const char* const subs[] = {"accuracy_param", "argmax_param", "concat_param", "contrastive_loss_param", "convolution_param",
        "data_param", "dropout_param", "dummy_data_param", "eltwise_param", "exp_param", "hdf5_data_param", "hdf5_output_param",
        "hinge_loss_param", "image_data_param", "infogain_loss_param", "inner_product_param", "lrn_param", "memory_data_param",
        "mvn_param", "pooling_param", "power_param", "relu_param", "sigmoid_param", "softmax_param", "slice_param", "tanh_param",
        "threshold_param", "window_data_param", "transform_param", "loss_param"};
    for (const char* n : subs) copy_all(n);
    if (v1.has("layer")) throw ParseError("Input NetParameter has V0 layer -- not supported (upgrade_proto.cpp:858-861 ignores it)");
    return out;
}

NetParameter NetParameter::FromText(const std::string& prototxt) {
    Message root = ParseTextFormat(prototxt);
    NetParameter np;
    np.name = root.str("name");
    np.force_backward = root.b("force_backward", false);
    const bool v1 = root.count("layers") > 0;                 // NetNeedsV1ToV2Upgrade, upgrade_proto.cpp:27-36
    if (v1 && root.count("layer"))
        throw ParseError("prototxt mixes V1 'layers' and 'layer' fields (upgrade_proto.cpp:655-660 refuses it too)");
    // legacy top-level inputs -> one Input layer named "input" placed first (upgrade_proto.cpp:953-992)
    int nin = root.count("input");
    if (nin) {
        auto lm = std::make_shared<Message>();
        lm->add("name", "input");
        lm->add("type", "Input");
        Message* ip = lm->mutable_msg("input_param");
        int nshape = root.count("input_shape"), ndim = root.count("input_dim");
        for (int i = 0; i < nin; i++) lm->add("top", root.str("input", i));
        if (nshape) {
            for (int i = 0; i < nshape; i++) {
                Field f;
                f.name = "shape"; f.is_msg = true;
                f.msg = std::make_shared<Message>(root.msg("input_shape", i));
                ip->fields.push_back(f);
            }
        } else if (ndim) {
            if (ndim % 4) throw ParseError("input_dim count must be a multiple of 4");
            for (int i = 0; i < ndim; i += 4) {
                Field f;
                f.name = "shape"; f.is_msg = true; f.msg = std::make_shared<Message>();
                for (int j = 0; j < 4; j++) f.msg->add("dim", root.str("input_dim", i + j));
                ip->fields.push_back(f);
            }
        }
        np.layers.emplace_back(lm);
    }
    for (const auto& f : root.fields) {
        if (f.name == "layer" && f.is_msg) np.layers.emplace_back(f.msg);
        if (f.name == "layers" && f.is_msg) np.layers.emplace_back(UpgradeV1Layer(*f.msg));
    }
    return np;
}

// ------------------------------------------------------------------------------------------
// Wire format
// ------------------------------------------------------------------------------------------
namespace {
struct Reader {
    const uint8_t* p;
    const uint8_t* end;
    bool ok() const { return p < end; }
    uint64_t varint() {
        uint64_t v = 0;
        int shift = 0;
        while (true) {
            if (p >= end) throw ParseError("caffemodel: truncated varint");
            uint8_t b = *p++;
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
            if (shift > 63) throw ParseError("caffemodel: varint too long");
        }
        return v;
    }
    Reader sub() {
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw ParseError("caffemodel: truncated length-delimited field");
        Reader r{p, p + n};
        p += n;
        return r;
    }
    void skip(int wt) {
        switch (wt) {
            case 0: varint(); break;
            case 1: if (end - p < 8) throw ParseError("caffemodel: truncated fixed64"); p += 8; break;
            case 2: sub(); break;
            case 5: if (end - p < 4) throw ParseError("caffemodel: truncated fixed32"); p += 4; break;
            default: throw ParseError("caffemodel: unsupported wire type");
        }
    }
};

BlobProtoData parse_blob(Reader r) {
    BlobProtoData b;
    int legacy[4] = {0, 0, 0, 0};
    bool has_legacy = false, has_shape = false;
    std::vector<double> dd;
    while (r.ok()) {
        uint64_t key = r.varint();
        int fn = (int)(key >> 3), wt = (int)(key & 7);
        if (fn >= 1 && fn <= 4 && wt == 0) { legacy[fn - 1] = (int)r.varint(); has_legacy = true; }
        else if (fn == 7 && wt == 2) {                       // BlobShape
            Reader s = r.sub();
            has_shape = true;
            while (s.ok()) {
                uint64_t k2 = s.varint();
                int f2 = (int)(k2 >> 3), w2 = (int)(k2 & 7);
                if (f2 == 1 && w2 == 2) { Reader d = s.sub(); while (d.ok()) b.shape.push_back((int)d.varint()); }
                else if (f2 == 1 && w2 == 0) b.shape.push_back((int)s.varint());
                else s.skip(w2);
            }
        } else if (fn == 5 && wt == 2) {                     // packed float data
            Reader d = r.sub();
            size_t n = (size_t)(d.end - d.p) / 4;
            size_t old = b.data.size();
            b.data.resize(old + n);
            memcpy(b.data.data() + old, d.p, n * 4);
        } else if (fn == 5 && wt == 5) {                     // unpacked float
            float v; memcpy(&v, r.p, 4); r.p += 4; b.data.push_back(v);
        } else if (fn == 8 && wt == 2) {                     // packed double_data
            Reader d = r.sub();
            size_t n = (size_t)(d.end - d.p) / 8;
            for (size_t i = 0; i < n; i++) { double v; memcpy(&v, d.p + 8 * i, 8); dd.push_back(v); }
        } else r.skip(wt);
    }
    if (b.data.empty() && !dd.empty()) for (double v : dd) b.data.push_back((float)v);   // blob.cpp:472-476
    if (!has_shape && has_legacy) b.shape.assign(legacy, legacy + 4);                     // blob.cpp:448-466
    return b;
}

LayerBlobs parse_layer(Reader r, bool v1) {
    LayerBlobs l;
    const int f_name = v1 ? 4 : 1, f_blobs = v1 ? 6 : 7;
    while (r.ok()) {
        uint64_t key = r.varint();
        int fn = (int)(key >> 3), wt = (int)(key & 7);
        if (fn == f_name && wt == 2) { Reader s = r.sub(); l.name.assign((const char*)s.p, s.end - s.p); }
        else if (!v1 && fn == 2 && wt == 2) { Reader s = r.sub(); l.type.assign((const char*)s.p, s.end - s.p); }
        else if (fn == f_blobs && wt == 2) l.blobs.push_back(parse_blob(r.sub()));
        else r.skip(wt);
    }
    return l;
}

void put_varint(std::string& o, uint64_t v) {
    while (v >= 0x80) { o += (char)((v & 0x7f) | 0x80); v >>= 7; }
    o += (char)v;
}
void put_key(std::string& o, int fn, int wt) { put_varint(o, ((uint64_t)fn << 3) | wt); }
void put_bytes(std::string& o, int fn, const std::string& s) {
    put_key(o, fn, 2);
    put_varint(o, s.size());
    o += s;
}
// BlobProto {data = 5 (packed), shape = 7 {dim = 1 (packed)}} as field fn of the enclosing message
void put_blob(std::string& o, int fn, const BlobProtoData& b) {
    std::string bb, dims, shape;
    for (int d : b.shape) put_varint(dims, (uint64_t)d);
    put_bytes(shape, 1, dims);
    put_bytes(bb, 5, std::string((const char*)b.data.data(), b.data.size() * 4));
    put_bytes(bb, 7, shape);
    put_bytes(o, fn, bb);
}
}  // namespace

std::vector<LayerBlobs> ParseCaffemodel(const void* bytes, size_t n) {
    Reader r{(const uint8_t*)bytes, (const uint8_t*)bytes + n};
    std::vector<LayerBlobs> out;
    while (r.ok()) {
        uint64_t key = r.varint();
        int fn = (int)(key >> 3), wt = (int)(key & 7);
        if (fn == 100 && wt == 2) out.push_back(parse_layer(r.sub(), false));
        else if (fn == 2 && wt == 2) out.push_back(parse_layer(r.sub(), true));
        else r.skip(wt);
    }
    return out;
}

std::string SerializeCaffemodel(const std::string& net_name, const std::vector<LayerBlobs>& layers) {
    std::string o;
    if (!net_name.empty()) put_bytes(o, 1, net_name);
    for (const auto& l : layers) {
        std::string lb;
        put_bytes(lb, 1, l.name);
        put_bytes(lb, 2, l.type);
        for (const auto& b : l.blobs) put_blob(lb, 7, b);
        put_bytes(o, 100, lb);
    }
    return o;
}

SolverStateData ParseSolverState(const void* bytes, size_t n) {
    Reader r{(const uint8_t*)bytes, (const uint8_t*)bytes + n};
    SolverStateData s;
    while (r.ok()) {
        uint64_t key = r.varint();
        int fn = (int)(key >> 3), wt = (int)(key & 7);
        if (fn == 1 && wt == 0) s.iter = (int)r.varint();
        else if (fn == 2 && wt == 2) { Reader t = r.sub(); s.learned_net.assign((const char*)t.p, t.end - t.p); }
        else if (fn == 3 && wt == 2) s.history.push_back(parse_blob(r.sub()));
        else if (fn == 4 && wt == 0) s.current_step = (int)r.varint();
        else r.skip(wt);
    }
    return s;
}

std::string SerializeSolverState(const SolverStateData& s) {
    std::string o;
    put_key(o, 1, 0); put_varint(o, (uint64_t)(int64_t)s.iter);
    put_bytes(o, 2, s.learned_net);
    for (const auto& b : s.history) put_blob(o, 3, b);
    put_key(o, 4, 0); put_varint(o, (uint64_t)(int64_t)s.current_step);
    return o;
}

// ------------------------------------------------------------------------------------------
// SolverParameter
// ------------------------------------------------------------------------------------------
SolverParameter SolverParameter::FromText(const std::string& text) {
    SolverParameter p;
    p.m = std::make_shared<Message>(ParseTextFormat(text));
    Message& m = *p.m;
    if (!m.has("solver_type")) return p;
    if (m.has("type"))
        throw ParseError("Failed to upgrade solver: old solver_type field (enum) and new type field (string) cannot be both "
                         "specified in solver proto text.");
    static const char* const kEnum[][3] = {{"SGD", "0", "SGD"}, {"NESTEROV", "1", "Nesterov"}, {"ADAGRAD", "2", "AdaGrad"},
                                           {"RMSPROP", "3", "RMSProp"}, {"ADADELTA", "4", "AdaDelta"}, {"ADAM", "5", "Adam"}};
    const std::string old = m.str("solver_type");
    std::string type;
    for (const auto& e : kEnum) if (old == e[0] || old == e[1]) type = e[2];
    if (type.empty()) throw ParseError("Unknown SolverParameter solver_type: " + old);
    std::vector<Field> kept;
    for (auto& f : m.fields) if (f.name != "solver_type") kept.push_back(f);
    m.fields = kept;
    m.set("type", type);
    return p;
}

std::string SolverParameter::Resolved() const {
    std::string s;
    char buf[64];
    auto num = [&](const char* name, double v, const char* fmt) { snprintf(buf, sizeof(buf), fmt, v); s += std::string(name) + ": " + buf + "\n"; };
    auto str = [&](const char* name, const std::string& v) { s += std::string(name) + ": \"" + v + "\"\n"; };
    str("type", type());
    num("base_lr", base_lr(), "%.9g");
    str("lr_policy", lr_policy());
    num("gamma", gamma(), "%.9g");
    num("power", power(), "%.9g");
    num("stepsize", stepsize(), "%.0f");
    for (int i = 0; i < stepvalue_size(); i++) num("stepvalue", stepvalue(i), "%.0f");
    num("max_iter", max_iter(), "%.0f");
    num("momentum", momentum(), "%.9g");
    num("momentum2", momentum2(), "%.9g");
    num("delta", delta(), "%.9g");
    num("weight_decay", weight_decay(), "%.9g");
    str("regularization_type", regularization_type());
    num("clip_gradients", clip_gradients(), "%.9g");
    num("iter_size", iter_size(), "%.0f");
    num("average_loss", average_loss(), "%.0f");
    num("snapshot", snapshot(), "%.0f");
    str("snapshot_prefix", snapshot_prefix());
    s += std::string("snapshot_after_train: ") + (snapshot_after_train() ? "true" : "false") + "\n";
    return s;
}

}  // namespace caffe
