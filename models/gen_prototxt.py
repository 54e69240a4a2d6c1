#!/usr/bin/env python
"""Writes the FlowNet2 deploy prototxt templates used by this repo.

NOT-IN-REF: the reference checkout ships no network definitions (models/download-models.sh only
wgets them), so these templates are authored here from the public description of the released
models (Ilg et al., CVPR'17) using exactly the layer types / parameters of the reference's
caffe.proto and the template variables of scripts/run-flownet.py:39-48
($TARGET_WIDTH$, $TARGET_HEIGHT$, $ADAPTED_WIDTH$, $ADAPTED_HEIGHT$, $SCALE_WIDTH$, $SCALE_HEIGHT$),
input blobs img0/img1 and output blob predict_flow_final (run-flownet.py:66-70,98).

    python models/gen_prototxt.py        # rewrites models/*_deploy.prototxt.template and models/*_train.prototxt.template
"""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


class P:
    def __init__(self):
        self.s = []
        self.frozen = False          # conv() then gives every parameter blob lr_mult 0 / decay_mult 0 (a frozen predecessor)

    def add(self, text):
        self.s.append(text)

    def layer(self, name, type_, bottoms, tops, body=""):
        b = "".join('  bottom: "%s"\n' % x for x in bottoms)
        t = "".join('  top: "%s"\n' % x for x in tops)
        self.s.append('layer {\n  name: "%s"\n  type: "%s"\n%s%s%s}\n' % (name, type_, b, t, body))

    def text(self):
        return "".join(self.s)


def header(p, name):
    p.add('name: "%s"\n' % name)
    for i in ("img0", "img1"):
        p.add('input: "%s"\ninput_shape {\n  dim: 1\n  dim: 3\n  dim: $TARGET_HEIGHT$\n  dim: $TARGET_WIDTH$\n}\n' % i)


def preprocess(p):
    for i in (0, 1):
        p.layer("Eltwise%d" % (i + 1), "Eltwise", ["img%d" % i], ["img%ds" % i],
                "  eltwise_param {\n    operation: SUM\n    coeff: 0.00392156862745\n  }\n")
    for i in (0, 1):
        p.layer("img%ds_aug" % i, "DataAugmentation", ["img%ds" % i], ["img%d_nomean" % i],
                "  propagate_down: false\n  augmentation_param {\n    augment_during_test: true\n"
                "    recompute_mean: 1000\n    mean_per_pixel: false\n    crop_width: $TARGET_WIDTH$\n"
                "    crop_height: $TARGET_HEIGHT$\n  }\n")
    for i in (0, 1):
        p.layer("Resample%d" % (i + 1), "Resample", ["img%d_nomean" % i], ["img%d_nomean_resize" % i],
                "  resample_param {\n    width: $ADAPTED_WIDTH$\n    height: $ADAPTED_HEIGHT$\n"
                "    type: LINEAR\n    antialias: true\n  }\n")
    return "img0_nomean_resize", "img1_nomean_resize"


FROZEN = "  param {\n    lr_mult: 0\n    decay_mult: 0\n  }\n"


def conv_body(num_output, k, stride, pad, bias_value=0.0, frozen=False):
    params = FROZEN * 2 if frozen else ("  param {\n    lr_mult: 1\n    decay_mult: 1\n  }\n"
                                        "  param {\n    lr_mult: 1\n    decay_mult: 0\n  }\n")
    return (params + "  convolution_param {\n    num_output: %d\n    pad: %d\n    kernel_size: %d\n    stride: %d\n"
            "    weight_filler {\n      type: \"msra\"\n    }\n    bias_filler {\n      type: \"constant\"\n"
            "      value: %g\n    }\n    engine: CUDNN\n  }\n" % (num_output, pad, k, stride, bias_value))


RELU = "  relu_param {\n    negative_slope: 0.1\n  }\n"


def conv(p, pre, name, bottoms, tops, num_output, k, stride, relu=True, deconv=False, pad=None):
    if pad is None:
        pad = (k - 1) // 2 if not deconv else 1
    p.layer(pre + name, "Deconvolution" if deconv else "Convolution", bottoms, tops,
            conv_body(num_output, k, stride, pad, frozen=p.frozen))
    if relu:
        for i, t in enumerate(tops):
            p.layer("%sReLU_%s%s" % (pre, name, "" if len(tops) == 1 else "_%d" % i), "ReLU", [t], [t], RELU)


def refinement(p, pre, skips, top6, inter=False):
    """Decoder shared by FlowNetS/C/SD.  skips: {5: blob, 4: blob, 3: blob, 2: blob}, top6: conv6_1."""
    feat = top6
    flow = None
    for lvl in (6, 5, 4, 3, 2):
        if lvl != 6:
            nch = {5: 512, 4: 256, 3: 128, 2: 64}[lvl]
            conv(p, pre, "deconv%d" % lvl, [feat], [pre + "deconv%d" % lvl], nch, 4, 2, relu=True, deconv=True)
            conv(p, pre, "upsample_flow%dto%d" % (lvl + 1, lvl), [flow], [pre + "upsampled_flow%d_to_%d" % (lvl + 1, lvl)],
                 2, 4, 2, relu=False, deconv=True)
            cat = pre + "concat%d" % lvl
            p.layer(pre + "Concat%d" % lvl, "Concat", [skips[lvl], pre + "deconv%d" % lvl,
                                                       pre + "upsampled_flow%d_to_%d" % (lvl + 1, lvl)], [cat],
                    "  concat_param {\n    axis: 1\n  }\n")
            feat = cat
        src = feat
        if inter and lvl != 6:
            conv(p, pre, "interconv%d" % lvl, [feat], [pre + "interconv%d" % lvl], {5: 512, 4: 256, 3: 128, 2: 64}[lvl],
                 3, 1, relu=False)
            src = pre + "interconv%d" % lvl
        flow = pre + "predict_flow%d" % lvl
        conv(p, pre, "predict_flow%d" % lvl, [src], [flow], 2, 3, 1, relu=False)
    return flow


def flownet_s(p, pre, inp):
    conv(p, pre, "conv1", [inp], [pre + "conv1"], 64, 7, 2)
    conv(p, pre, "conv2", [pre + "conv1"], [pre + "conv2"], 128, 5, 2)
    conv(p, pre, "conv3", [pre + "conv2"], [pre + "conv3"], 256, 5, 2)
    conv(p, pre, "conv3_1", [pre + "conv3"], [pre + "conv3_1"], 256, 3, 1)
    conv(p, pre, "conv4", [pre + "conv3_1"], [pre + "conv4"], 512, 3, 2)
    conv(p, pre, "conv4_1", [pre + "conv4"], [pre + "conv4_1"], 512, 3, 1)
    conv(p, pre, "conv5", [pre + "conv4_1"], [pre + "conv5"], 512, 3, 2)
    conv(p, pre, "conv5_1", [pre + "conv5"], [pre + "conv5_1"], 512, 3, 1)
    conv(p, pre, "conv6", [pre + "conv5_1"], [pre + "conv6"], 1024, 3, 2)
    conv(p, pre, "conv6_1", [pre + "conv6"], [pre + "conv6_1"], 1024, 3, 1)
    return refinement(p, pre, {5: pre + "conv5_1", 4: pre + "conv4_1", 3: pre + "conv3_1", 2: pre + "conv2"},
                      pre + "conv6_1")


def flownet_c(p, pre, img0, img1):
    conv(p, pre, "conv1", [img0, img1], [pre + "conv1a", pre + "conv1b"], 64, 7, 2)
    conv(p, pre, "conv2", [pre + "conv1a", pre + "conv1b"], [pre + "conv2a", pre + "conv2b"], 128, 5, 2)
    conv(p, pre, "conv3", [pre + "conv2a", pre + "conv2b"], [pre + "conv3a", pre + "conv3b"], 256, 5, 2)
    p.layer(pre + "corr", "Correlation", [pre + "conv3a", pre + "conv3b"], [pre + "corr"],
            "  correlation_param {\n    pad: 20\n    kernel_size: 1\n    max_displacement: 20\n    stride_1: 1\n"
            "    stride_2: 2\n  }\n")
    p.layer(pre + "ReLU_corr", "ReLU", [pre + "corr"], [pre + "corr"], RELU)
    conv(p, pre, "conv_redir", [pre + "conv3a"], [pre + "conv_redir"], 32, 1, 1)
    p.layer(pre + "Concat_corr", "Concat", [pre + "conv_redir", pre + "corr"], [pre + "blob_corr"],
            "  concat_param {\n    axis: 1\n  }\n")
    conv(p, pre, "conv3_1", [pre + "blob_corr"], [pre + "conv3_1"], 256, 3, 1)
    conv(p, pre, "conv4", [pre + "conv3_1"], [pre + "conv4"], 512, 3, 2)
    conv(p, pre, "conv4_1", [pre + "conv4"], [pre + "conv4_1"], 512, 3, 1)
    conv(p, pre, "conv5", [pre + "conv4_1"], [pre + "conv5"], 512, 3, 2)
    conv(p, pre, "conv5_1", [pre + "conv5"], [pre + "conv5_1"], 512, 3, 1)
    conv(p, pre, "conv6", [pre + "conv5_1"], [pre + "conv6"], 1024, 3, 2)
    conv(p, pre, "conv6_1", [pre + "conv6"], [pre + "conv6_1"], 1024, 3, 1)
    return refinement(p, pre, {5: pre + "conv5_1", 4: pre + "conv4_1", 3: pre + "conv3_1", 2: pre + "conv2a"},
                      pre + "conv6_1")


def flownet_sd(p, pre, inp):
    conv(p, pre, "conv0", [inp], [pre + "conv0"], 64, 3, 1)
    conv(p, pre, "conv1", [pre + "conv0"], [pre + "conv1"], 64, 3, 2)
    conv(p, pre, "conv1_1", [pre + "conv1"], [pre + "conv1_1"], 128, 3, 1)
    conv(p, pre, "conv2", [pre + "conv1_1"], [pre + "conv2"], 128, 3, 2)
    conv(p, pre, "conv2_1", [pre + "conv2"], [pre + "conv2_1"], 128, 3, 1)
    conv(p, pre, "conv3", [pre + "conv2_1"], [pre + "conv3"], 256, 3, 2)
    conv(p, pre, "conv3_1", [pre + "conv3"], [pre + "conv3_1"], 256, 3, 1)
    conv(p, pre, "conv4", [pre + "conv3_1"], [pre + "conv4"], 512, 3, 2)
    conv(p, pre, "conv4_1", [pre + "conv4"], [pre + "conv4_1"], 512, 3, 1)
    conv(p, pre, "conv5", [pre + "conv4_1"], [pre + "conv5"], 512, 3, 2)
    conv(p, pre, "conv5_1", [pre + "conv5"], [pre + "conv5_1"], 512, 3, 1)
    conv(p, pre, "conv6", [pre + "conv5_1"], [pre + "conv6"], 1024, 3, 2)
    conv(p, pre, "conv6_1", [pre + "conv6"], [pre + "conv6_1"], 1024, 3, 1)
    return refinement(p, pre, {5: pre + "conv5_1", 4: pre + "conv4_1", 3: pre + "conv3_1", 2: pre + "conv2_1"},
                      pre + "conv6_1", inter=True)


def scale(p, name, bottom, top, coeff):
    p.layer(name, "Eltwise", [bottom], [top], "  eltwise_param {\n    operation: SUM\n    coeff: %s\n  }\n" % coeff)


def upsample_to(p, name, bottom, top, like):
    # two-bottom Resample takes its output size from bottom[1] (resample_layer.cpp:44-46)
    p.layer(name, "Resample", [bottom, like], [top], "  resample_param {\n    type: LINEAR\n    antialias: true\n  }\n")


def warp_block(p, pre, flow_quarter, img0, img1):
    """flow at 1/4 res (network scale) -> full-res flow in pixels, warped img1, brightness error."""
    scale(p, pre + "flow_x20", flow_quarter, pre + "flow_x20", "20.0")
    upsample_to(p, pre + "Resample_flow", pre + "flow_x20", pre + "flow_full", img0)
    p.layer(pre + "FlowWarp", "FlowWarp", [img1, pre + "flow_full"], [pre + "img1_warped"])
    p.layer(pre + "Eltwise_err", "Eltwise", [img0, pre + "img1_warped"], [pre + "err"],
            "  eltwise_param {\n    operation: SUM\n    coeff: 1.0\n    coeff: -1.0\n  }\n")
    p.layer(pre + "ChannelNorm_err", "ChannelNorm", [pre + "err"], [pre + "err_norm"])
    scale(p, pre + "flow_scaled", pre + "flow_full", pre + "flow_scaled", "0.05")
    return pre + "flow_full", pre + "flow_scaled", pre + "img1_warped", pre + "err_norm"


def postprocess(p, flow, like_scale_quarter=True):
    """network-scale flow -> pixels at ADAPTED size -> TARGET size, rescaled (run-flownet.py:47-48)."""
    scale(p, "Eltwise_final_x20", flow, "predict_flow_x20", "20.0")
    p.layer("Resample_final", "Resample", ["predict_flow_x20"], ["predict_flow_resize"],
            "  resample_param {\n    width: $TARGET_WIDTH$\n    height: $TARGET_HEIGHT$\n    type: LINEAR\n"
            "    antialias: true\n  }\n")
    p.layer("scale_conv1", "Convolution", ["predict_flow_resize"], ["predict_flow_final"],
            "  param {\n    lr_mult: 0\n    decay_mult: 0\n  }\n  convolution_param {\n    num_output: 2\n    pad: 0\n"
            "    kernel_size: 1\n    stride: 1\n    bias_term: false\n    weight_filler {\n      type: \"diagonal\"\n"
            "      diag_val: $SCALE_WIDTH$\n      diag_val: $SCALE_HEIGHT$\n    }\n  }\n")


def concat(p, name, bottoms, top):
    p.layer(name, "Concat", bottoms, [top], "  concat_param {\n    axis: 1\n  }\n")


def build_s():
    p = P(); header(p, "FlowNet2-S"); a, b = preprocess(p)
    concat(p, "Concat_input", [a, b], "input")
    flow = flownet_s(p, "", "input")
    postprocess(p, flow)
    return p.text()


def build_c():
    p = P(); header(p, "FlowNet2-C"); a, b = preprocess(p)
    flow = flownet_c(p, "", a, b)
    postprocess(p, flow)
    return p.text()


def css_body(p, a, b, stages=(2, 3), frozen=()):
    """FlowNet-C (net1_) and one FlowNet-S per entry of `stages`, each fed through a warp block; prefixes in `frozen` get
    lr_mult 0."""
    p.frozen = "net1_" in frozen
    flow = flownet_c(p, "net1_", a, b)
    for k in stages:
        full, scaled, warped, err = warp_block(p, "net%d_in_" % k, flow, a, b)
        concat(p, "net%d_Concat_input" % k, [a, b, warped, scaled, err], "net%d_input" % k)
        p.frozen = "net%d_" % k in frozen
        flow = flownet_s(p, "net%d_" % k, "net%d_input" % k)
    p.frozen = False
    return flow


def build_css():
    p = P(); header(p, "FlowNet2-CSS"); a, b = preprocess(p)
    flow = css_body(p, a, b)
    postprocess(p, flow)
    return p.text()


def build_cs():
    p = P(); header(p, "FlowNet2-CS"); a, b = preprocess(p)
    flow = css_body(p, a, b, stages=(2,))
    postprocess(p, flow)
    return p.text()


def build_sd():
    p = P(); header(p, "FlowNet2-SD"); a, b = preprocess(p)
    concat(p, "Concat_input", [a, b], "input")
    flow = flownet_sd(p, "", "input")
    postprocess(p, flow)
    return p.text()


def build_full():
    p = P(); header(p, "FlowNet2"); a, b = preprocess(p)
    flow_css = css_body(p, a, b)
    concat(p, "netsd_Concat_input", [a, b], "netsd_input")
    flow_sd = flownet_sd(p, "netsd_", "netsd_input")
    flow = fusion(p, a, b, flow_css, flow_sd)
    # fusion output is already in pixels at ADAPTED size
    p.layer("Resample_final", "Resample", [flow], ["predict_flow_resize"],
            "  resample_param {\n    width: $TARGET_WIDTH$\n    height: $TARGET_HEIGHT$\n    type: LINEAR\n"
            "    antialias: true\n  }\n")
    p.layer("scale_conv1", "Convolution", ["predict_flow_resize"], ["predict_flow_final"],
            "  param {\n    lr_mult: 0\n    decay_mult: 0\n  }\n  convolution_param {\n    num_output: 2\n    pad: 0\n"
            "    kernel_size: 1\n    stride: 1\n    bias_term: false\n    weight_filler {\n      type: \"diagonal\"\n"
            "      diag_val: $SCALE_WIDTH$\n      diag_val: $SCALE_HEIGHT$\n    }\n  }\n")
    return p.text()


def fusion(p, a, b, flow_css, flow_sd):
    """The fusion network on the CSS and SD flows: -> fuse_predict_flow0, flow in pixels at the input's resolution."""
    # fusion inputs at full (adapted) resolution
    full1, _, _, err1 = warp_block(p, "fuse_css_", flow_css, a, b)
    full2, _, _, err2 = warp_block(p, "fuse_sd_", flow_sd, a, b)
    p.layer("fuse_css_mag", "ChannelNorm", [full1], ["fuse_css_mag"])
    p.layer("fuse_sd_mag", "ChannelNorm", [full2], ["fuse_sd_mag"])
    concat(p, "fuse_Concat_input", [a, full1, full2, "fuse_css_mag", "fuse_sd_mag", err1, err2], "fuse_input")
    pre = "fuse_"
    conv(p, pre, "conv0", ["fuse_input"], [pre + "conv0"], 64, 3, 1)
    conv(p, pre, "conv1", [pre + "conv0"], [pre + "conv1"], 64, 3, 2)
    conv(p, pre, "conv1_1", [pre + "conv1"], [pre + "conv1_1"], 128, 3, 1)
    conv(p, pre, "conv2", [pre + "conv1_1"], [pre + "conv2"], 128, 3, 2)
    conv(p, pre, "conv2_1", [pre + "conv2"], [pre + "conv2_1"], 128, 3, 1)
    conv(p, pre, "predict_flow2", [pre + "conv2_1"], [pre + "predict_flow2"], 2, 3, 1, relu=False)
    conv(p, pre, "deconv1", [pre + "conv2_1"], [pre + "deconv1"], 32, 4, 2, relu=True, deconv=True)
    conv(p, pre, "upsample_flow2to1", [pre + "predict_flow2"], [pre + "upsampled_flow2_to_1"], 2, 4, 2, relu=False, deconv=True)
    concat(p, pre + "Concat1", [pre + "conv1_1", pre + "deconv1", pre + "upsampled_flow2_to_1"], pre + "concat1")
    conv(p, pre, "interconv1", [pre + "concat1"], [pre + "interconv1"], 32, 3, 1, relu=False)
    conv(p, pre, "predict_flow1", [pre + "interconv1"], [pre + "predict_flow1"], 2, 3, 1, relu=False)
    conv(p, pre, "deconv0", [pre + "concat1"], [pre + "deconv0"], 16, 4, 2, relu=True, deconv=True)
    conv(p, pre, "upsample_flow1to0", [pre + "predict_flow1"], [pre + "upsampled_flow1_to_0"], 2, 4, 2, relu=False, deconv=True)
    concat(p, pre + "Concat0", [pre + "conv0", pre + "deconv0", pre + "upsampled_flow1_to_0"], pre + "concat0")
    conv(p, pre, "interconv0", [pre + "concat0"], [pre + "interconv0"], 16, 3, 1, relu=False)
    conv(p, pre, "predict_flow0", [pre + "interconv0"], [pre + "predict_flow0"], 2, 3, 1, relu=False)
    return pre + "predict_flow0"


# ---- FlowNet2-C training net (BASELINE.json config 5) ------------------------------------------------------------------------
# NOT-IN-REF like the deploy templates: authored from the public description of the FlowNetC training setup (FlyingChairs 512x384
# frames cropped to 448x320 by the augmentation, multi-scale end-point-error losses with weights 0.32 / 0.08 / 0.02 / 0.01 / 0.005,
# ground truth scaled by 1/20 and downsampled per level) with the layer types of the reference's caffe.proto.  The CustomData /
# LMDB reader is out of scope (SURVEY.md 8): img0, img1, flow_gt are Input blobs.
def _gen(kind, exp, mean, spread):
    return ('{ rand_type: "%s" exp: %s mean: %g spread: %g prob: 1.0 }' % (kind, "true" if exp else "false", mean, spread))


EIGVEC = [0.51, 0.56, 0.65, 0.79, 0.01, -0.62, 0.35, -0.83, 0.44]


def train_head(p, name, scale_gt=True):
    """Input frames and ground truth, augmentation of both frames and of the flow -> img0_aug, img1_aug, and the ground truth
    flow_gt_aug (pixels) or, with scale_gt, scaled_flow_gt_aug (network scale, x 0.05)."""
    p.add('name: "%s"\n' % name)
    p.layer("data", "Input", [], ["img0", "img1", "flow_gt"],
            "  input_param {\n" + "".join("    shape { dim: $BATCH$ dim: %d dim: $DATA_HEIGHT$ dim: $DATA_WIDTH$ }\n" % c for c in (3, 3, 2)) + "  }\n")
    for i in (0, 1):
        scale(p, "Eltwise%d" % (i + 1), "img%d" % i, "img%ds" % i, "0.00392156862745")
    ub, gb = "uniform_bernoulli", "gaussian_bernoulli"
    common = ("    max_multiplier: 1\n    augment_during_test: false\n    recompute_mean: 1000\n    mean_per_pixel: false\n"
              "    crop_width: $TARGET_WIDTH$\n    crop_height: $TARGET_HEIGHT$\n")
    spatial0 = ("    translate %s\n    rotate %s\n    zoom %s\n    squeeze %s\n"
                % (_gen(ub, False, 0, 0.4), _gen(ub, False, 0, 0.4), _gen(ub, True, 0.2, 0.4), _gen(ub, True, 0, 0.3)))
    chroma = "".join("    %s %s\n" % (n, g) for n, g in (
        ("lmult_pow", _gen(ub, True, -0.2, 0.4)), ("lmult_mult", _gen(ub, True, 0.0, 0.4)), ("lmult_add", _gen(ub, False, 0, 0.03)),
        ("sat_pow", _gen(ub, True, 0, 0.4)), ("sat_mult", _gen(ub, True, -0.3, 0.5)), ("sat_add", _gen(ub, False, 0, 0.03)),
        ("col_pow", _gen(gb, True, 0, 0.4)), ("col_mult", _gen(gb, True, 0, 0.2)), ("col_add", _gen(gb, False, 0, 0.02)),
        ("ladd_pow", _gen(gb, True, 0, 0.4)), ("ladd_mult", _gen(gb, True, 0.0, 0.4)), ("ladd_add", _gen(gb, False, 0, 0.04)),
        ("col_rotate", _gen(ub, False, 0, 1)), ("noise", _gen(ub, False, 0.03, 0.03))))
    eig = "".join("    chromatic_eigvec: %g\n" % e for e in EIGVEC)
    sched = "  coeff_schedule_param {\n    half_life: 50000\n    initial_coeff: 0.5\n    final_coeff: 1\n  }\n"
    p.layer("img0s_aug", "DataAugmentation", ["img0s"], ["img0_aug", "img0_aug_params"],
            "  propagate_down: false\n  augmentation_param {\n" + common + spatial0 + chroma + eig + "  }\n" + sched)
    # second frame: the first frame's coefficients plus a small relative transform and colour change
    p.layer("aug_params1", "GenerateAugmentationParameters", ["img0_aug_params", "img0s", "img0_aug"], ["img1_aug_params"],
            "  augmentation_param {\n    augment_during_test: false\n    mode: \"add\"\n"
            "    translate %s\n    rotate %s\n    zoom %s\n    gamma %s\n    brightness %s\n    contrast %s\n    color %s\n  }\n"
            % (_gen(ub, False, 0, 0.03), _gen(ub, False, 0, 0.03), _gen(ub, True, 0, 0.03), _gen(gb, True, 0, 0.02),
               _gen(gb, False, 0, 0.02), _gen(gb, True, 0, 0.02), _gen(gb, True, 0, 0.02)) + sched)
    p.layer("img1s_aug", "DataAugmentation", ["img1s", "img1_aug_params"], ["img1_aug"],
            "  propagate_down: false\n  propagate_down: false\n  augmentation_param {\n" + common + eig + "  }\n")
    p.layer("flow_aug", "FlowAugmentation", ["flow_gt", "img0_aug_params", "img1_aug_params"], ["flow_gt_aug"],
            "  augmentation_param {\n    crop_width: $TARGET_WIDTH$\n    crop_height: $TARGET_HEIGHT$\n  }\n")
    if scale_gt:
        scale(p, "scale_gt", "flow_gt_aug", "scaled_flow_gt_aug", "0.05")
    return "img0_aug", "img1_aug"


LOSS_WEIGHTS = ((6, 0.32), (5, 0.08), (4, 0.02), (3, 0.01), (2, 0.005))
# NOT-IN-REF and without a public source: the fusion network's loss weights (flow in pixels at 1/4, 1/2 and full resolution)
FUSION_LOSS_WEIGHTS = ((2, 0.005), (1, 0.01), (0, 0.02))


def losses(p, gt, pre, weights=LOSS_WEIGHTS):
    """End-point-error loss of <pre>predict_flow<level> against the ground truth `gt` downsampled to its size, per level."""
    for lvl, wgt in weights:
        pred = "%spredict_flow%d" % (pre, lvl)
        p.layer("Downsample%d" % lvl, "Downsample", [gt, pred], ["blob_gt%d" % lvl],
                "  propagate_down: false\n  propagate_down: false\n")
        p.layer("flow_loss%d" % lvl, "L1Loss", [pred, "blob_gt%d" % lvl], ["flow_loss%d" % lvl],
                "  loss_weight: %g\n  l1_loss_param {\n    l2_per_location: true\n  }\n" % wgt)


def build_c_train():
    p = P()
    a, b = train_head(p, "FlowNet2-C-train")
    flownet_c(p, "", a, b)
    losses(p, "scaled_flow_gt_aug", "")
    return p.text()


# ---- the stacked FlowNet2 training schedule: each stage trains its newest sub-network on top of frozen predecessors -----------
# NOT-IN-REF like the C template (the reference ships no training prototxts): the stages of Ilg et al. (CVPR'17) -- CS on a
# frozen C, CSS on a frozen CS, SD on its own, the fusion network on a frozen CSS and a frozen SD.  Layer names are those of
# the deploy templates, so a trained caffemodel loads into the matching deploy net by name.  The warp blocks read the
# augmented frames; Resample allows no backward, so no gradient ever reaches a warp block or a frozen predecessor.
def build_cs_train():
    p = P()
    a, b = train_head(p, "FlowNet2-CS-train")
    css_body(p, a, b, stages=(2,), frozen=("net1_",))
    losses(p, "scaled_flow_gt_aug", "net2_")
    return p.text()


def build_css_train():
    p = P()
    a, b = train_head(p, "FlowNet2-CSS-train")
    css_body(p, a, b, frozen=("net1_", "net2_"))
    losses(p, "scaled_flow_gt_aug", "net3_")
    return p.text()


def build_sd_train():
    p = P()
    a, b = train_head(p, "FlowNet2-SD-train")
    concat(p, "Concat_input", [a, b], "input")
    flownet_sd(p, "", "input")
    losses(p, "scaled_flow_gt_aug", "")
    return p.text()


def build_full_train():
    """The fusion stage.  The fusion network predicts flow in pixels, so its ground truth is not scaled."""
    p = P()
    a, b = train_head(p, "FlowNet2-train", scale_gt=False)
    flow_css = css_body(p, a, b, frozen=("net1_", "net2_", "net3_"))
    concat(p, "netsd_Concat_input", [a, b], "netsd_input")
    p.frozen = True
    flow_sd = flownet_sd(p, "netsd_", "netsd_input")
    p.frozen = False
    fusion(p, a, b, flow_css, flow_sd)
    losses(p, "flow_gt_aug", "fuse_", FUSION_LOSS_WEIGHTS)
    return p.text()


MODELS = {"FlowNet2-S": build_s, "FlowNet2-C": build_c, "FlowNet2-CS": build_cs, "FlowNet2-CSS": build_css,
          "FlowNet2-SD": build_sd, "FlowNet2": build_full}
TRAIN_MODELS = {"FlowNet2-C": build_c_train, "FlowNet2-CS": build_cs_train, "FlowNet2-CSS": build_css_train,
                "FlowNet2-SD": build_sd_train, "FlowNet2": build_full_train}

if __name__ == "__main__":
    for name, fn in MODELS.items():
        path = os.path.join(HERE, "%s_deploy.prototxt.template" % name)
        with open(path, "w") as f:
            f.write(fn())
        print("wrote", path)
    for name, fn in TRAIN_MODELS.items():
        path = os.path.join(HERE, "%s_train.prototxt.template" % name)
        with open(path, "w") as f:
            f.write(fn())
        print("wrote", path)
