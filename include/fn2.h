/*
 * fn2.h -- C-ABI of libfn2.so, the Hopper-native (sm_90a) FlowNet2 forward hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  Each entry
 * point names the reference (lmb-freiburg/flownet2 @ b92e198) function it replaces; the
 * reference-side binding (a Caffe Layer subclass whose Forward_gpu calls the entry point)
 * is shown in INTEGRATION.md.  The Caffe-surface C++ host (namespace caffe: Blob, Layer,
 * LayerParameter, LayerRegistry, Net) that sits above this ABI lives in
 * flownet2_b200/csrc/caffe/ and is itself reachable through the fn2_net_* functions below.
 *
 * Conventions
 *   - All data is fp32 on the device.  Tensors are described by fn2_tensor: logical Caffe
 *     dims (n,c,h,w) plus element strides, so both the reference's NCHW blobs
 *     (sn=c*h*w, sc=h*w, sh=w, sw=1) and the engine's internal NHWC activations
 *     (sc=1, sw=channel stride) and channel-offset views into concat buffers are expressible.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued asynchronously.
 *   - Return value: 0 = FN2_OK, negative = error (see fn2_status); fn2_last_error() returns a
 *     thread-local description.  Nothing here aborts the process (the reference CHECK-fails).
 */
#ifndef FN2_H_
#define FN2_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FN2_API __attribute__((visibility("default")))

typedef enum fn2_status {
    FN2_OK = 0,
    FN2_ERR_INVALID = -1,      /* bad argument / unsupported configuration */
    FN2_ERR_CUDA = -2,         /* CUDA runtime or driver error */
    FN2_ERR_PARSE = -3,        /* prototxt / caffemodel parse error */
    FN2_ERR_NOTFOUND = -4,     /* unknown blob / layer / type */
    FN2_ERR_WORKSPACE = -5     /* workspace too small */
} fn2_status;

typedef struct fn2_tensor {
    float* data;               /* device pointer */
    int32_t n, c, h, w;        /* logical Caffe dims */
    int64_t sn, sc, sh, sw;    /* element strides */
} fn2_tensor;

FN2_API const char* fn2_last_error(void);
FN2_API const char* fn2_version(void);
/* Number of kernels launched by this library on the calling thread since process start
 * (bench.py's gpu_launches). */
FN2_API uint64_t fn2_launch_count(void);
/* Allocations the Caffe-surface host has made since process start (device and pinned host blocks); *live_bytes (if not
 * NULL) receives the bytes it holds now.  For tests of steady-state allocation and leaks. */
FN2_API uint64_t fn2_device_allocations(uint64_t* live_bytes);

/* ------------------------------------------------------------------------------------ */
/* Correlation -- replaces CorrelationLayer::Forward_gpu / Backward_gpu                  */
/*   reference: src/caffe/layers/correlation_layer.cu:431-504 (fwd), :508-600 (bwd),      */
/*   shapes src/caffe/layers/correlation_layer.cpp:41-84.                                 */
/* corr_type: 0 MULTIPLY, 1 SUBTRACT (caffe.proto:639-643).                               */
/* ------------------------------------------------------------------------------------ */
FN2_API int fn2_correlation_shape(int H, int W, int pad, int kernel_size, int max_displacement,
                                  int stride1, int stride2, int* top_channels, int* top_h,
                                  int* top_w);
FN2_API int fn2_correlation_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size,
                                            int max_displacement, int stride1, int stride2,
                                            int corr_type, size_t* bytes);
FN2_API int fn2_correlation_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1,
                                    const fn2_tensor* top, int pad, int kernel_size,
                                    int max_displacement, int stride1, int stride2, int corr_type,
                                    void* workspace, size_t workspace_bytes, void* stream);
/* Gradients w.r.t. both bottoms: CorrelateDataBackward0/1 (:118-249), ...Subtract (:298-427), driver :508-600.  Computed through
 * the factorisation described in flownet2_b200/csrc/fn2_corr_bwd.cu (channel-free patch sum of top_diff, then a tiled
 * displacement-sum against the other map).  Workspace: N*H*W*D floats for the patch sum unless kernel_size 1, stride_1 1,
 * pad == max_displacement, and for FlowNet2-C's fast route (MULTIPLY, that identity patch walk, 21 x 21 displacements,
 * stride_2 <= 2, C % 32 == 0); plus N*H*W*C floats for the SUBTRACT sign map. */
FN2_API int fn2_correlation_backward_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size, int max_displacement,
                                                     int stride1, int stride2, int corr_type, size_t* bytes);
FN2_API int fn2_correlation_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1,
                                     const fn2_tensor* top_diff, const fn2_tensor* bottom0_diff,
                                     const fn2_tensor* bottom1_diff, int pad, int kernel_size,
                                     int max_displacement, int stride1, int stride2, int corr_type,
                                     void* workspace, size_t workspace_bytes, void* stream);

/* Correlation1D -- replaces Correlation1DLayer (correlation_layer1d.cpp:37-84 shapes, correlation_layer1d.cu:48-112 forward,
 * :116-247 backward): displacement along x only, rows are not padded.  single_direction: -1 left, 0 both, +1 right
 * (caffe.proto CorrelationParameter.single_direction); top channel tc <-> x offset (tc + x_shift) * stride_2. */
FN2_API int fn2_correlation1d_shape(int H, int W, int pad, int kernel_size, int max_displacement, int stride1, int stride2,
                                    int single_direction, int* top_channels, int* top_h, int* top_w);
FN2_API int fn2_correlation1d_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top, int pad,
                                      int kernel_size, int max_displacement, int stride1, int stride2, int single_direction,
                                      int corr_type, void* stream);
FN2_API int fn2_correlation1d_backward_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size, int max_displacement,
                                                       int stride1, int stride2, int single_direction, int corr_type, size_t* bytes);
FN2_API int fn2_correlation1d_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top_diff,
                                       const fn2_tensor* bottom0_diff, const fn2_tensor* bottom1_diff, int pad, int kernel_size,
                                       int max_displacement, int stride1, int stride2, int single_direction, int corr_type,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------ */
/* FlowWarp -- replaces FlowWarpLayer::Forward_gpu / Backward_gpu                         */
/*   reference: src/caffe/layers/flow_warp_layer.cu:357-458, :461-514; CPU twin           */
/*   flow_warp_layer.cpp:57-198.  fill_nan: 0 = ZERO, 1 = NOT_A_NUMBER (caffe.proto:553).  */
/* ------------------------------------------------------------------------------------ */
FN2_API int fn2_flow_warp_forward(const fn2_tensor* image, const fn2_tensor* flow,
                                  const fn2_tensor* warped, int fill_nan, void* stream);
FN2_API int fn2_flow_warp_backward(const fn2_tensor* image, const fn2_tensor* flow,
                                   const fn2_tensor* warped_diff, const fn2_tensor* image_diff,
                                   const fn2_tensor* flow_diff, void* stream);

/* ------------------------------------------------------------------------------------ */
/* Resample -- replaces ResampleLayer::Forward_gpu (resample_layer.cu:128-206).           */
/* type: 1 NEAREST, 2 LINEAR, 3 CUBIC (caffe.proto:666-671).                              */
/* ------------------------------------------------------------------------------------ */
FN2_API int fn2_resample_forward(const fn2_tensor* bottom, const fn2_tensor* top, int type,
                                 int antialias, void* stream);

/* The warp block between two stacked networks as one pass (what Net::Init substitutes for the layer chain
 * Resample(LINEAR, 2 bottoms) -> FlowWarp -> Eltwise(1, -1) -> ChannelNorm plus Eltwise(coeff) on the up-sampled flow):
 * flow_in (N,2,h,w) is up-sampled to flow_full (N,2,H,W); image1 is warped by it; err = image0 - warped; err_norm = |err|_2
 * over the channels; flow_scaled = scale_coeff * flow_full.  Bit-identical to the layer chain. */
FN2_API int fn2_warp_block_forward(const fn2_tensor* flow_in, const fn2_tensor* image0, const fn2_tensor* image1,
                                   const fn2_tensor* flow_full, const fn2_tensor* warped, const fn2_tensor* err,
                                   const fn2_tensor* err_norm, const fn2_tensor* flow_scaled, float scale_coeff, int fill_nan,
                                   void* stream);

/* ------------------------------------------------------------------------------------ */
/* DataAugmentation kernels -- replace the device side of                                 */
/* DataAugmentationLayer::Forward_gpu (data_augmentation_layer.cu:321-637).               */
/* ------------------------------------------------------------------------------------ */
/* SpatialAugmentation (:25-70).  trans_mats: device array, 6 floats per sample in NAME order
 * t0,t1,t2,t3,t4,t5 (xin = x*t0 + y*t2 + t4 ; yin = x*t1 + y*t3 + t5). */
FN2_API int fn2_spatial_augmentation(const fn2_tensor* bottom, const fn2_tensor* top,
                                     const float* trans_mats_dev, void* stream);
/* ColorContrastAugmentation (:73-117), in place.  chroma: device array, 6 floats per sample
 * {gamma, brightness, contrast, color0, color1, color2}. */
FN2_API int fn2_color_contrast_augmentation(const fn2_tensor* data, const float* chroma_dev,
                                            float max_multiplier, void* stream);
/* Running-mean update of :600-608: mean_pp = (mean_pp*(num_iter-1) + sum_n top_n/num)/num_iter,
 * mean_pc[c] = average of mean_pp over the area.  mean_pp is a (1,C,H,W)-shaped tensor. */
/* Training-time augmentations (3-channel data, in place).  Reference: ComputeChromaticEigenspace / ChromaticEigenAugmentation /
 * ApplyEffects, data_augmentation_layer.cu:148-318 and the host-side finalisation / noise of Forward_gpu :486-583.
 *   space_dev : 32 floats, 8-byte aligned: tChromaticEigenSpace (25 floats: mean_eig[3], mean_rgb[3], max_abs_eig[3],
 *               max_rgb[3], min_rgb[3], max_l, eigvec[9], augmentation_layer_base.hpp:117-129) + scratch
 *   coeffs_dev: N x 22 floats in tChromaticEigenCoeffs order (augmentation_layer_base.hpp:52-75)
 *   effects_dev: N x 9 floats in tEffectCoeffs order (fog_amount, fog_size, motion_blur_angle, motion_blur_size,
 *               shadow_nx, shadow_ny, shadow_distance, shadow_strength, noise); as in the reference only the shadow, the
 *               clamp and the additive Gaussian noise act.  The noise stream is this library's own counter-based generator
 *               (the reference's cuRAND stream is unpinned). */
FN2_API int fn2_chromatic_eigenspace(const fn2_tensor* data, const float* eigvec9_dev, float* space_dev, void* stream);
FN2_API int fn2_chromatic_eigen_augmentation(const fn2_tensor* data, const float* coeffs_dev, const float* space_dev,
                                             float max_multiplier, void* stream);
FN2_API int fn2_apply_effects(const fn2_tensor* data, const float* effects_dev, float max_multiplier,
                              unsigned long long noise_seed, int add_noise, void* stream);
FN2_API int fn2_mean_update(const fn2_tensor* top, const fn2_tensor* mean_pp, float* mean_pc_dev,
                            float num_iter, void* stream);
/* Mean subtraction :610-634: per_pixel != 0 subtracts mean_pp, else the per-channel values. */
FN2_API int fn2_mean_subtract(const fn2_tensor* top, const fn2_tensor* mean_pp,
                              const float* mean_pc_dev, int per_pixel, void* stream);

/* ------------------------------------------------------------------------------------ */
/* Convolution / Deconvolution (+ fused bias and leaky ReLU)                              */
/*   reference: conv_layer.cu:8-23, deconv_layer.cu:8-23, base_conv_layer.cpp:257-298,    */
/*   relu_layer.cu:9-14.                                                                  */
/* ------------------------------------------------------------------------------------ */
typedef struct fn2_conv_desc {
    int32_t ci, co;            /* channels in / out (group == 1 only) */
    int32_t kh, kw, stride_h, stride_w, pad_h, pad_w;
    int32_t deconv;            /* 0 convolution, 1 deconvolution (transposed) */
    int32_t has_bias;
    int32_t relu;              /* 1: apply x>0 ? x : x*negative_slope in the epilogue */
    float negative_slope;
    int32_t engine;            /* 0 default (tensor cores when eligible), 1 SIMT fp32, 2 tensor cores (wgmma 3xTF32) */
    int32_t input_guard_bytes; /* readable (never used) bytes the caller guarantees before AND after the bottom tensor's
                                * storage; >= 512 lets small-Ci convolutions fetch whole kernel rows per TMA box. 0 = none.
                                * Those rows include the padding channels of a bottom whose pixel stride is Ci rounded up
                                * to 4: with a guard band they must hold finite values (they meet zero weights, and
                                * 0 * NaN is NaN).  The SIMT flow-predictor kernels (Co = 2) read each pixel as whole
                                * float4 groups, so with a guard band the channels of a pixel's last group beyond Ci
                                * (padding, or a neighbouring view's channels) must be finite too.  Without one none of
                                * these channels is used. */
    int32_t out_pad_h, out_pad_w; /* deconvolution only: extra output rows / columns at the bottom / right (0 for every Caffe
                                * layer; the adjoint of a strided convolution needs (H + 2 pad - k) mod stride of them to
                                * reach the whole bottom, fn2_conv_backward_data_desc) */
} fn2_conv_desc;

/* Packed weight size (floats) and packing from Caffe layout: conv [co][ci][kh][kw]
 * (base_conv_layer.cpp:135-140), deconv [ci][co][kh][kw] (:125-137).  Packing happens once
 * at weight-load time.  ci_stride = padded channel count of the input tensor. */
FN2_API int fn2_conv_packed_floats(const fn2_conv_desc* d, int ci_stride, size_t* floats);
FN2_API int fn2_conv_pack_weights(const fn2_conv_desc* d, int ci_stride,
                                  const float* caffe_weights_dev, float* packed_dev, void* stream);
FN2_API int fn2_conv_out_shape(const fn2_conv_desc* d, int H, int W, int* Ho, int* Wo);
/* Scratch the forward may use for this shape (split-K partials of small spatial maps); may be 0.  It may start at any 4-byte
 * boundary.  Passing a NULL / too small workspace is allowed: the kernel then runs unsplit. */
FN2_API int fn2_conv_workspace_bytes(const fn2_conv_desc* d, int N, int H, int W, size_t* bytes);
/* Host-side plan of the tensor-core engine for a layer shape (introspection; needs no GPU): plan8 = {NT (output channels per
 * tile; 0 = a shape the engine does not take), tile units, K steps per tile, small-Ci mode (0 plain K blocks, 1 tap groups,
 * 2 kernel rows), first split tile, K ranges per split tile (1 = unsplit), 0, 0}.  The tiles from the first split tile on
 * have their K loops cut into that many ranges, which run on different SMs: all tiles of a layer whose tile list cannot fill
 * the GPU, else the tiles of the last, partial wave.  The taps-on-N engine (mode 3) reports {-accumulator columns of the
 * widest pass, 0, K blocks, 3, passes, strips, W stages (0: the whole packed weight matrix resident in shared memory, else
 * the depth of the weight-stage ring), tiles between two flushes of the output-row ring}. */
FN2_API int fn2_conv_plan(const fn2_conv_desc* d, int N, int H, int W, int ci_stride, int32_t* plan8);
FN2_API int fn2_conv_forward(const fn2_conv_desc* d, const fn2_tensor* bottom,
                             const float* packed_weights_dev, const float* bias_dev,
                             const fn2_tensor* top, void* workspace, size_t workspace_bytes, void* stream);

/* Gradients (config 5, the FlowNet2-C training step): ConvolutionLayer / DeconvolutionLayer::Backward_gpu
 * (conv_layer.cu:26-58, deconv_layer.cu:26-55 -> base_conv_layer.cpp:352-395 backward_gpu_gemm, weight_gpu_gemm,
 * backward_gpu_bias).
 *   fn2_conv_backward_params : weight gradient in Caffe layout (conv [co][ci][kh][kw], deconv [ci][co][kh][kw]) and bias
 *                              gradient; accumulate != 0 adds to the existing diffs (Caffe accumulates parameter diffs).
 *   fn2_conv_backward_data_desc : the FORWARD operator that computes the gradient w.r.t. the bottom: a stride-1 convolution's
 *                              adjoint is the convolution with flipped + transposed weights (needs_flip = 1: derive them with
 *                              fn2_conv_flip_transpose_weights and pack as usual), a strided convolution's adjoint is the
 *                              deconvolution with the same weight blob (out_pad = the bottom rows / columns the forward
 *                              convolution's last window does not start at but still covers) and vice versa; run it with
 *                              fn2_conv_forward on the top diff: the result has exactly the bottom's shape. */
FN2_API int fn2_conv_backward_params_workspace_bytes(const fn2_conv_desc* d, int N, int H, int W, size_t* bytes);
/* Host-side plan of fn2_conv_backward_params for a layer shape (introspection; needs no GPU).  It reports the choice the layer
 * shape makes, not whether this process can run the tensor cores.  "Small" is the top diff of a convolution and the bottom of
 * a deconvolution, "big" the other map.  plan8 = {route (1 SIMT, 2 tensor cores), small channels per tile NT, big-map rows
 * per tap G, tap groups TG, big-channel tiles BT, small-channel tiles ST, K ranges per tile S (SIMT: pixel splits), bias
 * blocks (0 without a bias)}; the SIMT route leaves slots 1-5 at 0. */
FN2_API int fn2_conv_wgrad_plan(const fn2_conv_desc* d, int N, int H, int W, int32_t* plan8);
FN2_API int fn2_conv_backward_params(const fn2_conv_desc* d, const fn2_tensor* bottom, const fn2_tensor* top_diff,
                                     float* weight_diff_dev, float* bias_diff_dev, int accumulate, void* workspace,
                                     size_t workspace_bytes, void* stream);
FN2_API int fn2_conv_backward_data_desc(const fn2_conv_desc* d, int bottom_h, int bottom_w, fn2_conv_desc* out, int* needs_flip);
FN2_API int fn2_conv_flip_transpose_weights(const fn2_conv_desc* d, const float* caffe_weights_dev, float* derived_dev, void* stream);

/* Training-side neighbours of config 5 (SURVEY.md 8 "next" row 2).
 * L1Loss -- replaces L1LossLayer::Forward_gpu / Backward_gpu (l1loss_layer.cu:67-192; the CPU paths are NOT_IMPLEMENTED in the
 * reference, l1loss_layer.cpp:93-102).  bottom1 may be NULL (single-bottom form).  state_dev: 4 device floats the forward
 * writes and the backward reads: {loss, normalize_coeff, masked sum, not-NaN count}; loss_dev (may be NULL) also receives the
 * loss.  workspace: at least fn2_l1loss_workspace_bytes(N, H, W) bytes, 4-byte aligned; a NULL or smaller one returns
 * FN2_ERR_WORKSPACE.  The forward reduces its per-block partials in a fixed order: equal inputs give bit-identical state.  top_diff_dev: device scalar (the loss weight).  The backward recomputes the difference and the NaN / plateau masks from
 * the bottoms; a NULL diff pointer means "do not propagate to this bottom"; accumulate != 0 adds to the diff. */
typedef struct fn2_l1loss_desc {
    int32_t l2_per_location, l2_prescale_by_channels, normalize_by_num_entries;   /* L1LossParameter, caffe.proto:619-625 */
    float epsilon, plateau;
} fn2_l1loss_desc;
FN2_API int fn2_l1loss_workspace_bytes(int N, int H, int W, size_t* bytes);
FN2_API int fn2_l1loss_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_l1loss_desc* d, float* state_dev,
                               float* loss_dev, void* workspace, size_t workspace_bytes, void* stream);
FN2_API int fn2_l1loss_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_l1loss_desc* d,
                                const float* state_dev, const float* top_diff_dev, const fn2_tensor* bottom0_diff,
                                const fn2_tensor* bottom1_diff, int accumulate0, int accumulate1, void* stream);
/* Downsample -- replaces DownsampleFeatures (downsample_layer.cu:15-80): NaN-aware weighted average around the rounded source
 * position; equal sizes copy (the reference shares the data, downsample_layer.cpp:55-58). */
FN2_API int fn2_downsample_forward(const fn2_tensor* bottom, const fn2_tensor* top, void* stream);
/* FlowAugmentation -- replaces WarpData (flow_augmentation_layer.cu:24-66).  mats: device arrays, 6 floats per sample in NAME
 * order t0..t5 as for fn2_spatial_augmentation; the second one already inverted (tTransMat::inverse,
 * augmentation_layer_base.cpp:51-68). */
FN2_API int fn2_flow_augmentation(const fn2_tensor* flow, const fn2_tensor* top, const float* mats1_dev,
                                  const float* mats2_inverse_dev, void* stream);

/* ------------------------------------------------------------------------------------ */
/* Glue: ReLU (relu_layer.cu:9-14), Eltwise SUM with coeffs (eltwise_layer.cu),           */
/* ChannelNorm (channel_norm_layer.cu:17-30), strided copy (Concat concat_layer.cu,        */
/* layout conversion), axpby, ReLU backward, fill.  Bit-exact on every layout.            */
/* ------------------------------------------------------------------------------------ */
FN2_API int fn2_relu_forward(const fn2_tensor* bottom, const fn2_tensor* top, float negative_slope,
                             void* stream);
FN2_API int fn2_eltwise_sum(const fn2_tensor* const* bottoms, const float* coeffs, int num_bottoms,
                            const fn2_tensor* top, void* stream);
FN2_API int fn2_channel_norm_forward(const fn2_tensor* bottom, const fn2_tensor* top, void* stream);
FN2_API int fn2_copy(const fn2_tensor* src, const fn2_tensor* dst, void* stream);
/* y = alpha * x + beta * y over strided views (gradient accumulation for blobs with several consumers; Eltwise / Concat /
 * Split backward: eltwise_layer.cu, concat_layer.cu, split_layer.cu).  beta == 0 overwrites without reading y. */
FN2_API int fn2_axpby(const fn2_tensor* x, float alpha, const fn2_tensor* y, float beta, void* stream);
/* ReLULayer::Backward_gpu (relu_layer.cu:29-38) from the TOP data (valid for in-place use with negative_slope >= 0):
 * g = top_diff * (top_data > 0 ? 1 : negative_slope), rounded; bottom_diff = accumulate ? bottom_diff + g : g. */
FN2_API int fn2_relu_backward(const fn2_tensor* top_data, const fn2_tensor* top_diff, const fn2_tensor* bottom_diff,
                              float negative_slope, int accumulate, void* stream);
FN2_API int fn2_fill(const fn2_tensor* dst, float value, void* stream);

/* ------------------------------------------------------------------------------------ */
/* Net -- replaces caffe::Net<float> as used by scripts/run-flownet.py:64-98              */
/*   (Net::Init net.cpp:40-286, CopyTrainedLayersFrom :752-802, ForwardFromTo :546-557).  */
/* ------------------------------------------------------------------------------------ */
typedef struct fn2_net fn2_net;

/* Parse a deploy prototxt (text format, $VARS$ already substituted) and build the graph on
 * the current CUDA device.  phase: 0 TRAIN, 1 TEST. */
FN2_API int fn2_net_create(const char* prototxt_text, int phase, fn2_net** out);
/* Same, overriding dim 0 of every Input shape with `batch` (> 0): the released deploy templates
 * say `dim: 1`; frame-batch sharding runs B pairs per replica. */
FN2_API int fn2_net_create_batch(const char* prototxt_text, int phase, int batch, fn2_net** out);
FN2_API void fn2_net_destroy(fn2_net* net);
/* Load weights from the bytes of a .caffemodel (binary NetParameter). */
FN2_API int fn2_net_copy_trained_layers(fn2_net* net, const void* caffemodel, size_t bytes);
/* Same, with source layer X filling target layer prefix + X (FlowNet2's stage hand-over: a FlowNet2-C caffemodel into the
 * net1_ layers of FlowNet2-CS, FlowNet2-SD into the netsd_ layers of FlowNet2).  Source layers with no target are ignored. */
FN2_API int fn2_net_copy_trained_layers_prefixed(fn2_net* net, const void* caffemodel, size_t bytes, const char* prefix);
/* Serialise current parameters as a .caffemodel.  Call with buf==NULL to query the size. */
FN2_API int fn2_net_to_caffemodel(fn2_net* net, void* buf, size_t* bytes);
/* Fill parameters from the prototxt's fillers (deterministic given seed); used for synthetic
 * benchmarks where no .caffemodel exists. */
FN2_API int fn2_net_fill_params(fn2_net* net, uint64_t seed);
/* Contiguous device arena holding every layer parameter (for one ncclBroadcast). */
FN2_API int fn2_net_param_arena(fn2_net* net, void** dev_ptr, size_t* bytes);
/* Re-derive packed weights after the arena was overwritten (e.g. by a broadcast). */
FN2_API int fn2_net_params_changed(fn2_net* net);

FN2_API int fn2_net_num_inputs(fn2_net* net);
FN2_API const char* fn2_net_input_name(fn2_net* net, int i);
FN2_API int fn2_net_num_outputs(fn2_net* net);
FN2_API const char* fn2_net_output_name(fn2_net* net, int i);
FN2_API int fn2_net_num_blobs(fn2_net* net);
FN2_API const char* fn2_net_blob_name(fn2_net* net, int i);
FN2_API int fn2_net_num_layers(fn2_net* net);
FN2_API const char* fn2_net_layer_name(fn2_net* net, int i);
FN2_API const char* fn2_net_layer_type(fn2_net* net, int i);
FN2_API int fn2_net_blob_shape(fn2_net* net, const char* blob, int shape[4]);

/* Host NCHW <-> blob.  set: H2D copy + layout conversion, asynchronous on the net's stream
 * (host buffer must stay valid until fn2_net_sync; pinned memory makes it truly async).
 * get: device->host, synchronises. */
FN2_API int fn2_net_set_input(fn2_net* net, const char* blob, const float* host_nchw);
FN2_API int fn2_net_get_blob(fn2_net* net, const char* blob, float* host_nchw);
/* Same with device NCHW buffers (no host round trip). */
FN2_API int fn2_net_set_input_device(fn2_net* net, const char* blob, const float* dev_nchw);
FN2_API int fn2_net_get_blob_device(fn2_net* net, const char* blob, float* dev_nchw);

/* Net::Forward.  Asynchronous on the net's stream; replayed from a CUDA graph when possible. */
FN2_API int fn2_net_forward(fn2_net* net);
FN2_API int fn2_net_sync(fn2_net* net);
/* Net::Backward (net.cpp:640-655): gradients from the loss tops (LayerParameter.loss_weight) and from every blob given a
 * gradient through fn2_net_set_diff, down to the parameters.  Parameter gradients ACCUMULATE like the reference's:
 * fn2_net_clear_param_diffs is Net::ClearParamDiffs (net.cpp:935-955), what Solver::Step calls before every iteration.
 * A fused conv+ReLU differentiates in place on its top diff, so a seed set with fn2_net_set_diff is consumed by the call.
 * fn2_net_param_diff_arena: all parameter gradients as ONE contiguous device range laid out like fn2_net_param_arena (a single
 * all-reduce makes the step data parallel). */
FN2_API int fn2_net_backward(fn2_net* net);
FN2_API int fn2_net_clear_param_diffs(fn2_net* net);
FN2_API int fn2_net_set_diff(fn2_net* net, const char* blob, const float* host_nchw);
FN2_API int fn2_net_get_diff(fn2_net* net, const char* blob, float* host_nchw);
FN2_API int fn2_net_param_diff_arena(fn2_net* net, void** dev_ptr, size_t* bytes);
/* The smallest range of that arena covering every parameter the backward pass writes (lr_mult != 0 in a layer that needs
 * backward).  A stage trained on top of frozen predecessors all-reduces only this range; the rest of the arena stays zero. */
FN2_API int fn2_net_trainable_diff_span(fn2_net* net, void** dev_ptr, size_t* bytes);
FN2_API int fn2_net_param_shape(fn2_net* net, const char* layer, int index, int shape[4]);
FN2_API int fn2_net_get_param(fn2_net* net, const char* layer, int index, int diff, float* host);
FN2_API int fn2_net_launches_per_backward(fn2_net* net);
/* 1 if Net::Backward runs this layer (net.cpp layer_need_backward_), 0 if not, -1 on a bad index */
FN2_API int fn2_net_layer_need_backward(fn2_net* net, int layer);
FN2_API void* fn2_net_stream(fn2_net* net);
/* Per-layer device time of one forward pass in the style of `caffe time`
 * (tools/caffe.cpp:346-385).  ms must hold fn2_net_num_layers() floats. */
FN2_API int fn2_net_time_layers(fn2_net* net, float* ms);
/* Algorithmic flops / bytes of one layer's forward (roofline reporting; SURVEY.md 8d). */
FN2_API int fn2_net_layer_work(fn2_net* net, int layer, double* flops, double* bytes);
/* Kernels launched by one forward pass. */
FN2_API int fn2_net_launches_per_forward(fn2_net* net);
/* 1 once the forward pass is replayed from a captured CUDA graph (0 while it still runs eagerly, e.g. a DataAugmentation
 * layer whose running mean is still being updated: data_augmentation_layer.cu:600-608). */
FN2_API int fn2_net_graph_active(fn2_net* net);

/* Host-only parser checks (no GPU needed; used by the CPU test-suite).
 * fn2_proto_canonical: parse a prototxt with the engine's text-format parser (after the legacy
 * `input:` upgrade) and print it back in canonical text format.  fn2_caffemodel_summary: parse a
 * .caffemodel and print one line per layer: name, type, then per blob shape and a checksum.
 * Both follow the size-query convention: call with out==NULL to get the needed size in *bytes. */
FN2_API int fn2_proto_canonical(const char* prototxt_text, char* out, size_t* bytes);
/* Coefficient sampling of DataAugmentationLayer (host logic only, no GPU): parses a prototxt fragment that contains a
 * DataAugmentation layer and draws the coefficients of `num` items exactly as the layer's forward does at iteration num_iter
 * (generators, discount schedule, 4-corner validity resampling: augmentation_layer_base.cpp:73-336,
 * data_augmentation_layer.cu:372-449).  coeffs_out: num x 42 floats in the array form of the parameter blob
 * (fields with default 1 as logarithms, augmentation_layer_base.cpp:352-365). */
FN2_API int fn2_aug_sample(const char* layer_prototxt, unsigned int seed, int num, int width, int height, float num_iter,
                           float* coeffs_out);
FN2_API int fn2_caffemodel_summary(const void* caffemodel, size_t n, char* out, size_t* bytes);
/* HDF5 weight files (.caffemodel.h5, net.cpp:823-870; hdf5_load_nd_dataset util/hdf5.cpp:20-76).  fn2_net_copy_trained_layers
 * recognises them by their signature.  fn2_hdf5_summary (host only): one line per dataset of the file: path, f32/f64, shape, count,
 * sum, first and last value.  The reader covers what libhdf5 writes for such files by default (superblock 0, symbol-table groups,
 * contiguous little-endian float datasets); chunked / gzip datasets and new-style groups return FN2_ERR_PARSE with the reason. */
FN2_API int fn2_hdf5_summary(const void* h5, size_t n, char* out, size_t* bytes);
/* Net::ToHDF5 (net.cpp:905-960): the weights as /data/<layer>/<index> float32 datasets (superblock 0, symbol-table groups, contiguous
 * data: the subset fn2_hdf5_summary / fn2_net_copy_trained_layers read).  Size-query convention (out / buf == NULL).
 * fn2_caffemodel_to_hdf5 converts a binary .caffemodel on the host (no GPU needed). */
FN2_API int fn2_caffemodel_to_hdf5(const void* caffemodel, size_t n, void* out, size_t* bytes);
FN2_API int fn2_net_to_hdf5(fn2_net* net, void* buf, size_t* bytes);

/* .flo files (util/output.cpp:16-64): "PIEH", int32 w, int32 h, interleaved (u,v) fp32. */
FN2_API int fn2_write_flo(const char* path, const float* flow_nchw_2hw, int h, int w);
FN2_API int fn2_read_flo(const char* path, float* flow_nchw_2hw, int* h, int* w, size_t capacity_floats);

#ifdef __cplusplus
}
#endif
#endif /* FN2_H_ */
