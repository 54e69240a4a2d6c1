// Streaming (HBM-bound) layers: FlowWarp, Resample, DataAugmentation kernels, ChannelNorm, the warp block, and the
// element-wise ops of the forward and backward passes (ReLU and its backward, Eltwise SUM, y = alpha*x + beta*y, strided
// copy and fill), the conversion of 8-bit frames into an input blob, the flow-file conversions, the flow colour coding and the
// forward-backward occlusion check.
//
// This translation unit is compiled with -fmad=false: every expression below is evaluated
// with separately rounded multiplies and adds in the order written, which is also how the CPU
// oracle (oracle/oracle.c, -ffp-contract=off) evaluates the reference arithmetic, so these
// layers are compared bit-for-bit.  They are bandwidth-bound; FMA contraction buys nothing.
//
// All kernels take strided tensor views (fn2::T4) so the same code serves the reference's NCHW
// blobs (drop-in use) and the engine's NHWC activations / concat views.  The per-pixel kernels run the grid-stride loops of
// fn2_common.cuh.  The warp block is built from the device functions of the stand-alone FlowWarp, Resample, Eltwise and
// ChannelNorm kernels: the compiler inlines the same functions in both places, so its tops are bit-identical to the layer chain's.
#include <math.h>
#include <algorithm>
#include <cfloat>
#include <initializer_list>

#include "fn2_common.cuh"
#include "../../include/fn2_frames.h"
#include "../../include/fn2_flow.h"

namespace fn2 {

// ---------------------------------------------------------------------------------------------
// FlowWarp forward.  Reference: flow_warp_layer.cpp:57-117 (CPU), flow_warp_layer.cu:59-122.
// One thread per output pixel; the reference's NCHW->NHWC transpose pass (.cu:24-52) is not
// needed: taps are read straight from the strided view.
// ---------------------------------------------------------------------------------------------
// Bilinear taps of the image point (x + u, y + v): inside tells whether it lies in the image (else the output is the fill
// value); then the four weights and the offsets of the four taps' channel 0.
struct WarpTaps {
    bool inside;
    float cTL, cTR, cBL, cBR;
    long long oTL, oTR, oBL, oBR;
};
__device__ __forceinline__ WarpTaps warp_taps(const T4& img, int n, int y, int x, float u, float v) {
    WarpTaps t;
    const float x2 = (float)x + u;
    const float y2 = (float)y + v;
    const int width = img.w, height = img.h;
    t.inside = x2 >= 0 && y2 >= 0 && x2 < width && y2 < height;      // flow_warp_layer.cpp:86
    if (!t.inside) return t;
    const int ix2_L = (int)x2;
    const int iy2_T = (int)y2;
    const int ix2_R = min(ix2_L + 1, width - 1);
    const int iy2_B = min(iy2_T + 1, height - 1);
    const float alpha = x2 - ix2_L;
    const float beta = y2 - iy2_T;
    t.cTL = (1 - alpha) * (1 - beta);
    t.cTR = alpha * (1 - beta);
    t.cBL = (1 - alpha) * beta;
    t.cBR = alpha * beta;
    t.oTL = img.off(n, 0, iy2_T, ix2_L); t.oTR = img.off(n, 0, iy2_T, ix2_R);
    t.oBL = img.off(n, 0, iy2_B, ix2_L); t.oBR = img.off(n, 0, iy2_B, ix2_R);
    return t;
}
__device__ __forceinline__ float warp_mix(const WarpTaps& t, float TL, float TR, float BL, float BR) {
    return ((t.cTL * TL + t.cTR * TR) + t.cBL * BL) + t.cBR * BR;
}
// Warped value of channel c (strided form)
__device__ __forceinline__ float warp_channel(const WarpTaps& t, const T4& img, int c) {
    const long long o = c * img.sc;
    return warp_mix(t, __ldg(img.p + t.oTL + o), __ldg(img.p + t.oTR + o), __ldg(img.p + t.oBL + o), __ldg(img.p + t.oBR + o));
}
// Warped values of channels 0..3 (float4 form: every pixel is one 16-byte group, one 128-bit load per tap)
__device__ __forceinline__ void warp_group(const WarpTaps& t, const T4& img, float v[4]) {
    const float4 TL = __ldg(reinterpret_cast<const float4*>(img.p + t.oTL)), TR = __ldg(reinterpret_cast<const float4*>(img.p + t.oTR));
    const float4 BL = __ldg(reinterpret_cast<const float4*>(img.p + t.oBL)), BR = __ldg(reinterpret_cast<const float4*>(img.p + t.oBR));
    v[0] = warp_mix(t, TL.x, TR.x, BL.x, BR.x);
    v[1] = warp_mix(t, TL.y, TR.y, BL.y, BR.y);
    v[2] = warp_mix(t, TL.z, TR.z, BL.z, BR.z);
    v[3] = warp_mix(t, TL.w, TR.w, BL.w, BR.w);
}

// F4: every image pixel is one float4 group (px_one_group).
template <bool F4>
__global__ void flow_warp_fwd_kernel(T4 img, T4 flow, T4 out, float fill) {
    for_each_pixel(out.n, out.h, out.w, [&](int n, int y, int x) {
        const WarpTaps t = warp_taps(img, n, y, x, flow.p[flow.off(n, 0, y, x)], flow.p[flow.off(n, 1, y, x)]);
        if (F4 && t.inside) {
            float v[4];
            warp_group(t, img, v);
#pragma unroll
            for (int c = 0; c < 4; c++)
                if (c < img.c) out.p[out.off(n, c, y, x)] = v[c];
        } else {
            for (int c = 0; c < img.c; c++) out.p[out.off(n, c, y, x)] = t.inside ? warp_channel(t, img, c) : fill;
        }
    });
}

// FlowWarp backward.  Reference: flow_warp_layer.cu:170-229 / flow_warp_layer.cpp:120-198.
// image_diff must be zero-filled by the caller side (done in the entry point).  Scatter via
// atomicAdd exactly like the reference (order-nondeterministic in the last ulp).
__global__ void flow_warp_bwd_kernel(T4 img, T4 flow, T4 wdiff, T4 idiff, T4 fdiff) {
    for_each_pixel(img.n, img.h, img.w, [&](int n, int y, int x) {
        const float x2 = (float)x + flow.p[flow.off(n, 0, y, x)];
        const float y2 = (float)y + flow.p[flow.off(n, 1, y, x)];
        const int width = img.w, height = img.h;
        float du = 0.f, dv = 0.f;
        if (x2 >= 0 && y2 >= 0 && x2 < width && y2 < height) {
            const int L = (int)x2, T = (int)y2;
            const int R = min(L + 1, width - 1), B = min(T + 1, height - 1);
            const float alpha = x2 - L, beta = y2 - T;
            const float gy = B - y2, gx = R - x2;
            for (int c = 0; c < img.c; c++) {
                const float wd = wdiff.p[wdiff.off(n, c, y, x)];
                atomicAdd(idiff.p + idiff.off(n, c, T, L), wd * (1 - alpha) * (1 - beta));
                atomicAdd(idiff.p + idiff.off(n, c, T, R), wd * alpha * (1 - beta));
                atomicAdd(idiff.p + idiff.off(n, c, B, L), wd * (1 - alpha) * beta);
                atomicAdd(idiff.p + idiff.off(n, c, B, R), wd * alpha * beta);
                const float TL = img.p[img.off(n, c, T, L)], TR = img.p[img.off(n, c, T, R)];
                const float BL = img.p[img.off(n, c, B, L)], BR = img.p[img.off(n, c, B, R)];
                float tu = 0; tu += gy * (TR - TL); tu += (1 - gy) * (BR - BL);
                float tv = 0; tv += gx * (BL - TL); tv += (1 - gx) * (BR - TR);
                du += wd * tu;
                dv += wd * tv;
            }
        }
        fdiff.p[fdiff.off(n, 0, y, x)] = du;
        fdiff.p[fdiff.off(n, 1, y, x)] = dv;
    });
}

// ---------------------------------------------------------------------------------------------
// Resample.  Reference: resample_layer.cu:14-33 (filters), :40-95 InterpolationKernel,
// :98-125 NearestNeighborKernel.  Including the swapped half-pixel offsets (:62-63).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float bicubicCoeff(float x_) {
    float x = fabsf(x_);
    if (x <= 1.0f) return x * x * (1.5f * x - 2.5f) + 1.0f;
    else if (x < 2.0f) return x * (x * (-0.5f * x + 2.5f) - 4.0f) + 2.0f;
    else return 0.0f;
}
__device__ __forceinline__ float triangleCoeff(float x) {
    if (-1 <= x && x < 0) return x + 1;
    if (0 <= x && x <= 1) return 1 - x;
    return 0;
}
// Source coordinate of output coordinate o; f is this axis's in/out ratio, g the other axis's (the swapped offsets).
__device__ __forceinline__ float resample_src(int o, float f, float g) { return (o * f + g / 2.0f) - 0.5f; }

// Filter window of TYPE 2 (triangle) or 3 (cubic) around the source point (x_in, y_in).  One thread per output pixel, all
// channels: the filter weights depend on the pixel only, and every channel accumulates its taps in the reference's order
// (y outer, x inner), so each channel's result is bit-identical to the per-element formulation.  The filters vanish outside
// |ax*dx| < support, so only the taps of the reference's window that can carry weight are visited, and taps whose weight is
// exactly zero are skipped: sum + 0*v == sum and wsum + 0 == wsum for finite v (the triangle filter of an up-sampling has 21
// zero taps out of 25).
template <int TYPE> struct ResampleWindow {
    static constexpr int MAXT = 8;
    float x_in, y_in, ax, ay;
    int xl, xh, yl, yh;
    bool pre;                     // at most MAXT columns: tx holds the x factors
    float tx[MAXT];
    __device__ static float coeff(float d) { return (TYPE == 3) ? bicubicCoeff(d) : triangleCoeff(d); }
    // (ax * cx) * ay of column x: the first two products of the reference's weight expression
    __device__ float xfactor(int x) const { return (ax * coeff(ax * (x_in - x))) * ay; }
    __device__ ResampleWindow(float x_in_, float y_in_, float fx, float fy, int antialias) : x_in(x_in_), y_in(y_in_) {
        const int kernel_width = (TYPE == 3) ? 4 : 2;
        ax = 1.0f / (antialias ? fx : 1.0f);
        ay = 1.0f / (antialias ? fy : 1.0f);
        const int x_in_round = (int)roundf(x_in);
        const int y_in_round = (int)roundf(y_in);
        const int rx = (fx < 1.0f) ? 2 : (int)ceilf((float)kernel_width / ax);
        const int ry = (fy < 1.0f) ? 2 : (int)ceilf((float)kernel_width / ay);
        const float sup = (TYPE == 3) ? 2.0f : 1.0f;
        xl = max(x_in_round - rx, (int)floorf(x_in - sup / ax)); xh = min(x_in_round + rx, (int)ceilf(x_in + sup / ax));
        yl = max(y_in_round - ry, (int)floorf(y_in - sup / ay)); yh = min(y_in_round + ry, (int)ceilf(y_in + sup / ay));
        pre = xh - xl < MAXT;
        if (pre) {
#pragma unroll
            for (int k = 0; k < MAXT; k++) tx[k] = xfactor(xl + k);
        }
    }
    // sum[j] += w * in(n, c0 + j, y, x) over the window's taps for j < nc; returns the sum of the weights
    __device__ float accumulate(const T4& in, int n, int c0, int nc, float sum[4]) const {
        float wsum = 0;
        for (int y = yl; y <= yh; y++) {
            if (y < 0 || y >= in.h) continue;
            const float cy = coeff(ay * (y_in - y));
            for (int x0 = xl; x0 <= xh; x0 += MAXT) {     // one pass when pre
#pragma unroll
                for (int k = 0; k < MAXT; k++) {
                    const int x = x0 + k;
                    if (x > xh) break;
                    if (x < 0 || x >= in.w) continue;
                    const float w = (pre ? tx[k] : xfactor(x)) * cy;
                    if (w == 0.f) continue;
                    const float* ip = in.p + in.off(n, c0, y, x);
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (j < nc) sum[j] = sum[j] + w * __ldg(ip + (long long)j * in.sc);
                    wsum += w;
                }
            }
        }
        return wsum;
    }
    __device__ static float value(float sum, float wsum) { return (!wsum) ? 0 : (sum / wsum); }
};

template <int TYPE>   // 1 nearest, 2 linear(triangle), 3 cubic
__global__ void resample_kernel(T4 in, T4 out, float fx, float fy, int antialias) {
    for_each_pixel(out.n, out.h, out.w, [&](int n, int y_out, int x_out) {
        const float x_in = resample_src(x_out, fx, fy), y_in = resample_src(y_out, fy, fx);
        if constexpr (TYPE == 1) {
            // the reference does not clamp (resample_layer.cu:120-123) and can read out of
            // bounds; clamp instead (documented deviation)
            const int xr = min(max((int)roundf(x_in), 0), in.w - 1);
            const int yr = min(max((int)roundf(y_in), 0), in.h - 1);
            for (int c = 0; c < out.c; c++) out.p[out.off(n, c, y_out, x_out)] = in.p[in.off(n, c, yr, xr)];
        } else {
            const ResampleWindow<TYPE> win(x_in, y_in, fx, fy, antialias);
            for (int c0 = 0; c0 < out.c; c0 += 4) {
                const int nc = min(4, out.c - c0);
                float sum[4] = {0.f, 0.f, 0.f, 0.f};
                const float wsum = win.accumulate(in, n, c0, nc, sum);
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (j < nc) out.p[out.off(n, c0 + j, y_out, x_out)] = ResampleWindow<TYPE>::value(sum[j], wsum);
            }
        }
    });
}

// ---------------------------------------------------------------------------------------------
// ChannelNorm (channel_norm_layer.cu:17-30) and the Eltwise SUM term (eltwise_layer.cpp:59-65).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float eltwise_term(float acc, float k, float v) { return acc + k * v; }
// ChannelNorm's running sum of squares; the output is its square root
__device__ __forceinline__ float norm_term(float norm, float v) { return norm + v * v; }

// F4: every input pixel is one float4 group (px_one_group).
template <bool F4>
__global__ void channel_norm_kernel(T4 in, T4 out) {
    for_each_pixel(in.n, in.h, in.w, [&](int n, int y, int x) {
        float norm = 0;
        if (F4) {
            const float4 q = *reinterpret_cast<const float4*>(in.p + in.off(n, 0, y, x));
            const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int c = 0; c < 4; c++) if (c < in.c) norm = norm_term(norm, v[c]);
        } else {
            for (int c = 0; c < in.c; c++) norm = norm_term(norm, in.p[in.off(n, c, y, x)]);
        }
        out.p[out.off(n, 0, y, x)] = sqrtf(norm);
    });
}

// ---------------------------------------------------------------------------------------------
// Warp block between two stacked networks (FlowNet2-CSS / FlowNet2): the chain
//   Resample(LINEAR, up-sampling) -> FlowWarp -> Eltwise(img0 - warped) -> ChannelNorm, and Eltwise(coeff * flow)
// as ONE pass: one thread per full-resolution pixel computes the interpolated flow, samples the second image, and writes all
// five tops (most of them channel ranges of the next network's input concat).  Every value comes from the device functions
// of the stand-alone kernels above (ResampleWindow<2> without antialias on channels 0-1, warp_taps / warp_group /
// warp_channel, eltwise_term with coefficients (1, -1) resp. (coeff), norm_term), so the tops are bit-identical to the layer
// chain's.  F4: every image1 pixel is one float4 group (px_one_group).
// ---------------------------------------------------------------------------------------------
template <bool F4>
__global__ void warp_block_kernel(T4 fin, T4 img0, T4 img1, T4 ffull, T4 warped, T4 err, T4 errn, T4 fscaled, float fx, float fy,
                                  float coeff, float fill) {
    for_each_pixel(ffull.n, ffull.h, ffull.w, [&](int n, int y, int x) {
        const ResampleWindow<2> win(resample_src(x, fx, fy), resample_src(y, fy, fx), fx, fy, 0);
        float f[4] = {0.f, 0.f, 0.f, 0.f};
        const float wsum = win.accumulate(fin, n, 0, 2, f);
#pragma unroll
        for (int c = 0; c < 2; c++) {
            f[c] = ResampleWindow<2>::value(f[c], wsum);
            ffull.p[ffull.off(n, c, y, x)] = f[c];
            fscaled.p[fscaled.off(n, c, y, x)] = eltwise_term(0.f, coeff, f[c]);
        }
        const WarpTaps t = warp_taps(img1, n, y, x, f[0], f[1]);
        float wv[4] = {fill, fill, fill, fill};
        if (t.inside && F4) warp_group(t, img1, wv);
        if (t.inside && !F4) {
#pragma unroll
            for (int c = 0; c < 4; c++)
                if (c < img1.c) wv[c] = warp_channel(t, img1, c);
        }
        float norm = 0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
            if (c >= img1.c) break;
            warped.p[warped.off(n, c, y, x)] = wv[c];
            const float e = eltwise_term(eltwise_term(0.f, 1.0f, img0.p[img0.off(n, c, y, x)]), -1.0f, wv[c]);
            err.p[err.off(n, c, y, x)] = e;
            norm = norm_term(norm, e);
        }
        errn.p[errn.off(n, 0, y, x)] = sqrtf(norm);
    });
}

// ---------------------------------------------------------------------------------------------
// DataAugmentation device kernels.
// SpatialAugmentation: data_augmentation_layer.cu:25-70.  The reference forms the flat source
// index in float arithmetic (:52), exact while the blob has < 2^24 elements; integer arithmetic
// here (identical in that range).  The min(idx, src_count) clamps of :53-55 can never trigger
// for width,height >= 2 because of the dim-1.05 clamp.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float clampf(float f, float a, float b) { return fmaxf(a, fminf(f, b)); }

__global__ void spatial_aug_kernel(T4 src, T4 dst, const float* __restrict__ mats) {
    for_each_pixel(dst.n, dst.h, dst.w, [&](int n, int y, int x) {
        const float* m = mats + 6 * n;
        float xpos = (x * m[0] + y * m[2]) + m[4];
        float ypos = (x * m[1] + y * m[3]) + m[5];
        xpos = clampf(xpos, 0.0f, (float)(src.w) - 1.05f);
        ypos = clampf(ypos, 0.0f, (float)(src.h) - 1.05f);
        const float tlx = floorf(xpos);
        const float tly = floorf(ypos);
        const int ix = (int)tlx, iy = (int)tly;
        const float xdist = xpos - tlx;
        const float ydist = ypos - tly;
        const float cTL = (1 - xdist) * (1 - ydist), cBR = xdist * ydist;
        const float cBL = (1 - xdist) * ydist, cTR = xdist * (1 - ydist);
        const long long oTL = src.off(n, 0, iy, ix);
        for (int c = 0; c < src.c; c++) {
            const float* s = src.p + oTL + c * src.sc;
            const float TL = __ldg(s), TR = __ldg(s + src.sw);
            const float BL = __ldg(s + src.sh), BR = __ldg(s + src.sh + src.sw);
            // term order TL, BR, BL, TR (data_augmentation_layer.cu:62-65)
            dst.p[dst.off(n, c, y, x)] = ((cTL * TL + cBR * BR) + cBL * BL) + cTR * TR;
        }
    });
}

// ColorContrastAugmentation: data_augmentation_layer.cu:73-117 (in place, 3 channels).
__global__ void color_contrast_kernel(T4 d, const float* __restrict__ chroma, float max_multiplier) {
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const float* ch = chroma + 6 * n;
        float rgb[3];
        float mean_in = 0, mean_out = 0;
        for (int c = 0; c < 3; c++) {
            rgb[c] = d.p[d.off(n, c, y, x)];
            mean_in += rgb[c];
            rgb[c] *= ch[3 + c];
            mean_out += rgb[c];
        }
        const float brightness_coeff = mean_in / (mean_out + 0.01f);
        for (int c = 0; c < 3; c++) {
            float v = clampf(rgb[c] * brightness_coeff, 0.f, 1.f);
            v = powf(v, ch[0]);
            v = v + ch[1];
            v = 0.5f + (v - 0.5f) * ch[2];
            d.p[d.off(n, c, y, x)] = clampf(v, 0.f, max_multiplier);
        }
    });
}

// Running mean update: data_augmentation_layer.cu:600-607 (scal, axpy per sample, scal).  One thread per (c, y, x).
__global__ void mean_update_kernel(T4 top, T4 mean, float num_iter) {
    for_each_pixel(top.c, top.h, top.w, [&](int c, int y, int x) {
        float* mp = mean.p + mean.off(0, c, y, x);
        float m = *mp * (num_iter - 1.0f);
        const float inv = 1.0f / (float)top.n;
        for (int n = 0; n < top.n; n++) m = m + inv * top.p[top.off(n, c, y, x)];
        *mp = m * (1.0f / num_iter);
    });
}
// Per-channel average of the mean image (caffe_gpu_gemv with ones, :608); one CTA per channel,
// double accumulation (the cuBLAS order is unpinned).
__global__ void mean_per_channel_kernel(T4 mean, float* __restrict__ mean_pc) {
    const int c = blockIdx.x;
    const int area = mean.h * mean.w;
    double acc = 0;
    for (int i = threadIdx.x; i < area; i += blockDim.x)
        acc += (double)mean.p[mean.off(0, c, i / mean.w, i % mean.w)];
    __shared__ double sh[256];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) mean_pc[c] = (float)((1.0 / (double)area) * sh[0]);
}
// Mean subtraction :610-634.
__global__ void mean_subtract_kernel(T4 top, T4 mean, const float* __restrict__ mean_pc, int per_pixel) {
    for_each_element(top, [&](Idx4 e, long long) {
        const float m = per_pixel ? mean.p[mean.off(0, e.c, e.y, e.x)] : mean_pc[e.c];
        float* t = top.p + top.off(e.n, e.c, e.y, e.x);
        *t = *t - m;
    });
}

// Tiled transpose copy between a channel-planar side and a channel-fast side: 32 pixels x 32
// channels per tile through shared memory so that both global sides are coalesced.
__global__ void copy_transpose_kernel(T4 src, T4 dst, int src_cfast) {
    __shared__ float tile[32][33];          // [channel][pixel]
    const long long hw = (long long)dst.h * dst.w;
    const int n = blockIdx.z;
    const long long p0 = (long long)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        // the fast thread index follows the source's contiguous dimension
        const int ci = src_cfast ? tx : j;
        const int pi = src_cfast ? j : tx;
        const long long p = p0 + pi;
        if (c0 + ci < dst.c && p < hw)
            tile[ci][pi] = src.p[src.off(n, c0 + ci, (int)(p / dst.w), (int)(p % dst.w))];
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        // ... and the destination's contiguous dimension on the way out
        const int ci = src_cfast ? j : tx;
        const int pi = src_cfast ? tx : j;
        const long long p = p0 + pi;
        if (c0 + ci < dst.c && p < hw)
            dst.p[dst.off(n, c0 + ci, (int)(p / dst.w), (int)(p % dst.w))] = tile[ci][pi];
    }
}

// ---------------------------------------------------------------------------------------------
// Element-wise ops: ReLU (relu_layer.cu:9-14) and its backward (relu_layer.cu:29-38), Eltwise SUM (eltwise_layer.cpp:59-65),
// y = alpha*x + beta*y, copy and fill.  Each op is a functor over its views that computes one float4 of lanes at a place
// `at` and stores them; ew_run picks one of two routes for it:
//   * channel groups, when every view the op touches is channel-fast and pixel-linear (T4::is_nhwc: every NHWC blob and
//     every concat child): thread = (pixel p, channels c0..c0+3), each view's lanes at p * sw + c0, float4 where the view
//     allows (vr below);
//   * strided, otherwise: thread = one element, in lane x; channel-fastest when the destination is channel-fast, else
//     width-fastest.
// Both routes evaluate the same expression per element, so they agree bit for bit.
//
// vr: the view may be READ as float4 groups (lanes beyond C are padding or a neighbour's channels -- read, never used).
// WRITES never touch a lane beyond C: a view cannot tell whether those lanes are its own padding or a sibling's channels
// inside a zero-copy Concat parent (a 2-channel child of a 2+2 parent has the same strides as a dense 2-channel blob), so the
// tail group is stored lane by lane; padding stays zero from the allocation.
// ---------------------------------------------------------------------------------------------
struct PxView { T4 t; int vr; };
static PxView px_view(const T4& t) { return {t, t.px_float4_groups()}; }
__device__ __forceinline__ float4 px_load(const PxView& v, long long o, int c0) {
    if (v.vr) return *reinterpret_cast<const float4*>(v.t.p + o + c0);
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c0 + 0 < v.t.c) r.x = v.t.p[o + c0 + 0];
    if (c0 + 1 < v.t.c) r.y = v.t.p[o + c0 + 1];
    if (c0 + 2 < v.t.c) r.z = v.t.p[o + c0 + 2];
    if (c0 + 3 < v.t.c) r.w = v.t.p[o + c0 + 3];
    return r;
}
__device__ __forceinline__ void px_store(const PxView& v, long long o, int c0, float4 r) {
    if (v.vr && c0 + 4 <= v.t.c) { *reinterpret_cast<float4*>(v.t.p + o + c0) = r; return; }
    if (v.vr && c0 + 2 == v.t.c) { *reinterpret_cast<float2*>(v.t.p + o + c0) = make_float2(r.x, r.y); return; }   // 2-channel flows
    if (c0 + 0 < v.t.c) v.t.p[o + c0 + 0] = r.x;
    if (c0 + 1 < v.t.c) v.t.p[o + c0 + 1] = r.y;
    if (c0 + 2 < v.t.c) v.t.p[o + c0 + 2] = r.z;
    if (c0 + 3 < v.t.c) v.t.p[o + c0 + 3] = r.w;
}
// Channel-group route: lanes c0..c0+3 of pixel p.  F4: every view the op touches is read and written as whole float4 groups
// (C a multiple of 4, every blob of a conv stack): straight-line 128-bit accesses.  Its loads may take the read-only path
// even where the op writes a view it reads (axpby, an in-place ReLU backward): every element is read only by the thread
// that writes it, and before it does.
template <bool F4> struct GroupAt {
    long long p; int c0;
    __device__ float4 load(const PxView& v) const {
        return F4 ? __ldg(reinterpret_cast<const float4*>(v.t.p + p * v.t.sw + c0)) : px_load(v, p * v.t.sw, c0);
    }
    __device__ void store(const PxView& v, float4 r) const {
        if (F4) *reinterpret_cast<float4*>(v.t.p + p * v.t.sw + c0) = r;
        else px_store(v, p * v.t.sw, c0, r);
    }
};
// Strided route: element (n, c, y, x) in lane x; the other lanes are never stored.
struct ElemAt {
    int n, c, y, x;
    __device__ float4 load(const PxView& v) const { return make_float4(v.t.p[v.t.off(n, c, y, x)], 0.f, 0.f, 0.f); }
    __device__ void store(const PxView& v, float4 r) const { v.t.p[v.t.off(n, c, y, x)] = r.x; }
};
template <class F> __device__ __forceinline__ float4 lanes(F f, float4 a) { return make_float4(f(a.x), f(a.y), f(a.z), f(a.w)); }
template <class F> __device__ __forceinline__ float4 lanes(F f, float4 a, float4 b) {
    return make_float4(f(a.x, b.x), f(a.y, b.y), f(a.z, b.z), f(a.w, b.w));
}

struct ReluOp {                                   // x > 0 ? x : x * slope
    PxView in, out; float slope;
    template <class At> __device__ void operator()(const At& at) const {
        const float s = slope;
        at.store(out, lanes([s](float v) { return v > 0 ? v : v * s; }, at.load(in)));
    }
};
// dx (+)= dy * (y > 0 ? 1 : slope) from the layer's TOP data (in-place ReLU keeps no bottom data; for slope > 0 the sign is the
// same).  The product is rounded before it is added, as in the reference, where ReLU writes it and a Split layer adds it in.
struct ReluBwdOp {
    PxView data, dy, dx; float slope; int accumulate;
    template <class At> __device__ void operator()(const At& at) const {
        const float s = slope;
        float4 g = lanes([s](float t, float d) { return d * (t > 0.f ? 1.f : s); }, at.load(data), at.load(dy));
        if (accumulate) g = lanes([](float o, float v) { return o + v; }, at.load(dx), g);
        at.store(dx, g);
    }
};
struct EltwiseSumOp {                             // zero, then acc + coeff * b in bottom order
    PxView b[4]; float coeff[4]; int nb; PxView out;
    template <class At> __device__ void operator()(const At& at) const {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = 0; i < nb; i++) {
            const float k = coeff[i];
            acc = lanes([k](float a, float v) { return eltwise_term(a, k, v); }, acc, at.load(b[i]));
        }
        at.store(out, acc);
    }
};
struct AxpbyOp {                                  // y = alpha * x + beta * y; beta == 0 does not read y
    PxView x, y; float alpha, beta;
    template <class At> __device__ void operator()(const At& at) const {
        const float a = alpha, b = beta;
        const float4 xv = at.load(x);
        if (b == 0.f) at.store(y, lanes([a](float v) { return a * v; }, xv));
        else at.store(y, lanes([a, b](float v, float w) { return fmaf(a, v, b * w); }, xv, at.load(y)));
    }
};
struct CopyOp {
    PxView src, dst;
    template <class At> __device__ void operator()(const At& at) const { at.store(dst, at.load(src)); }
};
struct FillOp {
    PxView dst; float v;
    template <class At> __device__ void operator()(const At& at) const { at.store(dst, make_float4(v, v, v, v)); }
};

template <bool F4, class Op>
__global__ void ew_group_kernel(Op op, long long pixels, int G) {
    const long long total = pixels * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx / G;
        op(GroupAt<F4>{p, 4 * (int)(idx - p * G)});
    }
}
template <class Op>
__global__ void ew_strided_kernel(Op op, T4 dst) {
    const long long total = dst.count();
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        int n, c, y, x;
        long long r = idx;
        if (dst.sc == 1) { c = (int)(r % dst.c); r /= dst.c; x = (int)(r % dst.w); r /= dst.w; y = (int)(r % dst.h); n = (int)(r / dst.h); }
        else { x = (int)(r % dst.w); r /= dst.w; y = (int)(r % dst.h); r /= dst.h; c = (int)(r % dst.c); n = (int)(r / dst.c); }
        op(ElemAt{n, c, y, x});
    }
}
// Runs op over dst's elements; srcs: the other views op touches.
template <class Op>
static int ew_run(const Op& op, const T4& dst, std::initializer_list<T4> srcs, void* stream) {
    bool group = dst.is_nhwc(), f4 = dst.c % 4 == 0 && dst.px_float4_groups();
    for (const T4& s : srcs) { group = group && s.is_nhwc(); f4 = f4 && s.px_float4_groups(); }
    if (!group) return ew_launch(ew_strided_kernel<Op>, dst.count(), stream, op, dst);
    const long long pixels = (long long)dst.n * dst.h * dst.w;
    const int G = (dst.c + 3) / 4;
    return f4 ? ew_launch(ew_group_kernel<true, Op>, pixels * G, stream, op, pixels, G)
              : ew_launch(ew_group_kernel<false, Op>, pixels * G, stream, op, pixels, G);
}

// ---------------------------------------------------------------------------------------------
// Training-time augmentations of DataAugmentation (3-channel data).  Chromatic-eigen: ComputeChromaticEigenspace
// data_augmentation_layer.cu:148-185 + host finalisation :517-531, ChromaticEigenAugmentation :190-292; effects:
// ApplyEffects :295-318 and the Gaussian noise of :575-583.  space = 25 floats (tChromaticEigenSpace,
// augmentation_layer_base.hpp:117-129) followed by 3 doubles of scratch for the channel sums.
// The reference sums the mean with float atomics (order dependent); here the per-channel sums are double atomics, whose
// rounding is far below one float ulp.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void atomic_max_f(float* addr, float v) {       // v >= 0 or any sign: CAS loop like the reference
    float old = *addr;
    while (old < v) {
        const float assumed = old;
        old = __uint_as_float(atomicCAS(reinterpret_cast<unsigned int*>(addr), __float_as_uint(assumed), __float_as_uint(v)));
        if (old == assumed) break;
    }
}
__device__ __forceinline__ void atomic_min_f(float* addr, float v) {
    float old = *addr;
    while (old > v) {
        const float assumed = old;
        old = __uint_as_float(atomicCAS(reinterpret_cast<unsigned int*>(addr), __float_as_uint(assumed), __float_as_uint(v)));
        if (old == assumed) break;
    }
}
__global__ void eigenspace_init_kernel(float* space, const float* eigvec9) {
    const int i = threadIdx.x;
    if (i < 16) space[i] = (i >= 12 && i < 15) ? FLT_MAX : 0.f;
    if (i < 9) space[16 + i] = eigvec9[i];
    if (i < 3) reinterpret_cast<double*>(space + 26)[i] = 0.0;
}
__global__ void eigenspace_stats_kernel(T4 d, float* space) {
    const float* ev = space + 16;
    float mx_eig[3] = {0, 0, 0}, mx[3] = {0, 0, 0}, mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    double sum[3] = {0, 0, 0};
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        float rgb[3];
        for (int c = 0; c < 3; c++) rgb[c] = d.p[d.off(n, c, y, x)];
        for (int c = 0; c < 3; c++) {
            const float eig = ev[3 * c] * rgb[0] + ev[3 * c + 1] * rgb[1] + ev[3 * c + 2] * rgb[2];
            mx_eig[c] = fmaxf(mx_eig[c], fabsf(eig));
            mx[c] = fmaxf(mx[c], rgb[c]);
            mn[c] = fminf(mn[c], rgb[c]);
            sum[c] += rgb[c];
        }
    });
    for (int c = 0; c < 3; c++) {
        for (int o = 16; o > 0; o >>= 1) {
            mx_eig[c] = fmaxf(mx_eig[c], __shfl_xor_sync(0xffffffffu, mx_eig[c], o));
            mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
            mn[c] = fminf(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o));
            sum[c] += __shfl_xor_sync(0xffffffffu, sum[c], o);
        }
        if ((threadIdx.x & 31) == 0) {
            atomic_max_f(space + 6 + c, mx_eig[c]);
            atomic_max_f(space + 9 + c, mx[c]);
            atomic_min_f(space + 12 + c, mn[c]);
            atomicAdd(reinterpret_cast<double*>(space + 26) + c, sum[c]);
        }
    }
}
__global__ void eigenspace_finish_kernel(float* space, int num, int height, int width) {
    if (threadIdx.x || blockIdx.x) return;
    float* mean_eig = space, *mean_rgb = space + 3, *max_abs_eig = space + 6;
    const float* ev = space + 16;
    const double* sum = reinterpret_cast<const double*>(space + 26);
    for (int c = 0; c < 3; c++) {
        mean_rgb[c] = (float)(sum[c] / (double)width / (double)height);
        mean_rgb[c] = mean_rgb[c] / num;
    }
    for (int c = 0; c < 3; c++) {
        mean_eig[c] = ev[3 * c] * mean_rgb[0] + ev[3 * c + 1] * mean_rgb[1] + ev[3 * c + 2] * mean_rgb[2];
        if (max_abs_eig[c] > 1e-2) mean_eig[c] = mean_eig[c] / max_abs_eig[c];
    }
    space[15] = sqrtf(max_abs_eig[0] * max_abs_eig[0] + max_abs_eig[1] * max_abs_eig[1] + max_abs_eig[2] * max_abs_eig[2]);
}
__global__ void chromatic_eigen_kernel(T4 d, const float* __restrict__ coeffs, const float* __restrict__ space, float max_multiplier) {
    const float* mean_eig = space, *mean_rgb = space + 3, *max_abs_eig = space + 6, *eigvec = space + 16;
    const float max_l = space[15];
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const float* ch = coeffs + 22 * n;
        float s, s1, l, l1 = 0.f;
        float rgb[3], eig[3];
        for (int c = 0; c < 3; c++) rgb[c] = d.p[d.off(n, c, y, x)] - mean_rgb[c];
        for (int c = 0; c < 3; c++) {
            eig[c] = eigvec[3 * c] * rgb[0] + eigvec[3 * c + 1] * rgb[1] + eigvec[3 * c + 2] * rgb[2];
            if (max_abs_eig[c] > 1e-2f) {
                eig[c] = eig[c] / max_abs_eig[c];
                eig[c] = copysignf(powf(fabsf(eig[c]), ch[c]), eig[c]);
                eig[c] = eig[c] + ch[3 + c];
                eig[c] = eig[c] * ch[6 + c];
            }
        }
        for (int c = 0; c < 3; c++) eig[c] = eig[c] + mean_eig[c];
        if (max_abs_eig[0] > 1e-2f) {
            eig[0] = copysignf(powf(fabsf(eig[0]), ch[9]), eig[0]);
            eig[0] = eig[0] + ch[12];
            eig[0] = eig[0] * ch[15];
        }
        s = sqrtf(eig[1] * eig[1] + eig[2] * eig[2]);
        s1 = s;
        if (s > 1e-2f) {
            s1 = powf(s1, ch[10]);
            s1 = fmaxf(s1 + ch[13], 0.f);
            s1 = s1 * ch[16];
        }
        if (ch[21] != 0) {
            const float t1 = cosf(ch[21]) * eig[1] - sinf(ch[21]) * eig[2];
            const float t2 = sinf(ch[21]) * eig[1] + cosf(ch[21]) * eig[2];
            eig[1] = t1; eig[2] = t2;
        }
        for (int c = 0; c < 3; c++) if (max_abs_eig[c] > 1e-2f) eig[c] = eig[c] * max_abs_eig[c];
        if (max_l > 1e-2f) {
            l1 = sqrtf(eig[0] * eig[0] + eig[1] * eig[1] + eig[2] * eig[2]);
            l1 = l1 / max_l;
        }
        if (s > 1e-2f) { eig[1] = eig[1] / s * s1; eig[2] = eig[2] / s * s1; }
        if (max_l > 1e-2f) {
            l = sqrtf(eig[0] * eig[0] + eig[1] * eig[1] + eig[2] * eig[2]);
            l1 = powf(l1, ch[18]);
            l1 = fmaxf(l1 + ch[19], 0.f);
            l1 = l1 * ch[20];
            l1 = l1 * max_l;
            if (l > 1e-2f)
                for (int c = 0; c < 3; c++) {
                    eig[c] = eig[c] / l * l1;
                    if (eig[c] > max_abs_eig[c]) eig[c] = max_abs_eig[c];
                }
        }
        for (int c = 0; c < 3; c++) {
            float v = eigvec[c] * eig[0] + eigvec[3 + c] * eig[1] + eigvec[6 + c] * eig[2];
            v = fminf(v, max_multiplier);
            v = fmaxf(v, 0.f);
            d.p[d.off(n, c, y, x)] = v;
        }
    });
}
__global__ void apply_effects_kernel(T4 d, const float* __restrict__ effects, float max_multiplier) {
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const float* e = effects + 9 * n;
        const bool shadow = (x - d.w / 2) * e[4] + (y - d.h / 2) * e[5] - e[6] > 0;
        for (int c = 0; c < d.c; c++) {
            float sample = d.p[d.off(n, c, y, x)];
            if (shadow) sample -= e[7];
            d.p[d.off(n, c, y, x)] = clampf(sample, 0.f, max_multiplier);
        }
    });
}
// counter-based generator (SplitMix64 of (seed, element index)) + Box-Muller.  The reference draws from cuRAND's default
// generator with an unpinned seed/offset: the noise field is not reproducible there either, only its distribution.
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__global__ void gaussian_noise_kernel(T4 d, const float* __restrict__ effects, unsigned long long seed) {
    for_each_element(d, [&](Idx4 e, long long idx) {
        const float sigma = effects[9 * e.n + 8];
        if (!(sigma > 0)) return;
        const unsigned long long h = splitmix64(seed ^ splitmix64((unsigned long long)idx));
        const float u1 = ((float)(h >> 40) + 1.0f) * (1.0f / 16777216.0f);                 // (0, 1]
        const float u2 = (float)((h >> 16) & 0xffffff) * (1.0f / 16777216.0f);
        const float g = sqrtf(-2.0f * logf(u1)) * cosf(6.28318530718f * u2);
        float* p = d.p + d.off(e.n, e.c, e.y, e.x);
        *p = *p + sigma * g;
    });
}

// 0xFFE00000, the reference GPU's NaN pattern (flow_warp_layer.cu:372-375), if fill_nan, else 0: FlowWarp's value outside the image
static float warp_fill(int fill_nan) {
    float fill = 0.f;
    if (fill_nan) { unsigned u = 0xFFE00000u; memcpy(&fill, &u, 4); }
    return fill;
}
// The F4 route of FlowWarp, ChannelNorm and the warp block: every pixel of t (c <= 4) is one 16-byte float4 group.
static bool px_one_group(const T4& t) { return t.c <= 4 && t.px_float4_groups(); }

// ---------------------------------------------------------------------------------------------
// 8-bit frames [N][H][W][K] -> (N, 3, H, W) BGR floats (scripts/run-flownet.py:30-35: HWC RGB to NCHW BGR; a gray frame is
// broadcast to the three channels like pycaffe's blob assignment, RGBA drops alpha).  One thread per pixel; byte loads need no
// alignment (W*K may be odd).  A byte converts to float exactly, so the blob equals one filled from image_to_blob's floats.
// Channel-fast views store through px_store (never a lane beyond C), others channel by channel.
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void frames_to_tensor_kernel(const uint8_t* __restrict__ frames, PxView dst) {
    const T4& d = dst.t;
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const uint8_t* p = frames + (((long long)n * d.h + y) * d.w + x) * K;
        const float4 r = K == 1 ? make_float4(p[0], p[0], p[0], 0.f) : make_float4(p[2], p[1], p[0], 0.f);
        if (d.sc == 1) {
            px_store(dst, d.off(n, 0, y, x), 0, r);
        } else {
            d.p[d.off(n, 0, y, x)] = r.x;
            d.p[d.off(n, 1, y, x)] = r.y;
            d.p[d.off(n, 2, y, x)] = r.z;
        }
    });
}

// ---------------------------------------------------------------------------------------------
// Flow payloads -> (N, 2, H, W) floats (include/fn2_flow.h).  .flo is [N][H][W][2]; PFM is [N][H][W][3] stored bottom-up,
// read top-down keeping channels 0, 1 (CImg load_pfm + mirror('y')), byte-swapped when big-endian.  UINT16FLOW restates the
// reference's short(32 v) / 32 round trip (convert_imageset_and_flow.cpp:168-179, custom_data_layer.cpp:88-107): 32 v is
// exact, trunc(32 v) in [-32768, 32766] survives as t / 32 (the int conversion turns a -0 truncation into +0), everything
// else -- NaN, 32767 and above, below -32768 -- is NaN.  Every step is exact.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float flow_value(uint32_t bits, bool swap, int quantise) {
    const float v = __uint_as_float(swap ? __byte_perm(bits, 0, 0x0123) : bits);
    if (!quantise) return v;
    const float s = v * 32.f;
    return s < 32767.f && s > -32769.f ? (float)__float2int_rz(s) * 0.03125f : __uint_as_float(0x7fc00000u);
}

template <int FMT>
__global__ void flow_to_tensor_kernel(const uint32_t* __restrict__ src, PxView dst, int quantise) {
    const T4& d = dst.t;
    constexpr int K = FMT == FN2_FLOW_FLO ? 2 : 3;
    constexpr bool swap = FMT == FN2_FLOW_PFM_BE;
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const int row = FMT == FN2_FLOW_FLO ? y : d.h - 1 - y;
        const uint32_t* p = src + (((long long)n * d.h + row) * d.w + x) * K;
        const float4 r = make_float4(flow_value(p[0], swap, quantise), flow_value(p[1], swap, quantise), 0.f, 0.f);
        if (d.sc == 1) {
            px_store(dst, d.off(n, 0, y, x), 0, r);
        } else {
            d.p[d.off(n, 0, y, x)] = r.x;
            d.p[d.off(n, 1, y, x)] = r.y;
        }
    });
}

// ---------------------------------------------------------------------------------------------
// KITTI flow PNGs (include/fn2_flow.h).  Decode: the unfiltered payload [N][H][W][3] big-endian uint16 -> (N, 2, H, W) floats,
// one thread per pixel; (R - 32768) / 64 is exact, an invalid pixel (B = 0) is NaN in both channels, and UINT16FLOW goes
// through flow_value's quantisation.  Encode: each thread encodes its own pixel and its left, up and up-left neighbours from
// the flow and Paeth-filters its 6 bytes against them, so no thread reads another's output; the thread of x = 0 also writes
// the row's filter byte.
// ---------------------------------------------------------------------------------------------
__global__ void kitti_samples_to_tensor_kernel(const uint16_t* __restrict__ src, PxView dst, int quantise) {
    const T4& d = dst.t;
    for_each_pixel(d.n, d.h, d.w, [&](int n, int y, int x) {
        const uint16_t* p = src + (((long long)n * d.h + y) * d.w + x) * 3;
        const uint32_t r = __byte_perm(p[0], 0, 0x4401), g = __byte_perm(p[1], 0, 0x4401), b = p[2];
        const float nan = __uint_as_float(0x7fc00000u);
        const float u = b ? flow_value(__float_as_uint((float)((int)r - 32768) * 0.015625f), false, quantise) : nan;
        const float v = b ? flow_value(__float_as_uint((float)((int)g - 32768) * 0.015625f), false, quantise) : nan;
        if (d.sc == 1) {
            px_store(dst, d.off(n, 0, y, x), 0, make_float4(u, v, 0.f, 0.f));
        } else {
            d.p[d.off(n, 0, y, x)] = u;
            d.p[d.off(n, 1, y, x)] = v;
        }
    });
}

// The stored samples (R, G, B) of flow pixel (n, y, x); (0, 0, 0) outside the image, PNG's value left of and above it.
struct KittiPx { uint32_t s[3]; };
__device__ __forceinline__ KittiPx kitti_encode(const T4& f, int n, int y, int x) {
    KittiPx r = {{0u, 0u, 0u}};
    if (x < 0 || y < 0) return r;
    const float u = f.p[f.off(n, 0, y, x)], v = f.p[f.off(n, 1, y, x)];
    if (!isfinite(u) || !isfinite(v)) return r;
    r.s[0] = __float2uint_rz(fmaxf(fminf(u * 64.f + 32768.f, 65535.f), 0.f));
    r.s[1] = __float2uint_rz(fmaxf(fminf(v * 64.f + 32768.f, 65535.f), 0.f));
    r.s[2] = 1u;
    return r;
}
__device__ __forceinline__ uint32_t paeth_predict(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (uint32_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

__global__ void flow_to_kitti_png_rows_kernel(T4 f, uint8_t* __restrict__ rows) {
    const long long row_bytes = 1 + 6LL * f.w;
    for_each_pixel(f.n, f.h, f.w, [&](int n, int y, int x) {
        const KittiPx self = kitti_encode(f, n, y, x), left = kitti_encode(f, n, y, x - 1), up = kitti_encode(f, n, y - 1, x),
                      upleft = kitti_encode(f, n, y - 1, x - 1);
        uint8_t* row = rows + ((long long)n * f.h + y) * row_bytes;
        if (x == 0) row[0] = 4;
        uint8_t* o = row + 1 + 6LL * x;
        #pragma unroll
        for (int i = 0; i < 6; i++) {
            const int sh = i & 1 ? 0 : 8;                                          // big-endian: the high byte first
            const int j = i >> 1;
            const uint32_t raw = (self.s[j] >> sh) & 0xff;
            o[i] = (uint8_t)(raw - paeth_predict((left.s[j] >> sh) & 0xff, (up.s[j] >> sh) & 0xff, (upleft.s[j] >> sh) & 0xff));
        }
    });
}

// ---------------------------------------------------------------------------------------------
// Flow colour coding (include/fn2_flow.h): the Middlebury colour wheel (Baker et al., colorcode.cpp), every pixel divided by
// a per-image scale.  flow_max_radius_kernel: grid (blocks, N), each block's largest float32 radius over its share of image
// n's known pixels folded into max[n] with an integer atomicMax (non-negative floats order as their bits; max[n] starts at
// -1, whose bits are negative), so the result is exact and independent of the order.  The colour kernels, one thread per
// pixel: the dense form writes the pixel's 3 bytes; the PNG form colours the pixel and its left, up and up-left neighbours and
// Paeth-filters its 3 bytes against them, as flow_to_kitti_png_rows_kernel does.  The arithmetic is float32 as written
// (-fmad=false) except atan2, evaluated in double and rounded to float32: atan2f's last-ulp errors would flip the many bytes
// that sit exactly on an integer (a channel whose two wheel entries are equal), so a host restatement could not reproduce them.
// ---------------------------------------------------------------------------------------------
__global__ void fill_minus_one_kernel(float* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = -1.f;
}

__global__ void flow_max_radius_kernel(T4 f, float* __restrict__ max_out) {
    const int n = blockIdx.y;
    const long long hw = (long long)f.h * f.w;
    float m = -1.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hw; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / f.w), x = (int)(i % f.w);
        const float u = f.p[f.off(n, 0, y, x)], v = f.p[f.off(n, 1, y, x)];
        if (flow_known(u, v)) m = fmaxf(m, sqrtf(u * u + v * v));
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float warp_max[32];
    if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, warp_max[w]);
        if (m >= 0.f) atomicMax(reinterpret_cast<int*>(max_out + n), __float_as_int(m));
    }
}

// Entry k of the 55-colour wheel, segments RY 15, YG 6, GC 4, CB 11, BM 13, MR 6, in integer arithmetic.
__device__ __forceinline__ void wheel_entry(int k, int (&w)[3]) {
    if (k < 15) { w[0] = 255; w[1] = 255 * k / 15; w[2] = 0; return; }
    k -= 15;
    if (k < 6) { w[0] = 255 - 255 * k / 6; w[1] = 255; w[2] = 0; return; }
    k -= 6;
    if (k < 4) { w[0] = 0; w[1] = 255; w[2] = 255 * k / 4; return; }
    k -= 4;
    if (k < 11) { w[0] = 0; w[1] = 255 - 255 * k / 11; w[2] = 255; return; }
    k -= 11;
    if (k < 13) { w[0] = 255 * k / 13; w[1] = 0; w[2] = 255; return; }
    k -= 13;
    w[0] = 255; w[1] = 0; w[2] = 255 - 255 * k / 6;
}

// The scale of image n: max_flow when positive, else max[n] (fallback[n] when max[n] is negative and fallback is given), and
// 1 when that is not positive.
__device__ __forceinline__ float colour_scale(const float* max, const float* fallback, float max_flow, int n) {
    if (max_flow > 0.f) return max_flow;
    float r = max[n];
    if (r < 0.f && fallback) r = fallback[n];
    return r > 0.f ? r : 1.f;
}

// The colour of flow pixel (n, y, x) as 0x00BBGGRR; 0 (black) for an unknown pixel and outside the image.
__device__ __forceinline__ uint32_t flow_colour(const T4& f, int n, int y, int x, float scale) {
    if (x < 0 || y < 0) return 0u;
    const float u = f.p[f.off(n, 0, y, x)], v = f.p[f.off(n, 1, y, x)];
    if (!flow_known(u, v)) return 0u;
    const float fx = u / scale, fy = v / scale;
    const float rad = sqrtf(fx * fx + fy * fy);
    const float a = (float)atan2(-(double)fy, -(double)fx) / 3.14159265358979323846f;      // a correctly rounded atan2f
    const float fk = (a + 1.f) / 2.f * 54.f;
    const int k0 = (int)fk, k1 = (k0 + 1) % 55;
    const float fr = fk - (float)k0;
    int w0[3], w1[3];
    wheel_entry(k0, w0);
    wheel_entry(k1, w1);
    uint32_t rgb = 0u;
    #pragma unroll
    for (int c = 0; c < 3; c++) {
        float col = (1.f - fr) * (float)w0[c] / 255.f + fr * (float)w1[c] / 255.f;
        col = rad <= 1.f ? 1.f - rad * (1.f - col) : col * 0.75f;
        rgb |= (uint32_t)(int)(255.f * col) << (8 * c);
    }
    return rgb;
}

__global__ void flow_to_color_kernel(T4 f, const float* __restrict__ max, const float* __restrict__ fallback, float max_flow,
                                     uint8_t* __restrict__ rgb) {
    for_each_pixel(f.n, f.h, f.w, [&](int n, int y, int x) {
        const uint32_t c = flow_colour(f, n, y, x, colour_scale(max, fallback, max_flow, n));
        uint8_t* o = rgb + (((long long)n * f.h + y) * f.w + x) * 3;
        o[0] = (uint8_t)c; o[1] = (uint8_t)(c >> 8); o[2] = (uint8_t)(c >> 16);
    });
}

__global__ void flow_to_color_png_rows_kernel(T4 f, const float* __restrict__ max, const float* __restrict__ fallback,
                                              float max_flow, uint8_t* __restrict__ rows) {
    const long long row_bytes = 1 + 3LL * f.w;
    for_each_pixel(f.n, f.h, f.w, [&](int n, int y, int x) {
        const float s = colour_scale(max, fallback, max_flow, n);
        const uint32_t self = flow_colour(f, n, y, x, s), left = flow_colour(f, n, y, x - 1, s),
                       up = flow_colour(f, n, y - 1, x, s), upleft = flow_colour(f, n, y - 1, x - 1, s);
        uint8_t* row = rows + ((long long)n * f.h + y) * row_bytes;
        if (x == 0) row[0] = 4;
        uint8_t* o = row + 1 + 3LL * x;
        #pragma unroll
        for (int c = 0; c < 3; c++) {
            const int sh = 8 * c;
            o[c] = (uint8_t)(((self >> sh) & 0xff) - paeth_predict((left >> sh) & 0xff, (up >> sh) & 0xff, (upleft >> sh) & 0xff));
        }
    });
}

// ---------------------------------------------------------------------------------------------
// Forward-backward consistency (include/fn2_flow.h; Sundaram, Brox and Keutzer, ECCV 2010).  The backward flow is sampled where
// the forward flow lands with FlowWarp's own taps and mix (warp_taps, warp_channel), so the sample is fn2_flow_warp_forward's
// output for image = bwd, flow = fwd, bit for bit.  Grid (blocks, N): pair blockIdx.y, its pixels in a grid-stride walk, one
// byte written per pixel.  Each pixel reads 8 bytes of forward flow and four backward taps, mostly its neighbours' (cache hits).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool fb_occluded(const T4& fwd, const T4& bwd, float alpha1, float alpha2, int n, int y, int x) {
    const float fu = fwd.p[fwd.off(n, 0, y, x)], fv = fwd.p[fwd.off(n, 1, y, x)];
    if (!isfinite(fu) || !isfinite(fv)) return true;
    const WarpTaps t = warp_taps(bwd, n, y, x, fu, fv);
    if (!t.inside) return true;
    const float bu = warp_channel(t, bwd, 0), bv = warp_channel(t, bwd, 1);
    if (!isfinite(bu) || !isfinite(bv)) return true;
    const float du = fu + bu, dv = fv + bv;
    const float lhs = du * du + dv * dv;
    const float mag = (fu * fu + fv * fv) + (bu * bu + bv * bv);
    return lhs > alpha1 * mag + alpha2;
}

__global__ void flow_fb_occlusion_kernel(T4 fwd, T4 bwd, float alpha1, float alpha2, uint8_t* __restrict__ out,
                                         long long row_stride, long long pair_stride) {
    const int n = blockIdx.y;
    const long long hw = (long long)fwd.h * fwd.w;
    uint8_t* o = out + n * pair_stride;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hw; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / fwd.w), x = (int)(i - (long long)y * fwd.w);
        o[y * row_stride + x] = fb_occluded(fwd, bwd, alpha1, alpha2, n, y, x) ? 255 : 0;
    }
}

}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2_flow_warp_forward(const fn2_tensor* image, const fn2_tensor* flow, const fn2_tensor* warped,
                          int fill_nan, void* stream) {
    FN2_CHECK_ARG(valid(image) && valid(flow) && valid(warped), "flow_warp: null/empty tensor");
    T4 img = view(image), fl = view(flow), out = view(warped);
    FN2_CHECK_ARG(fl.c == 2, "flow_warp: flow must have 2 channels (flow_warp_layer.cpp:46)");
    FN2_CHECK_ARG(fl.n == img.n && fl.h == img.h && fl.w == img.w,
                  "flow_warp: flow dims must match image (flow_warp_layer.cpp:45-48)");
    FN2_CHECK_ARG(same_dims(img, out), "flow_warp: top must have the image's shape");
    const float fill = warp_fill(fill_nan);
    const long long total = (long long)out.n * out.h * out.w;
    return px_one_group(img) ? ew_launch(flow_warp_fwd_kernel<true>, total, stream, img, fl, out, fill)
                             : ew_launch(flow_warp_fwd_kernel<false>, total, stream, img, fl, out, fill);
}

int fn2_flow_warp_backward(const fn2_tensor* image, const fn2_tensor* flow,
                           const fn2_tensor* warped_diff, const fn2_tensor* image_diff,
                           const fn2_tensor* flow_diff, void* stream) {
    FN2_CHECK_ARG(valid(image) && valid(flow) && valid(warped_diff) && valid(image_diff) && valid(flow_diff),
                  "flow_warp_backward: null/empty tensor");
    T4 img = view(image), fl = view(flow), wd = view(warped_diff), id = view(image_diff), fd = view(flow_diff);
    FN2_CHECK_ARG(fl.c == 2 && fd.c == 2 && same_dims(img, wd) && same_dims(img, id) && same_dims(fl, fd),
                  "flow_warp_backward: shape mismatch");
    const int rc = fn2_fill(image_diff, 0.f, stream);
    if (rc) return rc;
    return ew_launch(flow_warp_bwd_kernel, (long long)img.n * img.h * img.w, stream, img, fl, wd, id, fd);
}

int fn2_resample_forward(const fn2_tensor* bottom, const fn2_tensor* top, int type, int antialias,
                         void* stream) {
    FN2_CHECK_ARG(valid(bottom) && valid(top), "resample: null/empty tensor");
    T4 in = view(bottom), out = view(top);
    FN2_CHECK_ARG(in.n == out.n && in.c == out.c,
                  "resample: top channel count must match bottom (resample_layer.cu:143)");
    const float fx = (float)in.w / (float)out.w;
    const float fy = (float)in.h / (float)out.h;
    const int isDown = (fx > 1) || (fy > 1);
    const int aa = isDown && antialias;
    const long long total = (long long)out.n * out.h * out.w;
    if (type == 1) return ew_launch(resample_kernel<1>, total, stream, in, out, fx, fy, aa);
    if (type == 2) return ew_launch(resample_kernel<2>, total, stream, in, out, fx, fy, aa);
    if (type == 3) return ew_launch(resample_kernel<3>, total, stream, in, out, fx, fy, aa);
    set_error("resample: unsupported type %d (resample_layer.cu:204)", type);
    return FN2_ERR_INVALID;
}

int fn2_warp_block_forward(const fn2_tensor* flow_in, const fn2_tensor* image0, const fn2_tensor* image1, const fn2_tensor* flow_full,
                           const fn2_tensor* warped, const fn2_tensor* err, const fn2_tensor* err_norm, const fn2_tensor* flow_scaled,
                           float scale_coeff, int fill_nan, void* stream) {
    FN2_CHECK_ARG(valid(flow_in) && valid(image0) && valid(image1) && valid(flow_full) && valid(warped) && valid(err) && valid(err_norm) &&
                  valid(flow_scaled), "warp_block: null/empty tensor");
    T4 fin = view(flow_in), i0 = view(image0), i1 = view(image1), ff = view(flow_full), wp = view(warped), er = view(err), en = view(err_norm),
       fs = view(flow_scaled);
    FN2_CHECK_ARG(fin.c == 2 && ff.c == 2 && fs.c == 2 && en.c == 1 && i1.c <= 4, "warp_block: channel counts");
    FN2_CHECK_ARG(same_dims(i0, i1) && same_dims(i0, wp) && same_dims(i0, er) && same_dims(ff, fs) && ff.n == i0.n && ff.h == i0.h && ff.w == i0.w &&
                  en.n == i0.n && en.h == i0.h && en.w == i0.w && fin.n == ff.n, "warp_block: shape mismatch");
    const float fx = (float)fin.w / (float)ff.w, fy = (float)fin.h / (float)ff.h;
    FN2_CHECK_ARG(fx <= 1.f && fy <= 1.f, "warp_block: the flow must be up-sampled (use the layer chain otherwise)");
    const float fill = warp_fill(fill_nan);
    const long long total = (long long)ff.n * ff.h * ff.w;
    return px_one_group(i1) ? ew_launch(warp_block_kernel<true>, total, stream, fin, i0, i1, ff, wp, er, en, fs, fx, fy, scale_coeff, fill)
                            : ew_launch(warp_block_kernel<false>, total, stream, fin, i0, i1, ff, wp, er, en, fs, fx, fy, scale_coeff, fill);
}

int fn2_spatial_augmentation(const fn2_tensor* bottom, const fn2_tensor* top,
                             const float* trans_mats_dev, void* stream) {
    FN2_CHECK_ARG(valid(bottom) && valid(top) && trans_mats_dev, "spatial_augmentation: null argument");
    T4 in = view(bottom), out = view(top);
    FN2_CHECK_ARG(in.n == out.n && in.c == out.c, "spatial_augmentation: num/channels must match");
    FN2_CHECK_ARG(in.w >= 2 && in.h >= 2, "spatial_augmentation: bottom must be at least 2x2");
    return ew_launch(spatial_aug_kernel, (long long)out.n * out.h * out.w, stream, in, out, trans_mats_dev);
}

int fn2_color_contrast_augmentation(const fn2_tensor* data, const float* chroma_dev,
                                    float max_multiplier, void* stream) {
    FN2_CHECK_ARG(valid(data) && chroma_dev, "color_contrast: null argument");
    T4 d = view(data);
    FN2_CHECK_ARG(d.c == 3, "Chromatic augmentations only work with 3-channel input "
                            "(data_augmentation_layer.cu:561)");
    return ew_launch(color_contrast_kernel, (long long)d.n * d.h * d.w, stream, d, chroma_dev, max_multiplier);
}

int fn2_mean_update(const fn2_tensor* top, const fn2_tensor* mean_pp, float* mean_pc_dev,
                    float num_iter, void* stream) {
    FN2_CHECK_ARG(valid(top) && valid(mean_pp) && mean_pc_dev, "mean_update: null argument");
    T4 t = view(top), m = view(mean_pp);
    FN2_CHECK_ARG(m.n == 1 && m.c == t.c && m.h == t.h && m.w == t.w,
                  "mean_update: mean blob must be (1,C,H,W) (data_augmentation_layer.cu:603)");
    const int rc = ew_launch(mean_update_kernel, (long long)t.c * t.h * t.w, stream, t, m, num_iter);
    if (rc) return rc;
    mean_per_channel_kernel<<<t.c, 256, 0, (cudaStream_t)stream>>>(m, mean_pc_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_mean_subtract(const fn2_tensor* top, const fn2_tensor* mean_pp, const float* mean_pc_dev,
                      int per_pixel, void* stream) {
    FN2_CHECK_ARG(valid(top), "mean_subtract: null top");
    T4 t = view(top), m = t;
    if (per_pixel) {
        FN2_CHECK_ARG(valid(mean_pp), "mean_subtract: per-pixel mean missing");
        m = view(mean_pp);
        FN2_CHECK_ARG(m.c == t.c && m.h == t.h && m.w == t.w, "mean_subtract: mean shape mismatch");
    } else {
        FN2_CHECK_ARG(mean_pc_dev, "mean_subtract: per-channel mean missing");
    }
    return ew_launch(mean_subtract_kernel, t.count(), stream, t, m, mean_pc_dev, per_pixel);
}

int fn2_relu_forward(const fn2_tensor* bottom, const fn2_tensor* top, float negative_slope, void* stream) {
    FN2_CHECK_ARG(valid(bottom) && valid(top), "relu: null/empty tensor");
    T4 in = view(bottom), out = view(top);
    FN2_CHECK_ARG(same_dims(in, out), "relu: shape mismatch");
    return ew_run(ReluOp{px_view(in), px_view(out), negative_slope}, out, {in}, stream);
}

int fn2_relu_backward(const fn2_tensor* top_data, const fn2_tensor* top_diff, const fn2_tensor* bottom_diff, float negative_slope,
                      int accumulate, void* stream) {
    FN2_CHECK_ARG(valid(top_data) && valid(top_diff) && valid(bottom_diff), "relu_backward: null/empty tensor");
    T4 d = view(top_data), dy = view(top_diff), dx = view(bottom_diff);
    FN2_CHECK_ARG(same_dims(d, dy) && same_dims(d, dx), "relu_backward: shape mismatch");
    return ew_run(ReluBwdOp{px_view(d), px_view(dy), px_view(dx), negative_slope, accumulate}, dx, {d, dy}, stream);
}

int fn2_eltwise_sum(const fn2_tensor* const* bottoms, const float* coeffs, int num_bottoms,
                    const fn2_tensor* top, void* stream) {
    FN2_CHECK_ARG(bottoms && valid(top) && num_bottoms >= 1 && num_bottoms <= 4,
                  "eltwise_sum: need 1..4 bottoms");
    T4 out = view(top), b[4] = {out, out, out, out};
    EltwiseSumOp op{};
    op.nb = num_bottoms;
    op.out = px_view(out);
    for (int i = 0; i < num_bottoms; i++) {
        FN2_CHECK_ARG(valid(bottoms[i]), "eltwise_sum: null bottom");
        b[i] = view(bottoms[i]);
        FN2_CHECK_ARG(same_dims(b[i], out), "eltwise_sum: shape mismatch (eltwise_layer.cpp:33)");
        op.b[i] = px_view(b[i]);
        op.coeff[i] = coeffs ? coeffs[i] : 1.0f;
    }
    return ew_run(op, out, {b[0], b[1], b[2], b[3]}, stream);
}

int fn2_axpby(const fn2_tensor* x, float alpha, const fn2_tensor* y, float beta, void* stream) {
    FN2_CHECK_ARG(valid(x) && valid(y), "axpby: null/empty tensor");
    T4 xv = view(x), yv = view(y);
    FN2_CHECK_ARG(same_dims(xv, yv), "axpby: shape mismatch");
    return ew_run(AxpbyOp{px_view(xv), px_view(yv), alpha, beta}, yv, {xv}, stream);
}

int fn2_channel_norm_forward(const fn2_tensor* bottom, const fn2_tensor* top, void* stream) {
    FN2_CHECK_ARG(valid(bottom) && valid(top), "channel_norm: null/empty tensor");
    T4 in = view(bottom), out = view(top);
    FN2_CHECK_ARG(out.c == 1 && out.n == in.n && out.h == in.h && out.w == in.w,
                  "channel_norm: top must be (N,1,H,W) (channel_norm_layer.cpp:29)");
    const long long total = (long long)in.n * in.h * in.w;
    return px_one_group(in) ? ew_launch(channel_norm_kernel<true>, total, stream, in, out)
                            : ew_launch(channel_norm_kernel<false>, total, stream, in, out);
}

int fn2_copy(const fn2_tensor* src, const fn2_tensor* dst, void* stream) {
    FN2_CHECK_ARG(valid(src) && valid(dst), "copy: null/empty tensor");
    T4 s = view(src), d = view(dst);
    FN2_CHECK_ARG(same_dims(s, d), "copy: shape mismatch");
    cudaStream_t st = (cudaStream_t)stream;
    const bool s_cf = (s.sc == 1), d_cf = (d.sc == 1);
    const bool s_pl = (s.sw == 1), d_pl = (d.sw == 1);
    if (d.c >= 8 && ((s_cf && d_pl && !d_cf) || (s_pl && d_cf && !s_cf))) {
        const long long hw = (long long)d.h * d.w;
        dim3 grid((unsigned)((hw + 31) / 32), (unsigned)((d.c + 31) / 32), (unsigned)d.n);
        copy_transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(s, d, s_cf ? 1 : 0);
        FN2_LAUNCH_CHECK();
        return FN2_OK;
    }
    return ew_run(CopyOp{px_view(s), px_view(d)}, d, {s}, stream);
}

int fn2_chromatic_eigenspace(const fn2_tensor* data, const float* eigvec9_dev, float* space_dev, void* stream) {
    FN2_CHECK_ARG(valid(data) && eigvec9_dev && space_dev, "chromatic_eigenspace: null argument");
    T4 d = view(data);
    FN2_CHECK_ARG(d.c == 3, "Chromatic-Eigen augmentations only work with 3-channel input (data_augmentation_layer.cu:488)");
    FN2_CHECK_ARG(!((uintptr_t)space_dev & 7), "chromatic_eigenspace: space must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    eigenspace_init_kernel<<<1, 32, 0, st>>>(space_dev, eigvec9_dev);
    FN2_LAUNCH_CHECK();
    const int rc = ew_launch(eigenspace_stats_kernel, (long long)d.n * d.h * d.w, stream, d, space_dev);
    if (rc) return rc;
    eigenspace_finish_kernel<<<1, 32, 0, st>>>(space_dev, d.n, d.h, d.w);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_chromatic_eigen_augmentation(const fn2_tensor* data, const float* coeffs_dev, const float* space_dev,
                                     float max_multiplier, void* stream) {
    FN2_CHECK_ARG(valid(data) && coeffs_dev && space_dev, "chromatic_eigen: null argument");
    T4 d = view(data);
    FN2_CHECK_ARG(d.c == 3, "Chromatic-Eigen augmentations only work with 3-channel input (data_augmentation_layer.cu:551)");
    return ew_launch(chromatic_eigen_kernel, (long long)d.n * d.h * d.w, stream, d, coeffs_dev, space_dev, max_multiplier);
}

int fn2_apply_effects(const fn2_tensor* data, const float* effects_dev, float max_multiplier, unsigned long long noise_seed,
                      int add_noise, void* stream) {
    FN2_CHECK_ARG(valid(data) && effects_dev, "apply_effects: null argument");
    T4 d = view(data);
    FN2_CHECK_ARG(d.c == 3, "Effect augmentations only work with 3-channel input (data_augmentation_layer.cu:567)");
    const int rc = ew_launch(apply_effects_kernel, (long long)d.n * d.h * d.w, stream, d, effects_dev, max_multiplier);
    if (rc || !add_noise) return rc;
    return ew_launch(gaussian_noise_kernel, d.count(), stream, d, effects_dev, noise_seed);
}

int fn2_fill(const fn2_tensor* dst, float value, void* stream) {
    FN2_CHECK_ARG(valid(dst), "fill: null/empty tensor");
    T4 d = view(dst);
    return ew_run(FillOp{px_view(d), value}, d, {}, stream);
}

int fn2_frames_to_tensor(const void* frames_dev, int channels, const fn2_tensor* dst, void* stream) {
    FN2_CHECK_ARG(frames_dev, "frames_to_tensor: frames is null");
    FN2_CHECK_ARG(valid(dst), "frames_to_tensor: dst is null or empty");
    FN2_CHECK_ARG(channels == 1 || channels == 3 || channels == 4,
                  "frames_to_tensor: channels must be 1, 3 or 4 (gray, RGB, RGBA), got %d", channels);
    T4 d = view(dst);
    FN2_CHECK_ARG(d.c == 3, "frames_to_tensor: dst must have 3 channels (B, G, R), has %d", d.c);
    const uint8_t* f = static_cast<const uint8_t*>(frames_dev);
    const long long total = (long long)d.n * d.h * d.w;
    if (channels == 1) return ew_launch(frames_to_tensor_kernel<1>, total, stream, f, px_view(d));
    if (channels == 3) return ew_launch(frames_to_tensor_kernel<3>, total, stream, f, px_view(d));
    return ew_launch(frames_to_tensor_kernel<4>, total, stream, f, px_view(d));
}

int fn2_flow_to_tensor(const void* src_dev, int format, int flags, const fn2_tensor* dst, void* stream) {
    FN2_CHECK_ARG(src_dev, "flow_to_tensor: src is null");
    FN2_CHECK_ARG(format == FN2_FLOW_FLO || format == FN2_FLOW_PFM || format == FN2_FLOW_PFM_BE || format == FN2_FLOW_KITTI,
                  "flow_to_tensor: format must be FN2_FLOW_FLO, FN2_FLOW_PFM, FN2_FLOW_PFM_BE or FN2_FLOW_KITTI, got %d", format);
    const int align = format == FN2_FLOW_KITTI ? 2 : 4;
    FN2_CHECK_ARG((reinterpret_cast<uintptr_t>(src_dev) & (align - 1)) == 0, "flow_to_tensor: src must be %d-byte aligned", align);
    FN2_CHECK_ARG(valid(dst), "flow_to_tensor: dst is null or empty");
    FN2_CHECK_ARG((flags & ~FN2_FLOW_UINT16FLOW) == 0, "flow_to_tensor: unknown flags 0x%x", flags);
    T4 d = view(dst);
    FN2_CHECK_ARG(d.c == 2, "flow_to_tensor: dst must have 2 channels (u, v), has %d", d.c);
    const uint32_t* s = static_cast<const uint32_t*>(src_dev);
    const long long total = (long long)d.n * d.h * d.w;
    const int q = flags & FN2_FLOW_UINT16FLOW;
    if (format == FN2_FLOW_FLO) return ew_launch(flow_to_tensor_kernel<FN2_FLOW_FLO>, total, stream, s, px_view(d), q);
    if (format == FN2_FLOW_PFM) return ew_launch(flow_to_tensor_kernel<FN2_FLOW_PFM>, total, stream, s, px_view(d), q);
    if (format == FN2_FLOW_PFM_BE) return ew_launch(flow_to_tensor_kernel<FN2_FLOW_PFM_BE>, total, stream, s, px_view(d), q);
    return ew_launch(kitti_samples_to_tensor_kernel, total, stream, static_cast<const uint16_t*>(src_dev), px_view(d), q);
}

int fn2_flow_to_kitti_png_rows(const fn2_tensor* src, void* dst_dev, void* stream) {
    FN2_CHECK_ARG(valid(src), "flow_to_kitti_png_rows: src is null or empty");
    FN2_CHECK_ARG(dst_dev, "flow_to_kitti_png_rows: dst is null");
    FN2_CHECK_ARG((reinterpret_cast<uintptr_t>(src->data) & 3) == 0, "flow_to_kitti_png_rows: src must be 4-byte aligned");
    T4 f = view(src);
    FN2_CHECK_ARG(f.c == 2, "flow_to_kitti_png_rows: src must have 2 channels (u, v), has %d", f.c);
    return ew_launch(flow_to_kitti_png_rows_kernel, (long long)f.n * f.h * f.w, stream, f, static_cast<uint8_t*>(dst_dev));
}

int fn2_flow_max_radius(const fn2_tensor* src, float* max_dev, void* stream) {
    FN2_CHECK_ARG(valid(src), "flow_max_radius: src is null or empty");
    FN2_CHECK_ARG(max_dev, "flow_max_radius: max is null");
    FN2_CHECK_ARG((reinterpret_cast<uintptr_t>(src->data) & 3) == 0, "flow_max_radius: src must be 4-byte aligned");
    FN2_CHECK_ARG((reinterpret_cast<uintptr_t>(max_dev) & 3) == 0, "flow_max_radius: max must be 4-byte aligned");
    T4 f = view(src);
    FN2_CHECK_ARG(f.c == 2, "flow_max_radius: src must have 2 channels (u, v), has %d", f.c);
    FN2_CHECK_ARG(f.n <= 65535, "flow_max_radius: at most 65535 images, got %d", f.n);
    cudaStream_t s = (cudaStream_t)stream;
    fill_minus_one_kernel<<<(f.n + 255) / 256, 256, 0, s>>>(max_dev, f.n);
    FN2_LAUNCH_CHECK();
    const long long hw = (long long)f.h * f.w;
    const int blocks = (int)std::max(1LL, std::min((hw + 255) / 256, (long long)ew_grid(hw * f.n, 256) / f.n));
    flow_max_radius_kernel<<<dim3(blocks, f.n), 256, 0, s>>>(f, max_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

// The checks the two colour entry points share.
static int colour_args(const char* who, const fn2_tensor* src, const float* max_dev, const float* fallback_dev, float max_flow,
                       const void* dst_dev) {
    FN2_CHECK_ARG(valid(src), "%s: src is null or empty", who);
    FN2_CHECK_ARG(dst_dev, "%s: dst is null", who);
    FN2_CHECK_ARG((reinterpret_cast<uintptr_t>(src->data) & 3) == 0, "%s: src must be 4-byte aligned", who);
    FN2_CHECK_ARG(src->c == 2, "%s: src must have 2 channels (u, v), has %d", who, src->c);
    FN2_CHECK_ARG(max_flow == 0.f || (max_flow > 0.f && isfinite(max_flow)),
                  "%s: max_flow must be 0 (the per-image max) or finite and positive, got %g", who, (double)max_flow);
    FN2_CHECK_ARG(max_flow > 0.f || max_dev, "%s: max is null and max_flow is 0", who);
    FN2_CHECK_ARG(!((reinterpret_cast<uintptr_t>(max_dev) | reinterpret_cast<uintptr_t>(fallback_dev)) & 3),
                  "%s: max and fallback must be 4-byte aligned", who);
    return FN2_OK;
}

int fn2_flow_to_color(const fn2_tensor* src, const float* max_dev, const float* fallback_dev, float max_flow, void* dst_dev,
                      void* stream) {
    const int rc = colour_args("flow_to_color", src, max_dev, fallback_dev, max_flow, dst_dev);
    if (rc != FN2_OK) return rc;
    T4 f = view(src);
    return ew_launch(flow_to_color_kernel, (long long)f.n * f.h * f.w, stream, f, max_dev, fallback_dev, max_flow,
                     static_cast<uint8_t*>(dst_dev));
}

int fn2_flow_to_color_png_rows(const fn2_tensor* src, const float* max_dev, const float* fallback_dev, float max_flow,
                               void* dst_dev, void* stream) {
    const int rc = colour_args("flow_to_color_png_rows", src, max_dev, fallback_dev, max_flow, dst_dev);
    if (rc != FN2_OK) return rc;
    T4 f = view(src);
    return ew_launch(flow_to_color_png_rows_kernel, (long long)f.n * f.h * f.w, stream, f, max_dev, fallback_dev, max_flow,
                     static_cast<uint8_t*>(dst_dev));
}

int fn2_flow_fb_occlusion(const fn2_tensor* fwd, const fn2_tensor* bwd, float alpha1, float alpha2, void* out_dev,
                          size_t row_stride, size_t pair_stride, void* stream) {
    FN2_CHECK_ARG(valid(fwd) && valid(bwd), "flow_fb_occlusion: a flow is null or empty");
    FN2_CHECK_ARG(out_dev, "flow_fb_occlusion: out is null");
    FN2_CHECK_ARG(!((reinterpret_cast<uintptr_t>(fwd->data) | reinterpret_cast<uintptr_t>(bwd->data)) & 3),
                  "flow_fb_occlusion: the flows must be 4-byte aligned");
    const T4 f = view(fwd), b = view(bwd);
    FN2_CHECK_ARG(same_dims(f, b), "flow_fb_occlusion: fwd is %dx%dx%dx%d but bwd is %dx%dx%dx%d", f.n, f.c, f.h, f.w, b.n, b.c,
                  b.h, b.w);
    FN2_CHECK_ARG(f.c == 2, "flow_fb_occlusion: flows need 2 channels (u, v), got %d", f.c);
    FN2_CHECK_ARG(isfinite(alpha1) && alpha1 >= 0.f && isfinite(alpha2) && alpha2 >= 0.f,
                  "flow_fb_occlusion: alpha1 and alpha2 must be finite and non-negative, got %g and %g", (double)alpha1,
                  (double)alpha2);
    FN2_CHECK_ARG(row_stride >= (size_t)f.w, "flow_fb_occlusion: row stride %zu is below W = %d", row_stride, f.w);
    FN2_CHECK_ARG(pair_stride >= (size_t)f.h * row_stride, "flow_fb_occlusion: pair stride %zu is below H * row stride = %zu",
                  pair_stride, (size_t)f.h * row_stride);
    FN2_CHECK_ARG(f.n <= 65535, "flow_fb_occlusion: %d pairs, at most 65535", f.n);
    const long long hw = (long long)f.h * f.w;
    const int blocks = (int)std::max(1LL, std::min((hw + 255) / 256, (long long)ew_grid(hw * f.n, 256) / f.n));
    flow_fb_occlusion_kernel<<<dim3(blocks, f.n), 256, 0, (cudaStream_t)stream>>>(f, b, alpha1, alpha2, static_cast<uint8_t*>(out_dev),
                                                                                  (long long)row_stride, (long long)pair_stride);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // extern "C"
