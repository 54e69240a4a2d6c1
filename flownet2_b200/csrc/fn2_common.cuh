// Shared device/host helpers for libfn2.so kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/fn2.h"

namespace fn2 {

// Thread-local last error + launch counter (fn2_last_error / fn2_launch_count).
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define FN2_CHECK_ARG(cond, ...)                     \
    do {                                             \
        if (!(cond)) {                               \
            ::fn2::set_error(__VA_ARGS__);           \
            return FN2_ERR_INVALID;                  \
        }                                            \
    } while (0)

#define FN2_CUDA(call)                                                              \
    do {                                                                            \
        cudaError_t e__ = (call);                                                   \
        if (e__ != cudaSuccess) {                                                   \
            ::fn2::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                             __FILE__, __LINE__);                                   \
            return FN2_ERR_CUDA;                                                    \
        }                                                                           \
    } while (0)

#define FN2_LAUNCH_CHECK()                                                          \
    do {                                                                            \
        ::fn2::count_launch();                                                      \
        cudaError_t e__ = cudaGetLastError();                                       \
        if (e__ != cudaSuccess) {                                                   \
            ::fn2::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), \
                             __FILE__, __LINE__);                                   \
            return FN2_ERR_CUDA;                                                    \
        }                                                                           \
    } while (0)

// Device-side view of fn2_tensor (passed by value to kernels).
struct T4 {
    float* p;
    int n, c, h, w;
    long long sn, sc, sh, sw;
    __host__ __device__ __forceinline__ long long off(int in, int ic, int ih, int iw) const {
        return in * sn + ic * sc + ih * sh + iw * sw;
    }
    __host__ __device__ __forceinline__ long long count() const { return (long long)n * c * h * w; }
    __host__ __device__ bool is_nchw() const {
        return sw == 1 && sh == w && sc == (long long)h * w && sn == (long long)c * h * w;
    }
    // channel-contiguous ("NHWC") with arbitrary pixel stride sw >= c
    __host__ __device__ bool is_nhwc() const {
        return sc == 1 && sh == (long long)w * sw && sn == (long long)h * w * sw;
    }
    // every pixel starts on a 16-byte boundary with its channels contiguous, so it can be read as float4 groups; how many
    // groups a pixel may be read as (its extent) is for the caller to check
    bool px_float4() const {
        return sc == 1 && !((uintptr_t)p & 15) && !(sn & 3) && !(sh & 3) && !(sw & 3);
    }
    // every pixel can be read as ceil(c/4) float4 groups (lanes beyond c are padding or a neighbour's channels)
    bool px_float4_groups() const { return px_float4() && sw >= 4 * ((c + 3) / 4); }
};

inline T4 view(const fn2_tensor* t) {
    T4 v;
    v.p = t->data; v.n = t->n; v.c = t->c; v.h = t->h; v.w = t->w;
    v.sn = t->sn; v.sc = t->sc; v.sh = t->sh; v.sw = t->sw;
    return v;
}
inline bool same_dims(const T4& a, const T4& b) {
    return a.n == b.n && a.c == b.c && a.h == b.h && a.w == b.w;
}
inline bool valid(const fn2_tensor* t) {
    return t && t->data && t->n > 0 && t->c > 0 && t->h > 0 && t->w > 0;
}

// Output parity classes and kernel-tap table of a convolution or deconvolution (fn2_conv.cu), shared by the per-tap engines.
// Class c covers the output pixels (u*ou + oy0[c], v*ov + ox0[c]), u < Hu[c], v < Wu[c]; its taps t = tap0[c] ..
// tap0[c] + ntaps[c] - 1 read the input at (u*stride_h + dy[t], v*stride_w + dx[t]) (stride 1 for a deconvolution) with the
// weights of kernel position widx[t].  A convolution is one class with all taps.  A deconvolution (gather form of col2im,
// util/im2col.cpp:158-190) has one class per output parity (oy mod stride_h, ox mod stride_w) present in the output, holding
// the taps that reach it: every tap belongs to exactly one class, and a class may have none.
// Needs kh*kw <= 49 and, for a deconvolution, stride_h*stride_w <= 16.
struct ConvTaps {
    int ncls, ou, ov;
    int Hu[16], Wu[16], oy0[16], ox0[16], tap0[16], ntaps[16];
    short dy[49], dx[49], widx[49];
};
void conv_taps(const fn2_conv_desc* d, int Ho, int Wo, ConvTaps* c);

// Geometry of a Correlation (dims 2) or Correlation1D (dims 1) layer (fn2_corr.cu, corr_geometry): top pixel (x, y) compares
// the k x k patch of bottom0 at (x*s1 + md - pad, y*s1 + y0) with the bottom1 patch displaced by
// ((tc % Dx + xs) * s2, (tc / Dx + ys) * s2) for top channel tc; R = md / s2.
struct CorrGeo {
    int dims;
    int topC, topH, topW;
    int k, s1, md, pad, y0;
    int Dx, xs, ys, s2, R;
};

inline int num_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}
// Grid for grid-stride elementwise kernels: enough CTAs to cover, capped at a multiple of the
// SM count (132 SMs x 8 resident 256-thread CTAs).
inline int ew_grid(long long total, int block) {
    long long need = (total + block - 1) / block;
    long long cap = (long long)num_sms() * 8;
    return (int)(need < cap ? (need > 0 ? need : 1) : cap);
}
// Launches kernel over total work items (ew_grid(total, 256) CTAs of 256 threads) on stream: FN2_OK or the launch error.
template <class... P, class... A>
inline int ew_launch(void (*kernel)(P...), long long total, void* stream, const A&... args) {
    kernel<<<ew_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(args...);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

// A known flow pixel (Middlebury's rule, UNKNOWN_FLOW_THRESH = 1e9): both components finite and at most 1e9 in absolute value.
// A ground-truth pixel is scored (fn2_eval.cu) and a flow pixel is coloured (fn2_ops.cu) only when it is known.
constexpr float kUnknownFlow = 1e9f;
__device__ __forceinline__ bool flow_known(float u, float v) {
    return fabsf(u) <= kUnknownFlow && fabsf(v) <= kUnknownFlow;                   // false for NaN, Inf and unknown
}

// Grid-stride loops of the per-pixel and per-element kernels.  Each thread visits the same indices in the same order whatever
// the kernel does with them, so per-thread partial sums (L1Loss, the eigenspace statistics) and index-seeded noise stay fixed.
// f(n, y, x) for every pixel of an n x h x w extent, x fastest.
template <class F>
__device__ __forceinline__ void for_each_pixel(int n, int h, int w, const F& f) {
    const long long total = (long long)n * h * w;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x)
        f((int)(idx / ((long long)w * h)), (int)((idx / w) % h), (int)(idx % w));
}
// (n, c, y, x) of element i of t in NCHW-logical order (x fastest, then y, c, n)
struct Idx4 { int n, c, y, x; };
__device__ __forceinline__ Idx4 nchw_index(const T4& t, long long i) {
    Idx4 r;
    r.x = (int)(i % t.w); i /= t.w;
    r.y = (int)(i % t.h); i /= t.h;
    r.c = (int)(i % t.c); r.n = (int)(i / t.c);
    return r;
}
// f(e, idx) for every element of t: e its (n, c, y, x), idx its NCHW-logical linear index
template <class F>
__device__ __forceinline__ void for_each_element(const T4& t, const F& f) {
    const long long total = t.count();
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x)
        f(nchw_index(t, idx), idx);
}

}  // namespace fn2
