// Correlation cost volume: CorrelationLayer (reference: src/caffe/layers/correlation_layer.{cpp,cu}) and Correlation1DLayer
// (correlation_layer1d.{cpp,cu}).
//
// Both layers have one geometry (CorrGeo, filled by corr_geometry): top pixel (x, y) compares the k x k patch of bottom0 at
// (x * stride_1 + md - pad, y * stride_1 + y0), in unpadded coordinates, with the bottom1 patch displaced by
//     dx = (tc mod Dx + xs) * stride_2,   dy = (tc div Dx + ys) * stride_2          for top channel tc.
// 2-D: (Dx, xs, ys) = (2R+1, -R, -R), y0 = md - pad (correlation_layer.cu:56-57, :81-82).  1-D: (D, x_shift, 0), y0 = 0: rows
// are neither padded nor displaced (correlation_layer1d.cu:56-57, :83).  R = md / stride_2.
//
// Forward routes, chosen by corr_fwd_plan (from the shape) and corr_fwd_route (from the layouts and the workspace):
//   * tc      -- FlowNet2-C's layer (MULTIPLY, k 1, stride_1 1, pad = md, R = 10, stride_2 <= 2, C % 32 == 0) on channel-fast
//                maps with 16-byte aligned pixels, when the workspace holds the TF32 copy of map 1: the conv engine's wgmma
//                pipeline (fn2_conv_tc.cu, corr_tc_forward).
//   * fast    -- the 2-D parameter class MULTIPLY, k 1, stride_1 1, pad = md, md % stride_2 == 0 with R = 10 or R = 4 and
//                C % 8 == 0, any layout: FP32 SIMT on the stride_2 parity planes (fn2_corr_fast.cu).  Needs the workspace
//                fn2_correlation_workspace_bytes reports; a non-null workspace that is too small is an error.
//   * generic -- every other shape, Correlation1D, and any call without workspace (this file): one CTA per output pixel like
//                the reference's CorrelateData (:46-114), but the zero padded NHWC copies (:24-42, :447-458) are never
//                materialised (a tap outside the image contributes a * 0) and the per-displacement reduction is a warp shuffle
//                instead of the reference's serial lane-0 sum (:101-105, which races with the next iteration's
//                `sum[ch_off] = 0` on post-Volta parts).
// The backward of both layers is fn2_corr_bwd.cu.
#include "fn2_common.cuh"

namespace fn2 {

bool corr_tc_available();
size_t corr_tc_workspace_floats(int N, int C, int H, int W);
int corr_tc_forward(const T4& b0, const T4& b1, const T4& top, int R, int s2, float* ws, cudaStream_t st);
size_t corr_fast_workspace_bytes(int N, int C, int H, int W, int R, int s2);
int corr_fast_forward(const T4& b0, const T4& b1, const T4& top, int R, int s2, void* ws, cudaStream_t st);
size_t corr_bwd_workspace_floats(const CorrGeo& g, int N, int C, int H, int W, int corr_type);
int corr_backward(const CorrGeo& g, const T4& b0, const T4& b1, const T4& td, const T4& d0, const T4& d1, int corr_type,
                  float* ws, size_t ws_floats, cudaStream_t st);

namespace {

const char* corr_name(int dims) { return dims == 2 ? "correlation" : "correlation1d"; }

// Validates the parameters of a Correlation (dims 2) or Correlation1D (dims 1) layer on H x W bottoms and fills its geometry.
int corr_geometry(int dims, int H, int W, int pad, int k, int md, int s1, int s2, int single_direction, CorrGeo* g) {
    const bool two = dims == 2;
    if (k < 1 || k % 2 == 0) {
        set_error("Odd kernel size required (%s:22)", two ? "correlation_layer.cpp" : "correlation_layer1d.cpp");
        return FN2_ERR_INVALID;
    }
    if (s1 < 1 || s2 < 1 || md < 0 || pad < 0) { set_error("%s: bad stride/displacement/pad", corr_name(dims)); return FN2_ERR_INVALID; }
    if (!two && (single_direction < -1 || single_direction > 1)) {
        set_error("single_direction must be -1 (left), 0 (off), or 1 (right)");
        return FN2_ERR_INVALID;
    }
    const int kr = (k - 1) / 2, border = md + kr;
    // correlation_layer.cpp:59-60; correlation_layer1d.cpp:55-56 (rows are not padded)
    const int w = (int)ceilf((float)(W + 2 * pad - border * 2) / (float)s1);
    const int h = two ? (int)ceilf((float)(H + 2 * pad - border * 2) / (float)s1) : (int)ceilf((float)(H - kr * 2) / (float)s1);
    if (w < 1 || h < 1) {
        set_error(two ? "Correlation cannot be done with current settings. Neighborhood and kernel don't fit in blob "
                        "(correlation_layer.cpp:62-63)"
                      : "Correlation cannot be done with current settings. Neighborhood and kernel don't fit in blob");
        return FN2_ERR_INVALID;
    }
    const int R = md / s2;
    g->dims = dims;
    g->topH = h; g->topW = w;
    g->k = k; g->s1 = s1; g->md = md; g->pad = pad; g->s2 = s2; g->R = R;
    if (two) {
        g->y0 = md - pad;
        g->Dx = 2 * R + 1; g->xs = g->ys = -R;
        g->topC = g->Dx * g->Dx;
    } else {
        g->y0 = 0;
        g->Dx = single_direction != 0 ? R + 1 : 2 * R + 1;                    // correlation_layer1d.cpp:64-68
        // correlation_layer1d.cu Forward_gpu: -R, "to the left" -grid_width (sic: one stride_2 step beyond -max_displacement),
        // "to the right" 0
        g->xs = single_direction == 1 ? 0 : (single_direction == -1 ? -(R + 1) : -R);
        g->ys = 0;
        g->topC = g->Dx;
    }
    return FN2_OK;
}

// One CTA (4 warps) per output pixel.  Patch of bottom0 staged in shared memory; each warp owns
// displacements tc = warp, warp+4, ...; lanes stride the channel dimension.
__global__ void __launch_bounds__(128) corr_generic_kernel(T4 b0, T4 b1, T4 top, CorrGeo g, int type) {
    extern __shared__ float patch[];                  // [k*k][C]
    const int x = blockIdx.x, y = blockIdx.y, n = blockIdx.z;
    const int C = b0.c, H = b0.h, W = b0.w;
    // upper-left of the patch in UNPADDED coordinates: padded x1 = x*s1 + md (:56), minus pad
    const int x1 = x * g.s1 + g.md - g.pad;
    const int y1 = y * g.s1 + g.y0;
    for (int idx = threadIdx.x; idx < g.k * g.k * C; idx += blockDim.x) {
        const int ch = idx % C, ji = idx / C;
        const int j = ji / g.k, i = ji % g.k;
        const int yy = y1 + j, xx = x1 + i;
        patch[idx] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? b0.p[b0.off(n, ch, yy, xx)] : 0.f;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sumelems = g.k * g.k * C;
    for (int tc = warp; tc < g.topC; tc += 4) {
        const int s2o = (tc % g.Dx + g.xs) * g.s2;     // :81
        const int s2p = (tc / g.Dx + g.ys) * g.s2;     // :82
        float acc = 0.f;
        for (int j = 0; j < g.k; j++) {
            const int yy = y1 + s2p + j;
            for (int i = 0; i < g.k; i++) {
                const int xx = x1 + s2o + i;
                const bool inb = (yy >= 0 && yy < H && xx >= 0 && xx < W);
                const float* ap = patch + (j * g.k + i) * C;
                if (type == 0) {
                    if (!inb) {
                        // a * 0, as the reference's zero-padded copy: nothing for a finite a, NaN for a non-finite one
                        for (int ch = lane; ch < C; ch += 32) acc = fmaf(ap[ch], 0.f, acc);
                        continue;
                    }
                    const float* bp = b1.p + b1.off(n, 0, yy, xx);
                    for (int ch = lane; ch < C; ch += 32) acc = fmaf(ap[ch], __ldg(bp + ch * b1.sc), acc);
                } else if (inb) {
                    const float* bp = b1.p + b1.off(n, 0, yy, xx);
                    for (int ch = lane; ch < C; ch += 32) acc += fabsf(ap[ch] - __ldg(bp + ch * b1.sc));
                } else {
                    for (int ch = lane; ch < C; ch += 32) acc += fabsf(ap[ch]);   // |a - 0|
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) top.p[top.off(n, tc, y, x)] = acc / (float)sumelems;   // :106-108
    }
}

enum class CorrRoute { generic, tc, fast };

struct CorrFwdPlan {
    CorrRoute route;        // generic or fast: the tensor-core route is chosen from the layouts (corr_fwd_route)
    size_t ws_bytes;        // the fast route's parity-planar copies of both maps; 0 for the generic route
};

// Shape part of the forward route: the FP32 fast route's parameter class and its workspace.
CorrFwdPlan corr_fwd_plan(const CorrGeo& g, int N, int C, int H, int W, int corr_type) {
    const bool fast = g.dims == 2 && corr_type == 0 && g.k == 1 && g.s1 == 1 && g.pad == g.md && g.md % g.s2 == 0 &&
                      (g.R == 10 || g.R == 4) &&                       // the radii corr_fast_kernel is instantiated for
                      C % 8 == 0 &&                                    // channels per pipeline stage
                      (long long)N * g.s2 * g.s2 <= 65535LL * 1024;
    if (!fast) return {CorrRoute::generic, 0};
    return {CorrRoute::fast, corr_fast_workspace_bytes(N, C, H, W, g.R, g.s2)};
}

// Layout and workspace part.  A null workspace runs the generic kernel.  Otherwise the R = 10 class runs on the tensor cores
// when the maps are channel-fast with 16-byte aligned pixels, C % 32 == 0, stride_2 <= 2 and the workspace holds the
// tensor-core need (which never exceeds the fast route's); else the fast route runs, and a workspace too small for it is an
// error.
int corr_fwd_route(const CorrFwdPlan& pl, const CorrGeo& g, const T4& b0, const T4& b1, const T4& top, const void* ws,
                   size_t ws_bytes, CorrRoute* route) {
    *route = pl.route;
    if (pl.route == CorrRoute::generic) return FN2_OK;
    if (ws && g.R == 10 && g.s2 <= 2 && b0.c % 32 == 0 && b0.px_float4() && b1.px_float4() && top.sc == 1 &&
        corr_tc_available() && ws_bytes >= corr_tc_workspace_floats(b0.n, b0.c, b0.h, b0.w) * sizeof(float)) {
        *route = CorrRoute::tc;
        return FN2_OK;
    }
    if (ws && ws_bytes >= pl.ws_bytes) return FN2_OK;
    if (ws || ws_bytes) {
        set_error("correlation: workspace too small (%zu < %zu)", ws_bytes, pl.ws_bytes);
        return FN2_ERR_WORKSPACE;
    }
    *route = CorrRoute::generic;
    return FN2_OK;
}

int corr_forward(int dims, const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top, int pad, int k, int md,
                 int s1, int s2, int single_direction, int corr_type, void* ws, size_t ws_bytes, void* stream) {
    const char* name = corr_name(dims);
    FN2_CHECK_ARG(valid(bottom0) && valid(bottom1) && valid(top), "%s: null/empty tensor", name);
    const T4 b0 = view(bottom0), b1 = view(bottom1), tp = view(top);
    FN2_CHECK_ARG(same_dims(b0, b1), "Both bottom blobs must have same shape (%s)",
                  dims == 2 ? "correlation_layer.cpp:46-48" : "correlation_layer1d.cpp:44-46");
    FN2_CHECK_ARG(corr_type == 0 || corr_type == 1, "%s: unknown correlation_type %d", name, corr_type);
    CorrGeo g;
    int rc = corr_geometry(dims, b0.h, b0.w, pad, k, md, s1, s2, single_direction, &g);
    if (rc) return rc;
    FN2_CHECK_ARG(tp.n == b0.n && tp.c == g.topC && tp.h == g.topH && tp.w == g.topW, "%s: top must be (%d,%d,%d,%d)", name, b0.n,
                  g.topC, g.topH, g.topW);
    const CorrFwdPlan pl = corr_fwd_plan(g, b0.n, b0.c, b0.h, b0.w, corr_type);
    CorrRoute route;
    rc = corr_fwd_route(pl, g, b0, b1, tp, ws, ws_bytes, &route);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (route == CorrRoute::tc) return corr_tc_forward(b0, b1, tp, g.R, g.s2, (float*)ws, st);
    if (route == CorrRoute::fast) return corr_fast_forward(b0, b1, tp, g.R, g.s2, ws, st);
    const size_t smem = (size_t)k * k * b0.c * sizeof(float);
    FN2_CHECK_ARG(smem <= 200 * 1024, "%s: k*k*C patch does not fit in shared memory", name);
    if (smem > 48 * 1024)
        FN2_CUDA(cudaFuncSetAttribute(corr_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_generic_kernel<<<dim3(g.topW, g.topH, b0.n), 128, smem, st>>>(b0, b1, tp, g, corr_type);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int corr_backward_entry(int dims, const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top_diff,
                        const fn2_tensor* bottom0_diff, const fn2_tensor* bottom1_diff, int pad, int k, int md, int s1, int s2,
                        int single_direction, int corr_type, void* ws, size_t ws_bytes, void* stream) {
    const char* name = dims == 2 ? "correlation_backward" : "correlation1d_backward";
    FN2_CHECK_ARG(valid(bottom0) && valid(bottom1) && valid(top_diff) && valid(bottom0_diff) && valid(bottom1_diff),
                  "%s: null/empty tensor", name);
    const T4 b0 = view(bottom0), b1 = view(bottom1), td = view(top_diff), d0 = view(bottom0_diff), d1 = view(bottom1_diff);
    FN2_CHECK_ARG(same_dims(b0, b1) && same_dims(b0, d0) && same_dims(b0, d1), "%s: bottom shape mismatch", name);
    FN2_CHECK_ARG(corr_type == 0 || corr_type == 1, "%s: unknown correlation_type %d", name, corr_type);
    FN2_CHECK_ARG(corr_type == 0 || pad <= md, "%s: SUBTRACT needs pad <= max_displacement (the reference reads past its padded "
                  "buffers otherwise)", name);
    CorrGeo g;
    int rc = corr_geometry(dims, b0.h, b0.w, pad, k, md, s1, s2, single_direction, &g);
    if (rc) return rc;
    FN2_CHECK_ARG(td.n == b0.n && td.c == g.topC && td.h == g.topH && td.w == g.topW, "%s: top_diff shape mismatch", name);
    return corr_backward(g, b0, b1, td, d0, d1, corr_type, (float*)ws, ws_bytes / sizeof(float), (cudaStream_t)stream);
}

int corr_shape_entry(int dims, int H, int W, int pad, int k, int md, int s1, int s2, int single_direction, int* top_channels,
                     int* top_h, int* top_w) {
    CorrGeo g;
    int rc = corr_geometry(dims, H, W, pad, k, md, s1, s2, single_direction, &g);
    if (rc) return rc;
    if (top_channels) *top_channels = g.topC;
    if (top_h) *top_h = g.topH;
    if (top_w) *top_w = g.topW;
    return FN2_OK;
}

int corr_bwd_workspace_entry(int dims, int N, int C, int H, int W, int pad, int k, int md, int s1, int s2, int single_direction,
                             int corr_type, size_t* bytes) {
    CorrGeo g;
    int rc = corr_geometry(dims, H, W, pad, k, md, s1, s2, single_direction, &g);
    if (rc) return rc;
    *bytes = corr_bwd_workspace_floats(g, N, C, H, W, corr_type) * sizeof(float);
    return FN2_OK;
}

}  // namespace
}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2_correlation_shape(int H, int W, int pad, int kernel_size, int max_displacement, int stride1,
                          int stride2, int* top_channels, int* top_h, int* top_w) {
    return corr_shape_entry(2, H, W, pad, kernel_size, max_displacement, stride1, stride2, 0, top_channels, top_h, top_w);
}

int fn2_correlation_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size,
                                    int max_displacement, int stride1, int stride2, int corr_type,
                                    size_t* bytes) {
    FN2_CHECK_ARG(bytes, "correlation_workspace_bytes: null out pointer");
    *bytes = 0;
    CorrGeo g;
    int rc = corr_geometry(2, H, W, pad, kernel_size, max_displacement, stride1, stride2, 0, &g);
    if (rc) return rc;
    *bytes = corr_fwd_plan(g, N, C, H, W, corr_type).ws_bytes;
    return FN2_OK;
}

int fn2_correlation_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top,
                            int pad, int kernel_size, int max_displacement, int stride1, int stride2,
                            int corr_type, void* workspace, size_t workspace_bytes, void* stream) {
    return corr_forward(2, bottom0, bottom1, top, pad, kernel_size, max_displacement, stride1, stride2, 0, corr_type, workspace,
                        workspace_bytes, stream);
}

int fn2_correlation_backward_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size, int max_displacement,
                                             int stride1, int stride2, int corr_type, size_t* bytes) {
    FN2_CHECK_ARG(bytes, "correlation_backward_workspace_bytes: null out pointer");
    return corr_bwd_workspace_entry(2, N, C, H, W, pad, kernel_size, max_displacement, stride1, stride2, 0, corr_type, bytes);
}

int fn2_correlation_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1,
                             const fn2_tensor* top_diff, const fn2_tensor* bottom0_diff,
                             const fn2_tensor* bottom1_diff, int pad, int kernel_size,
                             int max_displacement, int stride1, int stride2, int corr_type,
                             void* workspace, size_t workspace_bytes, void* stream) {
    return corr_backward_entry(2, bottom0, bottom1, top_diff, bottom0_diff, bottom1_diff, pad, kernel_size, max_displacement,
                               stride1, stride2, 0, corr_type, workspace, workspace_bytes, stream);
}

/* Correlation1D (correlation_layer1d.{cpp,cu}): displacement along x only; single_direction -1 left, 0 both, +1 right. */
int fn2_correlation1d_shape(int H, int W, int pad, int kernel_size, int max_displacement, int stride1, int stride2,
                            int single_direction, int* top_channels, int* top_h, int* top_w) {
    return corr_shape_entry(1, H, W, pad, kernel_size, max_displacement, stride1, stride2, single_direction, top_channels, top_h,
                            top_w);
}

int fn2_correlation1d_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top, int pad, int kernel_size,
                              int max_displacement, int stride1, int stride2, int single_direction, int corr_type, void* stream) {
    return corr_forward(1, bottom0, bottom1, top, pad, kernel_size, max_displacement, stride1, stride2, single_direction, corr_type,
                        nullptr, 0, stream);
}

int fn2_correlation1d_backward_workspace_bytes(int N, int C, int H, int W, int pad, int kernel_size, int max_displacement, int stride1,
                                               int stride2, int single_direction, int corr_type, size_t* bytes) {
    FN2_CHECK_ARG(bytes, "correlation1d_backward_workspace_bytes: null out pointer");
    return corr_bwd_workspace_entry(1, N, C, H, W, pad, kernel_size, max_displacement, stride1, stride2, single_direction,
                                    corr_type, bytes);
}

int fn2_correlation1d_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_tensor* top_diff,
                               const fn2_tensor* bottom0_diff, const fn2_tensor* bottom1_diff, int pad, int kernel_size,
                               int max_displacement, int stride1, int stride2, int single_direction, int corr_type,
                               void* workspace, size_t workspace_bytes, void* stream) {
    return corr_backward_entry(1, bottom0, bottom1, top_diff, bottom0_diff, bottom1_diff, pad, kernel_size, max_displacement,
                               stride1, stride2, single_direction, corr_type, workspace, workspace_bytes, stream);
}

}  // extern "C"
