// Scoring a predicted flow against ground truth (include/fn2_eval.h): per pair, the valid-pixel count, the EPE sum, KITTI's Fl
// outliers, the non-finite predictions and the three Sintel speed bands, in one pass over both flows.
//
// flow_error_kernel: grid (blocks per pair, N); each thread visits its pair's pixels in a fixed grid-stride order and keeps the
// ten fields in double registers; the block folds them with warp butterflies and a fixed-order sum over its warps into one
// partial record.  flow_error_final_kernel adds each pair's partials in block order.  The per-pixel arithmetic is float32 and
// this file is compiled with -fmad=false (flownet2_b200/build.py), so a float32 restatement on the host reproduces every EPE,
// |gt|, band and outlier decision bit for bit; only the order of the double sums differs.  The pass reads 16 bytes per pixel
// (two float2) and writes nothing per pixel: it is bound by HBM traffic.
#include <math.h>

#include "fn2_common.cuh"
#include "../../include/fn2_eval.h"

namespace fn2 {

namespace {

constexpr int kFields = FN2_FLOW_ERROR_FIELDS;
constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr float kUnknownFlow = 1e9f;                                    // Middlebury's UNKNOWN_FLOW_THRESH

// Adds one pixel (ground truth gu, gv; prediction pu, pv) to the ten fields.
__device__ __forceinline__ void score_pixel(float gu, float gv, float pu, float pv, double (&acc)[kFields]) {
    if (!(fabsf(gu) <= kUnknownFlow && fabsf(gv) <= kUnknownFlow)) return;          // NaN, Inf or unknown: not counted
    acc[FN2_FLOW_ERROR_VALID] += 1.0;
    if (!(isfinite(pu) && isfinite(pv))) {
        acc[FN2_FLOW_ERROR_NONFINITE] += 1.0;
        return;
    }
    const float du = pu - gu, dv = pv - gv;
    const float epe = sqrtf(du * du + dv * dv);
    const float mag = sqrtf(gu * gu + gv * gv);
    acc[FN2_FLOW_ERROR_EPE_SUM] += (double)epe;
    if (epe > 3.f && epe > 0.05f * mag) acc[FN2_FLOW_ERROR_OUTLIERS] += 1.0;
    if (mag < 10.f) {
        acc[FN2_FLOW_ERROR_N_S0_10] += 1.0; acc[FN2_FLOW_ERROR_SUM_S0_10] += (double)epe;
    } else if (mag < 40.f) {
        acc[FN2_FLOW_ERROR_N_S10_40] += 1.0; acc[FN2_FLOW_ERROR_SUM_S10_40] += (double)epe;
    } else {
        acc[FN2_FLOW_ERROR_N_S40] += 1.0; acc[FN2_FLOW_ERROR_SUM_S40] += (double)epe;
    }
}

// Each step of a thread covers kUnroll pixels kThreads apart: their 4 * kUnroll loads are issued before any is scored, so a
// thread keeps that many reads in flight.  A pixel beyond the pair reads as invalid ground truth.
__global__ void __launch_bounds__(kThreads) flow_error_kernel(T4 pred, T4 gt, double* __restrict__ part /* [N][bpp][kFields] */) {
    const int n = blockIdx.y;
    const int hw = pred.h * pred.w;
    double acc[kFields];
#pragma unroll
    for (int f = 0; f < kFields; f++) acc[f] = 0.0;
    for (int i0 = blockIdx.x * kThreads * kUnroll + threadIdx.x; i0 < hw; i0 += gridDim.x * kThreads * kUnroll) {
        float v[kUnroll][4];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const int i = i0 + u * kThreads;
            if (i < hw) {
                const int y = i / pred.w, x = i - y * pred.w;
                v[u][0] = __ldg(gt.p + gt.off(n, 0, y, x)); v[u][1] = __ldg(gt.p + gt.off(n, 1, y, x));
                v[u][2] = __ldg(pred.p + pred.off(n, 0, y, x)); v[u][3] = __ldg(pred.p + pred.off(n, 1, y, x));
            } else {
                v[u][0] = v[u][1] = v[u][2] = v[u][3] = __int_as_float(0x7fffffff);
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++) score_pixel(v[u][0], v[u][1], v[u][2], v[u][3], acc);
    }
    __shared__ double warp_sum[kThreads / 32][kFields];
#pragma unroll
    for (int f = 0; f < kFields; f++) {
        for (int o = 16; o; o >>= 1) acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], o);
        if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5][f] = acc[f];
    }
    __syncthreads();
    if (threadIdx.x < kFields) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; w++) s += warp_sum[w][threadIdx.x];
        part[((long long)n * gridDim.x + blockIdx.x) * kFields + threadIdx.x] = s;
    }
}

// One thread per (pair, field): the pair's block partials added in block order.
__global__ void flow_error_final_kernel(const double* __restrict__ part, int N, int bpp, double* __restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * kFields) return;
    const int n = t / kFields, f = t - n * kFields;
    double s = 0.0;
    for (int b = 0; b < bpp; b++) s += part[((long long)n * bpp + b) * kFields + f];
    out[t] = s;
}

// Blocks per pair: enough to cover the pair's pixels, at most one wave of resident blocks over all N pairs (a second, partial
// wave would leave most of the device idle while it runs).
int eval_blocks(int N, int H, int W) {
    static int per_sm = 0;
    if (!per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flow_error_kernel, kThreads, 0) != cudaSuccess ||
                    per_sm < 1)) {
        cudaGetLastError();
        per_sm = 1;
    }
    const long long need = ((long long)H * W + kThreads * kUnroll - 1) / (kThreads * kUnroll);
    const long long cap = max(1LL, (long long)num_sms() * per_sm / N);
    return (int)max(1LL, min(need, cap));
}

}  // namespace
}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2_flow_error_workspace_bytes(int N, int H, int W, size_t* bytes) {
    FN2_CHECK_ARG(bytes && N > 0 && H > 0 && W > 0, "flow_error_workspace_bytes: bad argument");
    *bytes = (size_t)N * eval_blocks(N, H, W) * kFields * sizeof(double);
    return FN2_OK;
}

int fn2_flow_error(const fn2_tensor* pred, const fn2_tensor* gt, double* out_dev, void* workspace, size_t workspace_bytes,
                   void* stream) {
    FN2_CHECK_ARG(valid(pred) && valid(gt) && out_dev, "flow_error: null argument");
    const T4 p = view(pred), g = view(gt);
    FN2_CHECK_ARG(same_dims(p, g), "flow_error: pred is %dx%dx%dx%d but gt is %dx%dx%dx%d", p.n, p.c, p.h, p.w, g.n, g.c, g.h, g.w);
    FN2_CHECK_ARG(p.c == 2, "flow_error: flows need 2 channels, got %d", p.c);
    FN2_CHECK_ARG(p.n <= 65535 && (long long)p.h * p.w <= (1LL << 30), "flow_error: %d pairs of %dx%d is too large", p.n, p.w, p.h);
    const int bpp = eval_blocks(p.n, p.h, p.w);
    const size_t need = (size_t)p.n * bpp * kFields * sizeof(double);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 7)) {
        set_error("flow_error: workspace too small or not 8-byte aligned (%zu bytes, %zu needed)", workspace_bytes, need);
        return FN2_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    flow_error_kernel<<<dim3(bpp, p.n), kThreads, 0, st>>>(p, g, (double*)workspace);
    FN2_LAUNCH_CHECK();
    const int total = p.n * kFields;
    flow_error_final_kernel<<<(total + 127) / 128, 128, 0, st>>>((const double*)workspace, p.n, bpp, out_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // extern "C"
