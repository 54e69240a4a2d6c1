// Scoring a predicted flow against ground truth (include/fn2_eval.h): per pair, the valid-pixel count, the EPE sum, KITTI's Fl
// outliers, the non-finite predictions and the three Sintel speed bands, in one pass over both flows; the same scores by region
// (occlusion, distance to the occlusion boundary, object map) in a second pass; the boundary distance itself; and the
// confusion counts of a predicted occlusion mask against a ground-truth one.
//
// flow_error_kernel: grid (blocks per pair, N); each thread visits its pair's pixels in a fixed grid-stride order and keeps the
// ten fields in double registers; the block folds them with warp butterflies and a fixed-order sum over its warps into one
// partial record.  final_kernel adds each pair's partials in block order.  The per-pixel arithmetic is float32 and
// this file is compiled with -fmad=false (flownet2_b200/build.py), so a float32 restatement on the host reproduces every EPE,
// |gt|, band and outlier decision bit for bit; only the order of the double sums differs.  The pass reads 16 bytes per pixel
// (two float2) and writes nothing per pixel: it is bound by HBM traffic.  flow_region_kernel is the same pass over the 21
// region fields; it also reads the masks' bytes and the int32 boundary distance, 22 bytes per pixel with both masks.
//
// The boundary distance is an exact Euclidean distance transform in two separable passes, all in integers.
// boundary_column_kernel, one thread per column (a warp's loads are consecutive bytes of a row): a downward sweep finds the
// boundary pixels from the mask and writes each pixel's distance to the nearest one at or above it, an upward sweep folds in
// the nearest one below and writes the vertical distance squared (FN2_DIST2_NONE for a column without a boundary pixel).
// boundary_row_kernel, one block per row: the row is staged in shared memory, one thread builds the lower envelope of the
// parabolas (x - i)^2 + g(i) of the row's columns (Meijster, Roerdink and Hesselink, 2000: the integer separator
// (u^2 - i^2 + g(u) - g(i)) div 2(u - i)), and every thread fills its pixels by a binary search of the envelope's segments.
// The output plane holds the first pass's result, so no workspace is needed.
#include <math.h>

#include "fn2_common.cuh"
#include "../../include/fn2_eval.h"

namespace fn2 {

namespace {

constexpr int kFields = FN2_FLOW_ERROR_FIELDS;
constexpr int kRegionFields = FN2_FLOW_REGION_FIELDS;
constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kNone = FN2_DIST2_NONE;
constexpr int kMaxSide = 16384;                                         // (2 * 16383^2 < 2^31: every dist2 fits in int32)
constexpr int kColThreads = 32;                                         // a Sintel batch's 8 x 1024 columns: 256 blocks
constexpr int kChunk = 8;
constexpr int kRowThreads = 64;

// fn2_flow_error's definitions, shared by both scoring kernels: a pixel counts when its ground truth is valid (flow_known,
// fn2_common.cuh) and its prediction finite; its EPE and |gt| are float32 with separately rounded products; it is an outlier
// (KITTI's Fl) when EPE > 3 and EPE > 5 % of |gt|.
__device__ __forceinline__ float pixel_epe(float gu, float gv, float pu, float pv) {
    const float du = pu - gu, dv = pv - gv;
    return sqrtf(du * du + dv * dv);
}
__device__ __forceinline__ float gt_mag(float gu, float gv) { return sqrtf(gu * gu + gv * gv); }
__device__ __forceinline__ bool outlier(float epe, float mag) { return epe > 3.f && epe > 0.05f * mag; }

// Adds one pixel (ground truth gu, gv; prediction pu, pv) to the ten fields.
__device__ __forceinline__ void score_pixel(float gu, float gv, float pu, float pv, double (&acc)[kFields]) {
    if (!flow_known(gu, gv)) return;
    acc[FN2_FLOW_ERROR_VALID] += 1.0;
    if (!(isfinite(pu) && isfinite(pv))) {
        acc[FN2_FLOW_ERROR_NONFINITE] += 1.0;
        return;
    }
    const float epe = pixel_epe(gu, gv, pu, pv);
    const float mag = gt_mag(gu, gv);
    acc[FN2_FLOW_ERROR_EPE_SUM] += (double)epe;
    if (outlier(epe, mag)) acc[FN2_FLOW_ERROR_OUTLIERS] += 1.0;
    if (mag < 10.f) {
        acc[FN2_FLOW_ERROR_N_S0_10] += 1.0; acc[FN2_FLOW_ERROR_SUM_S0_10] += (double)epe;
    } else if (mag < 40.f) {
        acc[FN2_FLOW_ERROR_N_S10_40] += 1.0; acc[FN2_FLOW_ERROR_SUM_S10_40] += (double)epe;
    } else {
        acc[FN2_FLOW_ERROR_N_S40] += 1.0; acc[FN2_FLOW_ERROR_SUM_S40] += (double)epe;
    }
}

// A counted pixel into the region whose count is at index R (its EPE sum at R + 1, its outliers at R + 2).  R is a template
// argument so that acc stays in registers.
template <int R>
__device__ __forceinline__ void add_region(double epe, double out, double (&acc)[kRegionFields]) {
    acc[R] += 1.0; acc[R + 1] += epe; acc[R + 2] += out;
}

// Adds one pixel to the 21 region fields: occluded (occ) and its boundary distance squared (d2) when has_occ, foreground (fg)
// when has_obj.
__device__ __forceinline__ void score_region(float gu, float gv, float pu, float pv, bool has_occ, bool occ, int d2, bool has_obj,
                                             bool fg, double (&acc)[kRegionFields]) {
    if (!(flow_known(gu, gv) && isfinite(pu) && isfinite(pv))) return;
    const float epe = pixel_epe(gu, gv, pu, pv);
    const double e = (double)epe, o = outlier(epe, gt_mag(gu, gv)) ? 1.0 : 0.0;
    if (has_occ) {
        if (occ) add_region<FN2_FLOW_REGION_N_UNMATCHED>(e, o, acc);
        else add_region<FN2_FLOW_REGION_N_MATCHED>(e, o, acc);
        if (d2 < 100) add_region<FN2_FLOW_REGION_N_D0_10>(e, o, acc);
        else if (d2 < 3600) add_region<FN2_FLOW_REGION_N_D10_60>(e, o, acc);
        else if (d2 < 19600) add_region<FN2_FLOW_REGION_N_D60_140>(e, o, acc);
    }
    if (has_obj) {
        if (fg) add_region<FN2_FLOW_REGION_N_FG>(e, o, acc);
        else add_region<FN2_FLOW_REGION_N_BG>(e, o, acc);
    }
}

// The block's F fields (each thread's acc) folded into its partial record part[n][blockIdx.x]: warp butterflies, then the warps
// in index order.
template <int F>
__device__ __forceinline__ void block_partial(double (&acc)[F], int n, double* __restrict__ part) {
    __shared__ double warp_sum[kThreads / 32][F];
#pragma unroll
    for (int f = 0; f < F; f++) {
        for (int o = 16; o; o >>= 1) acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], o);
        if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5][f] = acc[f];
    }
    __syncthreads();
    if (threadIdx.x < F) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; w++) s += warp_sum[w][threadIdx.x];
        part[((long long)n * gridDim.x + blockIdx.x) * F + threadIdx.x] = s;
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
    block_partial(acc, n, part);
}

// flow_error_kernel's walk over the pixels, with each pixel's mask bytes and boundary distance loaded beside its flows.  A NULL
// mask is never read.
__global__ void __launch_bounds__(kThreads) flow_region_kernel(T4 pred, T4 gt, const unsigned char* __restrict__ occ,
                                                               const unsigned char* __restrict__ obj, long long mstride,
                                                               const int* __restrict__ dist2,
                                                               double* __restrict__ part /* [N][bpp][kRegionFields] */) {
    const int n = blockIdx.y;
    const int hw = pred.h * pred.w;
    const bool has_occ = occ != nullptr, has_obj = obj != nullptr;
    const unsigned char* occ_n = has_occ ? occ + n * mstride : nullptr;
    const unsigned char* obj_n = has_obj ? obj + n * mstride : nullptr;
    const int* d2_n = has_occ ? dist2 + (long long)n * hw : nullptr;
    double acc[kRegionFields];
#pragma unroll
    for (int f = 0; f < kRegionFields; f++) acc[f] = 0.0;
    for (int i0 = blockIdx.x * kThreads * kUnroll + threadIdx.x; i0 < hw; i0 += gridDim.x * kThreads * kUnroll) {
        float v[kUnroll][4];
        bool oc[kUnroll], fg[kUnroll];
        int d2[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const int i = i0 + u * kThreads;
            oc[u] = fg[u] = false;
            d2[u] = kNone;
            if (i < hw) {
                const int y = i / pred.w, x = i - y * pred.w;
                v[u][0] = __ldg(gt.p + gt.off(n, 0, y, x)); v[u][1] = __ldg(gt.p + gt.off(n, 1, y, x));
                v[u][2] = __ldg(pred.p + pred.off(n, 0, y, x)); v[u][3] = __ldg(pred.p + pred.off(n, 1, y, x));
                if (has_occ) {
                    oc[u] = __ldg(occ_n + i) != 0;
                    d2[u] = __ldg(d2_n + i);
                }
                if (has_obj) fg[u] = __ldg(obj_n + i) != 0;
            } else {
                v[u][0] = v[u][1] = v[u][2] = v[u][3] = __int_as_float(0x7fffffff);
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; u++)
            score_region(v[u][0], v[u][1], v[u][2], v[u][3], has_occ, oc[u], d2[u], has_obj, fg[u], acc);
    }
    block_partial(acc, n, part);
}

// One thread per (pair, field): the pair's block partials added in block order.
template <int F>
__global__ void final_kernel(const double* __restrict__ part, int N, int bpp, double* __restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * F) return;
    const int n = t / F, f = t - n * F;
    double s = 0.0;
    for (int b = 0; b < bpp; b++) s += part[((long long)n * bpp + b) * F + f];
    out[t] = s;
}

// Blocks per pair of a scoring kernel (per_sm: its resident blocks per SM, found on the first call): enough to cover the pair's
// pixels, at most one wave of resident blocks over all N pairs (a second, partial wave would leave most of the device idle
// while it runs).
int blocks_per_pair(const void* kernel, int& per_sm, int N, int H, int W) {
    if (!per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1)) {
        cudaGetLastError();
        per_sm = 1;
    }
    const long long need = ((long long)H * W + kThreads * kUnroll - 1) / (kThreads * kUnroll);
    const long long cap = max(1LL, (long long)num_sms() * per_sm / N);
    return (int)max(1LL, min(need, cap));
}

int eval_blocks(int N, int H, int W) {
    static int per_sm = 0;
    return blocks_per_pair((const void*)flow_error_kernel, per_sm, N, H, W);
}

int region_blocks(int N, int H, int W) {
    static int per_sm = 0;
    return blocks_per_pair((const void*)flow_region_kernel, per_sm, N, H, W);
}

// Pass 1 of the distance: one thread per column x of pair blockIdx.y.  A pixel is on the boundary when a 4-neighbour inside the
// image has the other label.  Each sweep goes kChunk rows at a time, every load of a chunk issued before its first use: the
// sweeps are serial in y, and a load per row waited for one by one would leave them bound by memory latency.
__global__ void __launch_bounds__(kColThreads) boundary_column_kernel(const unsigned char* __restrict__ masks, long long stride,
                                                                      int H, int W, int* __restrict__ dist2) {
    const int x = blockIdx.x * kColThreads + threadIdx.x;
    if (x >= W) return;
    const unsigned char* m = masks + blockIdx.y * stride;
    int* d = dist2 + (long long)blockIdx.y * H * W;
    auto label = [&](int y, int xx) { return __ldg(m + (long long)y * W + xx) != 0; };
    int run = kNone;                                                    // rows since the last boundary pixel at or above
    for (int y0 = 0; y0 < H; y0 += kChunk) {
        bool left[kChunk], right[kChunk], col[kChunk + 2];              // col[j]: row y0 - 1 + j
#pragma unroll
        for (int j = 0; j < kChunk; j++) {
            const int y = y0 + j;
            left[j] = y < H && x > 0 && label(y, x - 1);
            right[j] = y < H && x + 1 < W && label(y, x + 1);
        }
#pragma unroll
        for (int j = 0; j < kChunk + 2; j++) {
            const int y = y0 - 1 + j;
            col[j] = y >= 0 && y < H && label(y, x);
        }
#pragma unroll
        for (int j = 0; j < kChunk; j++) {
            const int y = y0 + j;
            if (y >= H) break;
            const bool here = col[j + 1];
            const bool edge = (x > 0 && left[j] != here) || (x + 1 < W && right[j] != here) || (y > 0 && col[j] != here) ||
                              (y + 1 < H && col[j + 2] != here);
            run = edge ? 0 : (run == kNone ? kNone : run + 1);
            d[(long long)y * W + x] = run;
        }
    }
    run = kNone;                                                        // rows since the last boundary pixel at or below
    for (int y1 = H - 1; y1 >= 0; y1 -= kChunk) {
        int v[kChunk];
#pragma unroll
        for (int j = 0; j < kChunk; j++) v[j] = y1 - j >= 0 ? d[(long long)(y1 - j) * W + x] : 0;
#pragma unroll
        for (int j = 0; j < kChunk; j++) {
            const int y = y1 - j;
            if (y < 0) break;
            run = v[j] == 0 ? 0 : (run == kNone ? kNone : run + 1);
            const int g = min(v[j], run);
            d[(long long)y * W + x] = g == kNone ? kNone : g * g;
        }
    }
}

// Pass 2: row blockIdx.x of pair blockIdx.y, in place.  Shared memory: g (the row's vertical distances squared), s and t (the
// envelope's parabola columns and the first x of each one's segment), 3 W ints.  Columns without a boundary pixel (kNone) are
// no parabola; a row without any means a pair without a boundary, and every pixel of it gets kNone.
__global__ void __launch_bounds__(kRowThreads) boundary_row_kernel(int H, int W, int* __restrict__ dist2) {
    extern __shared__ int sm[];
    int* g = sm;
    int* s = sm + W;
    int* t = sm + 2 * W;
    __shared__ int top;
    int* row = dist2 + ((long long)blockIdx.y * H + blockIdx.x) * W;
    for (int x = threadIdx.x; x < W; x += kRowThreads) g[x] = row[x];
    __syncthreads();
    if (threadIdx.x == 0) {
        auto f = [&](int x, int i) { return (x - i) * (x - i) + g[i]; };
        int q = -1;
        for (int u = 0; u < W; u++) {
            if (g[u] == kNone) continue;
            while (q >= 0 && f(t[q], s[q]) > f(t[q], u)) q--;
            if (q < 0) {
                q = 0; s[0] = u; t[0] = 0;
            } else {
                // after the pops s[q] is no worse than u at t[q] >= 0, so the numerator is >= 0 and / is floor division
                const int i = s[q];
                const int w = 1 + (u * u - i * i + g[u] - g[i]) / (2 * (u - i));
                if (w < W) {
                    q++; s[q] = u; t[q] = w;
                }
            }
        }
        top = q;
    }
    __syncthreads();
    const int q = top;
    for (int x = threadIdx.x; x < W; x += kRowThreads) {
        if (q < 0) {
            row[x] = kNone;
            continue;
        }
        int lo = 0, hi = q;                                             // the last segment j with t[j] <= x
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (t[mid] <= x) lo = mid;
            else hi = mid - 1;
        }
        const int i = s[lo];
        row[x] = (x - i) * (x - i) + g[i];
    }
}

// Confusion counts of two 8-bit masks: grid (blocks per pair, N).  Each thread counts its pixels' TP, FP and FN, each warp sums
// them with a shuffle reduction and its lane 0 adds them to the pair's 64-bit counters (out, zeroed first) with atomicAdd:
// integer sums, so the counts do not depend on the order.  confusion_final_kernel derives TN and stores the four as doubles
// in place.
__global__ void __launch_bounds__(kThreads) mask_confusion_kernel(const unsigned char* __restrict__ pred,
                                                                  const unsigned char* __restrict__ gt, long long stride, int hw,
                                                                  unsigned long long* __restrict__ out) {
    const int n = blockIdx.y;
    const unsigned char* p = pred + n * stride;
    const unsigned char* g = gt + n * stride;
    unsigned tp = 0, fp = 0, fn = 0;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < hw; i += gridDim.x * kThreads) {
        const bool a = __ldg(p + i) != 0, b = __ldg(g + i) != 0;
        tp += a && b;
        fp += a && !b;
        fn += !a && b;
    }
    tp = __reduce_add_sync(0xffffffffu, tp);
    fp = __reduce_add_sync(0xffffffffu, fp);
    fn = __reduce_add_sync(0xffffffffu, fn);
    if ((threadIdx.x & 31) == 0 && (tp | fp | fn)) {
        unsigned long long* o = out + (long long)n * 4;
        atomicAdd(o + 0, (unsigned long long)tp);
        atomicAdd(o + 1, (unsigned long long)fp);
        atomicAdd(o + 2, (unsigned long long)fn);
    }
}

__global__ void confusion_final_kernel(int N, long long hw, unsigned long long* __restrict__ counts) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    unsigned long long* c = counts + (long long)n * 4;
    const unsigned long long tp = c[0], fp = c[1], fn = c[2];
    double* d = reinterpret_cast<double*>(c);
    d[0] = (double)tp;
    d[1] = (double)fp;
    d[2] = (double)fn;
    d[3] = (double)(hw - (long long)(tp + fp + fn));
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
    final_kernel<kFields><<<(total + 127) / 128, 128, 0, st>>>((const double*)workspace, p.n, bpp, out_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_occlusion_boundary_dist2(const void* masks_dev, size_t pair_stride, int N, int H, int W, int32_t* dist2_dev,
                                 void* stream) {
    FN2_CHECK_ARG(masks_dev && dist2_dev && N > 0 && H > 0 && W > 0, "occlusion_boundary_dist2: bad argument");
    FN2_CHECK_ARG(H <= kMaxSide && W <= kMaxSide, "occlusion_boundary_dist2: %dx%d masks, at most %d on a side", W, H, kMaxSide);
    FN2_CHECK_ARG(N <= 65535, "occlusion_boundary_dist2: %d pairs, at most 65535", N);
    FN2_CHECK_ARG(pair_stride >= (size_t)H * W, "occlusion_boundary_dist2: pair stride %zu is below H * W = %lld", pair_stride,
                  (long long)H * W);
    const int smem = 3 * W * (int)sizeof(int);                          // up to 192 KiB at W = 16384
    if (smem > 48 * 1024) FN2_CUDA(cudaFuncSetAttribute(boundary_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaStream_t st = (cudaStream_t)stream;
    boundary_column_kernel<<<dim3((W + kColThreads - 1) / kColThreads, N), kColThreads, 0, st>>>(
        (const unsigned char*)masks_dev, (long long)pair_stride, H, W, dist2_dev);
    FN2_LAUNCH_CHECK();
    boundary_row_kernel<<<dim3(H, N), kRowThreads, smem, st>>>(H, W, dist2_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_flow_error_regions_workspace_bytes(int N, int H, int W, size_t* bytes) {
    FN2_CHECK_ARG(bytes && N > 0 && H > 0 && W > 0, "flow_error_regions_workspace_bytes: bad argument");
    *bytes = (size_t)N * region_blocks(N, H, W) * kRegionFields * sizeof(double);
    return FN2_OK;
}

int fn2_flow_error_regions(const fn2_tensor* pred, const fn2_tensor* gt, const void* occ_dev, const void* obj_dev,
                           size_t mask_pair_stride, const int32_t* dist2_dev, double* out_dev, void* workspace,
                           size_t workspace_bytes, void* stream) {
    FN2_CHECK_ARG(valid(pred) && valid(gt) && out_dev, "flow_error_regions: null argument");
    const T4 p = view(pred), g = view(gt);
    FN2_CHECK_ARG(same_dims(p, g), "flow_error_regions: pred is %dx%dx%dx%d but gt is %dx%dx%dx%d", p.n, p.c, p.h, p.w, g.n, g.c,
                  g.h, g.w);
    FN2_CHECK_ARG(p.c == 2, "flow_error_regions: flows need 2 channels, got %d", p.c);
    FN2_CHECK_ARG(p.n <= 65535 && (long long)p.h * p.w <= (1LL << 30), "flow_error_regions: %d pairs of %dx%d is too large", p.n,
                  p.w, p.h);
    FN2_CHECK_ARG(!occ_dev == !dist2_dev, "flow_error_regions: dist2 is required with an occlusion mask and only with one");
    FN2_CHECK_ARG(!(occ_dev || obj_dev) || mask_pair_stride >= (size_t)p.h * p.w,
                  "flow_error_regions: mask pair stride %zu is below H * W = %lld", mask_pair_stride, (long long)p.h * p.w);
    const int bpp = region_blocks(p.n, p.h, p.w);
    const size_t need = (size_t)p.n * bpp * kRegionFields * sizeof(double);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 7)) {
        set_error("flow_error_regions: workspace too small or not 8-byte aligned (%zu bytes, %zu needed)", workspace_bytes, need);
        return FN2_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    flow_region_kernel<<<dim3(bpp, p.n), kThreads, 0, st>>>(p, g, (const unsigned char*)occ_dev, (const unsigned char*)obj_dev,
                                                           (long long)mask_pair_stride, dist2_dev, (double*)workspace);
    FN2_LAUNCH_CHECK();
    const int total = p.n * kRegionFields;
    final_kernel<kRegionFields><<<(total + 127) / 128, 128, 0, st>>>((const double*)workspace, p.n, bpp, out_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_mask_confusion(const void* pred_dev, const void* gt_dev, size_t pair_stride, int N, int H, int W, double* out_dev,
                       void* stream) {
    FN2_CHECK_ARG(pred_dev && gt_dev && out_dev && N > 0 && H > 0 && W > 0, "mask_confusion: bad argument");
    FN2_CHECK_ARG(N <= 65535 && (long long)H * W <= (1LL << 30), "mask_confusion: %d pairs of %dx%d is too large", N, W, H);
    FN2_CHECK_ARG(pair_stride >= (size_t)H * W, "mask_confusion: pair stride %zu is below H * W = %lld", pair_stride,
                  (long long)H * W);
    FN2_CHECK_ARG(!((uintptr_t)out_dev & 7), "mask_confusion: out must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    FN2_CUDA(cudaMemsetAsync(out_dev, 0, (size_t)N * 4 * sizeof(double), st));
    const int hw = H * W;
    const int bpp = (int)max(1LL, min(((long long)hw + kThreads - 1) / kThreads, (long long)ew_grid((long long)hw * N, kThreads) / N));
    unsigned long long* counts = reinterpret_cast<unsigned long long*>(out_dev);
    mask_confusion_kernel<<<dim3(bpp, N), kThreads, 0, st>>>((const unsigned char*)pred_dev, (const unsigned char*)gt_dev,
                                                             (long long)pair_stride, hw, counts);
    FN2_LAUNCH_CHECK();
    confusion_final_kernel<<<(N + 127) / 128, 128, 0, st>>>(N, (long long)hw, counts);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // extern "C"
