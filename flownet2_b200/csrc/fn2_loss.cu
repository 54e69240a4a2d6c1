// Training-side neighbours of the FlowNet2-C training step (SURVEY.md 8 row "next" 2): L1Loss, Downsample, FlowAugmentation.
//
// L1Loss (l1loss_layer.cpp:11-90, l1loss_layer.cu:67-192).  The reference chains an Eltwise difference, a NaN mask, optional
// Power(2) -> 1x1 sum convolution -> Power(0.5, shift = epsilon) ("l2_per_location", the end-point error), a plateau mask and two
// cuBLAS dot products through six intermediate blobs.  Here ONE pass over the two bottoms computes the masked loss sum and the
// not-NaN count per block, a second tiny kernel reduces the block partials in a fixed order (deterministic; cublasSdot's order is
// not) and writes loss and normaliser; the backward recomputes difference, masks and signs from the bottoms instead of reading
// stored intermediates: 2 reads forward, 2 reads + 2 writes backward, nothing else touches HBM.  Both passes call the same
// device functions for the difference and the per-location sum with its plateau mask (l1_diff, l1_keep, l2_location), so they
// see the same masks.
// state (device, 4 floats): [0] loss, [1] normalize_coeff, [2] masked sum, [3] not-NaN count.
//
// LpqLoss (lpq_loss_layer.cpp:19-82, lpq_loss_layer.cu:96-245; include/fn2_lpq.h).  The reference chains an Eltwise
// difference, four element-wise kernels (NaN mask, KillMasked, ComputeSign, abs by multiplying with the sign), Power(p), a 1x1
// sum convolution, Power(q), a cuBLAS dot and a host read; the backward runs the chain in reverse.  Here it has L1Loss's shape:
// one pass writes a (loss, not-NaN count) partial per block, l1loss_final_kernel reduces them in a fixed order, and the
// backward recomputes difference, mask, sign, the location's channel sum and both power derivatives from the bottoms.  p and
// q are read from the state (state[4], state[5]), which the layer writes when its schedule step changes.
//
// Downsample (downsample_layer.cu:15-80): weighted box average around the rounded source position, NaN aware; the narrow and
// the wide kernel share the centre, the tap and the final value (ds_centre, ds_tap, ds_value).
// This file is compiled with FMA contraction (unlike fn2_ops.cu): moving code between the two changes its rounding.
// FlowAugmentation (flow_augmentation_layer.cu:24-66): flow field of the augmented pair from the two spatial transforms.
#include "fn2_common.cuh"
#include "../../include/fn2_lpq.h"

namespace fn2 {

namespace {

struct L1P {
    int l2_per_location, two, plateau_on;
    float wsum, eps, plateau;
};

// The per-element difference of the Eltwise layer: bottom0 - bottom1, or bottom0 alone
__device__ __forceinline__ float l1_diff(const T4& a, const T4& b, const L1P& p, int n, int c, int y, int x) {
    float d = a.p[a.off(n, c, y, x)];
    if (p.two) d -= b.p[b.off(n, c, y, x)];
    return d;
}
// L1 route: d counts (FindNotNaNs, then MaskPlateauValues)
__device__ __forceinline__ bool l1_keep(const L1P& p, float d) { return d == d && !(p.plateau_on && fabsf(d) < p.plateau); }
// L2 route: the per-location sum s = sum_c wsum * d^2 over the not-NaN d (KillMasked, Power(2), then the 1x1 sum convolution),
// zeroed by the plateau mask (MaskPlateauValuesInitial + KillMasked), which kill reports.  cnt counts the not-NaN d.
__device__ __forceinline__ float l2_location(const T4& a, const T4& b, const L1P& p, int n, int y, int x, float& cnt, bool& kill) {
    float s = 0.f;
    for (int c = 0; c < a.c; c++) {
        const float d = l1_diff(a, b, p, n, c, y, x);
        const bool ok = d == d;
        cnt += ok ? 1.f : 0.f;
        const float dz = ok ? d : 0.f;
        s += p.wsum * (dz * dz);
    }
    kill = p.plateau_on && fabsf(s) < p.plateau * p.plateau;
    return kill ? 0.f : s;
}

// The block's (loss, count) partial into part[2 * blockIdx.x], part[2 * blockIdx.x + 1]: warp butterflies, then the first warp
// over the warps' sums (L1Loss and LpqLoss forwards)
__device__ __forceinline__ void block_partial(float loss, float cnt, float* __restrict__ part) {
    __shared__ float sl[32], sc[32];
    for (int o = 16; o; o >>= 1) { loss += __shfl_xor_sync(0xffffffffu, loss, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
    if ((threadIdx.x & 31) == 0) { sl[threadIdx.x >> 5] = loss; sc[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int nw = blockDim.x >> 5;
        loss = threadIdx.x < nw ? sl[threadIdx.x] : 0.f;
        cnt = threadIdx.x < nw ? sc[threadIdx.x] : 0.f;
        for (int o = 16; o; o >>= 1) { loss += __shfl_xor_sync(0xffffffffu, loss, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
        if (threadIdx.x == 0) { part[2 * blockIdx.x] = loss; part[2 * blockIdx.x + 1] = cnt; }
    }
}

template <bool L2>
__global__ void l1loss_fwd_kernel(T4 a, T4 b, L1P p, float* __restrict__ part /* [grid][2] */) {
    float loss = 0.f, cnt = 0.f;
    for_each_pixel(a.n, a.h, a.w, [&](int n, int y, int x) {
        if constexpr (L2) {
            bool kill;
            const float s = l2_location(a, b, p, n, y, x, cnt, kill);
            loss += sqrtf(s + p.eps);                                   // Power(0.5, shift = epsilon)
        } else {
            for (int c = 0; c < a.c; c++) {
                const float d = l1_diff(a, b, p, n, c, y, x);
                cnt += d == d ? 1.f : 0.f;
                loss += l1_keep(p, d) ? fabsf(d) : 0.f;                 // d * sign(d)
            }
        }
    });
    block_partial(loss, cnt, part);
}

// Also LpqLoss's final kernel: its normaliser is L1Loss's (lpq_loss_layer.cu:156-161), and it leaves p and q (state[4..5]) alone.
__global__ void l1loss_final_kernel(const float* __restrict__ part, int blocks, int num, int channels, int by_entries,
                                    float* __restrict__ state, float* __restrict__ loss_out) {
    if (threadIdx.x || blockIdx.x) return;
    double loss = 0.0, cnt = 0.0;
    for (int i = 0; i < blocks; i++) { loss += (double)part[2 * i]; cnt += (double)part[2 * i + 1]; }
    const float norm = by_entries ? (float)cnt / (float)channels : (float)num;      // l1loss_layer.cu:83-88
    const float l = (float)loss / norm;
    state[0] = l; state[1] = norm; state[2] = (float)loss; state[3] = (float)cnt;
    if (loss_out) *loss_out = l;
}

template <bool L2>
__global__ void l1loss_bwd_kernel(T4 a, T4 b, L1P p, const float* __restrict__ state, const float* __restrict__ top_diff,
                                  T4 da, T4 db, int prop_a, int prop_b, int acc_a, int acc_b) {
    const float alpha = top_diff[0] / state[1];                         // l1loss_layer.cu:152
    for_each_pixel(a.n, a.h, a.w, [&](int n, int y, int x) {
        float gs = 0.f;
        if (L2) {
            float cnt = 0.f;
            bool kill;
            const float s = l2_location(a, b, p, n, y, x, cnt, kill);
            const float root = sqrtf(s + p.eps);
            // PowerLayer::Backward (power_layer.cu:49-84): shift != 0: top_data / (x + shift) * power; shift == 0: top_data / x * power
            gs = (root / (s + p.eps)) * 0.5f * alpha;
            if (kill) gs = 0.f;                                         // KillMasked(plateau_l2_) on the sum's diff
        }
        for (int c = 0; c < a.c; c++) {
            const float d = l1_diff(a, b, p, n, c, y, x);
            float g;
            if (L2) {
                const bool ok = d == d;
                const float dz = ok ? d : 0.f;
                g = (2.f * dz) * (p.wsum * gs);                         // Power(2) backward of the sum convolution's backward
                if (!ok) g = 0.f;                                       // KillMasked(mask_)
            } else {
                const bool keep = l1_keep(p, d);
                const float dz = keep ? d : 0.f;
                g = keep ? alpha * (dz > 0.f ? 1.f : -1.f) : 0.f;       // ComputeSign: 0 -> -1
            }
            if (prop_a) { float* o = da.p + da.off(n, c, y, x); *o = acc_a ? *o + g : g; }
            if (prop_b && p.two) { float* o = db.p + db.off(n, c, y, x); *o = acc_b ? *o - g : -g; }
        }
    });
}

// ---- LpqLoss ---------------------------------------------------------------------------------------------------------------
struct LpqP {
    int two;
    float w, pe, qe;    // channel weight of the sum convolution, the p and q Power layers' shifts
};

// PowerLayer::Forward_gpu (power_layer.cu:8-30) with scale 1: power 0 gives 1 (diff_scale_ == 0); the shift is added when it is
// not 0; powf (caffe_gpu_powx's pow(float, float)) runs only when power != 1.
__device__ __forceinline__ float lpq_pow(float x, float shift, float power) {
    if (power == 0.f) return 1.f;
    const float t = shift != 0.f ? __fadd_rn(x, shift) : x;
    return power != 1.f ? powf(t, power) : t;
}
// PowerLayer::Backward_gpu (power_layer.cu:32-84) before its product with the top diff, y = lpq_pow(x): power 0: 0; power 1:
// 1; power 2: 2x + 2 shift; shift 0: power * y / x; otherwise power * y / (x + shift).  One deviation: with shift 0 the
// reference divides 0 / 0 = NaN at x == 0 (an exactly-zero difference for p, a zero channel sum for q) and the NaN reaches the
// weights; here the derivative is 0 there (the subgradient; for power > 1 the true derivative).
__device__ __forceinline__ float lpq_dpow(float x, float y, float shift, float power) {
    if (power == 0.f) return 0.f;
    if (power == 1.f) return 1.f;
    if (power == 2.f) { const float g = __fmul_rn(2.f, x); return shift != 0.f ? __fadd_rn(g, __fmul_rn(2.f, shift)) : g; }
    if (shift == 0.f) return x == 0.f ? 0.f : __fmul_rn(__fdiv_rn(y, x), power);
    return __fmul_rn(__fdiv_rn(y, __fadd_rn(x, shift)), power);
}
// |d| as the reference forms it: KillMasked zeroes a NaN d BEFORE the powers (lpq_loss_layer.cu:163-169), so a NaN entry
// still adds w * P(0) = w * p_epsilon^p, and a location whose channels are all NaN still adds Q(...) >= q_epsilon^q; then
// ComputeSign (0 -> -1) and the product with the sign (:172-185), i.e. |d|.
__device__ __forceinline__ float lpq_abs(float d) { return d == d ? fabsf(d) : 0.f; }
// The location's channel sum s = sum_c w * P(|d_c|) (the 1x1 convolution with constant weight w, lpq_loss_layer.cpp:118-135);
// cnt counts the not-NaN d (FindNotNaNs).
__device__ __forceinline__ float lpq_location(const T4& a, const T4& b, const LpqP& lp, float p, int n, int y, int x, float& cnt) {
    float s = 0.f;
    for (int c = 0; c < a.c; c++) {
        const float d = a.p[a.off(n, c, y, x)] - (lp.two ? b.p[b.off(n, c, y, x)] : 0.f);
        cnt += d == d ? 1.f : 0.f;
        s += lp.w * lpq_pow(lpq_abs(d), lp.pe, p);
    }
    return s;
}

__global__ void lpqloss_fwd_kernel(T4 a, T4 b, LpqP lp, const float* __restrict__ state, float* __restrict__ part /* [grid][2] */) {
    const float p = state[4], q = state[5];
    float loss = 0.f, cnt = 0.f;
    for_each_pixel(a.n, a.h, a.w, [&](int n, int y, int x) {
        loss += lpq_pow(lpq_location(a, b, lp, p, n, y, x, cnt), lp.qe, q);
    });
    block_partial(loss, cnt, part);
}

__global__ void lpqloss_bwd_kernel(T4 a, T4 b, LpqP lp, const float* __restrict__ state, const float* __restrict__ top_diff,
                                   T4 da, T4 db, int prop_a, int prop_b, int acc_a, int acc_b) {
    const float alpha = top_diff[0] / state[1];                         // lpq_loss_layer.cu:214
    const float p = state[4], q = state[5];
    for_each_pixel(a.n, a.h, a.w, [&](int n, int y, int x) {
        float cnt = 0.f;
        const float s = lpq_location(a, b, lp, p, n, y, x, cnt);
        // Power(q) backward, then the sum convolution's data gradient: w * alpha * Q'(s) for every channel
        const float gs = __fmul_rn(lp.w, __fmul_rn(alpha, lpq_dpow(s, lpq_pow(s, lp.qe, q), lp.qe, q)));
        for (int c = 0; c < a.c; c++) {
            const float d = a.p[a.off(n, c, y, x)] - (lp.two ? b.p[b.off(n, c, y, x)] : 0.f);
            const bool ok = d == d;
            const float ad = lpq_abs(d);
            float g = __fmul_rn(gs, lpq_dpow(ad, lpq_pow(ad, lp.pe, p), lp.pe, p));   // Power(p) backward
            g = __fmul_rn(g, ok && d > 0.f ? 1.f : -1.f);               // times the sign of the zeroed d (:225-231)
            if (!ok) g = 0.f;                                           // KillMasked (:233-238)
            if (prop_a) { float* o = da.p + da.off(n, c, y, x); *o = acc_a ? *o + g : g; }
            if (prop_b && lp.two) { float* o = db.p + db.off(n, c, y, x); *o = acc_b ? *o - g : -g; }   // Eltwise coeff -1
        }
    });
}

// ---- Downsample ------------------------------------------------------------------------------------------------------------
// Output (dx, dy) averages the source window around the rounded centre (bx, by) with tent weights of radius (wscale, hscale).
// The narrow kernel takes one output per thread, the wide one a block per output (ds_wide).
struct DsCentre { float bx, by; int ix, iy; };
__device__ __forceinline__ DsCentre ds_centre(const T4& src, const T4& dst, int dx, int dy) {
    DsCentre r;
    r.bx = ((float)dx / (float)(dst.w - 1)) * (float)(src.w - 1);
    r.by = ((float)dy / (float)(dst.h - 1)) * (float)(src.h - 1);
    r.ix = (int)roundf(r.bx); r.iy = (int)roundf(r.by);
    return r;
}
// Adds source pixel (sx, sy) of channel (n, c): a NaN sample adds its weight to wnan instead of val and wsum.
__device__ __forceinline__ void ds_tap(const T4& src, int n, int c, int sx, int sy, const DsCentre& o, float wscale, float hscale,
                                       float& val, float& wsum, float& wnan) {
    if (sx < 0 || sy < 0 || sx >= src.w || sy >= src.h) return;
    float sample = src.p[src.off(n, c, sy, sx)];
    float wgt = fmaxf(0.f, 1.f - fabsf((float)sx - o.bx) / wscale) * fmaxf(0.f, 1.f - fabsf((float)sy - o.by) / hscale);
    if (sample != sample) { wnan += wgt; sample = 0.f; wgt = 0.f; }
    val += sample * wgt;
    wsum += wgt;
}
// NaN when NaN samples carry more than half of the weight, else the weighted mean
__device__ __forceinline__ float ds_value(float val, float wsum, float wnan) {
    return (wnan / wsum > 0.5f) ? __int_as_float(0x7fffffff) : val / wsum;
}

__global__ void downsample_kernel(T4 src, T4 dst, float wscale, float hscale, int wrad, int hrad) {
    for_each_element(dst, [&](Idx4 e, long long) {
        const DsCentre o = ds_centre(src, dst, e.x, e.y);
        float val = 0.f, wsum = 0.f, wnan = 0.f;
        for (int yo = -hrad; yo <= hrad; yo++)
            for (int xo = -wrad; xo <= wrad; xo++) ds_tap(src, e.n, e.c, o.ix + xo, o.iy + yo, o, wscale, hscale, val, wsum, wnan);
        dst.p[dst.off(e.n, e.c, e.y, e.x)] = ds_value(val, wsum, wnan);
    });
}

// Wide windows (the 1/64 level averages 161 x 151 source pixels per output): one warp-group per output element, the window
// spread over the threads, fixed-order tree reduction.
__global__ void downsample_wide_kernel(T4 src, T4 dst, float wscale, float hscale, int wrad, int hrad) {
    const Idx4 e = nchw_index(dst, blockIdx.x);
    const DsCentre o = ds_centre(src, dst, e.x, e.y);
    const int ww = 2 * wrad + 1, wh = 2 * hrad + 1;
    float val = 0.f, wsum = 0.f, wnan = 0.f;
    for (int t = threadIdx.x; t < ww * wh; t += blockDim.x)
        ds_tap(src, e.n, e.c, o.ix - wrad + t % ww, o.iy - hrad + t / ww, o, wscale, hscale, val, wsum, wnan);
    __shared__ float s[3][8];
    for (int k = 16; k; k >>= 1) {
        val += __shfl_xor_sync(0xffffffffu, val, k); wsum += __shfl_xor_sync(0xffffffffu, wsum, k); wnan += __shfl_xor_sync(0xffffffffu, wnan, k);
    }
    if ((threadIdx.x & 31) == 0) { s[0][threadIdx.x >> 5] = val; s[1][threadIdx.x >> 5] = wsum; s[2][threadIdx.x >> 5] = wnan; }
    __syncthreads();
    if (threadIdx.x == 0) {
        val = wsum = wnan = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) { val += s[0][i]; wsum += s[1][i]; wnan += s[2][i]; }
        dst.p[dst.off(e.n, e.c, e.y, e.x)] = ds_value(val, wsum, wnan);
    }
}

// The wide kernel, a block of 256 threads per output, when the window has at least one tap per thread and the outputs fit
// in one grid row (at most 2^20 blocks); one thread per output otherwise.
static bool ds_wide(int wrad, int hrad, long long outputs) { return (2 * wrad + 1) * (2 * hrad + 1) >= 256 && outputs <= (1 << 20); }

// ---- FlowAugmentation ------------------------------------------------------------------------------------------------------
// m1 / m2: 6 floats per sample in NAME order t0..t5 (x' = x*t0 + y*t2 + t4, y' = x*t1 + y*t3 + t5); m2 is already inverted.
__global__ void flow_aug_kernel(T4 src, T4 dst, const float* __restrict__ m1, const float* __restrict__ m2) {
    const long long src_count = src.count();
    for_each_pixel(dst.n, dst.h, dst.w, [&](int n, int yi, int xi) {
        const float x = (float)xi, y = (float)yi;
        const float* a = m1 + 6 * n;
        const float* b = m2 + 6 * n;
        const float x1 = x * a[0] + y * a[2] + a[4];
        const float y1 = x * a[1] + y * a[3] + a[5];
        // nearest flow sample; the reference indexes the dense NCHW array with an UNCHECKED position (only min(idx, count)), so
        // a position outside the image reads a neighbouring row / sample or out of bounds.  Same linear index here, clamped into
        // the array (identical whenever the reference's read is in bounds).
        const int sy = (int)(y1 + 0.5f), sx = (int)(x1 + 0.5f);
        long long ou = (long long)src.w * ((long long)src.h * (2 * n + 0) + sy) + sx;
        long long ov = (long long)src.w * ((long long)src.h * (2 * n + 1) + sy) + sx;
        ou = max(0LL, min(ou, src_count - 1));
        ov = max(0LL, min(ov, src_count - 1));
        auto at = [&](long long lin) { const Idx4 e = nchw_index(src, lin); return src.p[src.off(e.n, e.c, e.y, e.x)]; };
        const float x2 = x1 + at(ou), y2 = y1 + at(ov);
        const float x3 = x2 * b[0] + y2 * b[2] + b[4];
        const float y3 = x2 * b[1] + y2 * b[3] + b[5];
        dst.p[dst.off(n, 0, yi, xi)] = x3 - x;
        dst.p[dst.off(n, 1, yi, xi)] = y3 - y;
    });
}

int loss_grid(long long P) { return (int)max(1LL, min((long long)num_sms() * 4, (P + 255) / 256)); }

L1P l1_params(const fn2_l1loss_desc* d, const T4& a, bool two) {
    L1P p;
    p.l2_per_location = d->l2_per_location; p.two = two ? 1 : 0; p.plateau_on = d->plateau > 0.f; p.plateau = d->plateau;
    p.eps = d->epsilon; p.wsum = d->l2_prescale_by_channels ? 1.f / (float)a.c : 1.f;
    return p;
}

LpqP lpq_params(const fn2_lpqloss_desc* d, const T4& a, bool two) {
    LpqP p;
    p.two = two ? 1 : 0; p.pe = d->p_epsilon; p.qe = d->q_epsilon;
    p.w = d->l2_prescale_by_channels ? 1.f / (float)a.c : 1.f;        // lpq_loss_layer.cpp:123-131
    return p;
}

}  // namespace
}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2_l1loss_workspace_bytes(int N, int H, int W, size_t* bytes) {
    FN2_CHECK_ARG(bytes && N > 0 && H > 0 && W > 0, "l1loss_workspace_bytes: bad argument");
    *bytes = (size_t)loss_grid((long long)N * H * W) * 2 * sizeof(float);
    return FN2_OK;
}

int fn2_l1loss_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_l1loss_desc* d, float* state_dev,
                       float* loss_dev, void* workspace, size_t workspace_bytes, void* stream) {
    FN2_CHECK_ARG(valid(bottom0) && d && state_dev, "l1loss_forward: null argument");
    T4 a = view(bottom0), b = a;
    if (bottom1) { FN2_CHECK_ARG(valid(bottom1), "l1loss_forward: bad second bottom"); b = view(bottom1); FN2_CHECK_ARG(same_dims(a, b), "l1loss_forward: bottoms differ in shape"); }
    const long long P = (long long)a.n * a.h * a.w;
    const int grid = loss_grid(P);
    if (!workspace || workspace_bytes < (size_t)grid * 2 * sizeof(float)) {
        set_error("l1loss_forward: workspace too small (%zu < %zu)", workspace_bytes, (size_t)grid * 2 * sizeof(float));
        return FN2_ERR_WORKSPACE;
    }
    const L1P p = l1_params(d, a, bottom1);
    cudaStream_t st = (cudaStream_t)stream;
    if (p.l2_per_location) l1loss_fwd_kernel<true><<<grid, 256, 0, st>>>(a, b, p, (float*)workspace);
    else l1loss_fwd_kernel<false><<<grid, 256, 0, st>>>(a, b, p, (float*)workspace);
    FN2_LAUNCH_CHECK();
    l1loss_final_kernel<<<1, 32, 0, st>>>((const float*)workspace, grid, a.n, a.c, d->normalize_by_num_entries, state_dev, loss_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_l1loss_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_l1loss_desc* d, const float* state_dev,
                        const float* top_diff_dev, const fn2_tensor* bottom0_diff, const fn2_tensor* bottom1_diff,
                        int accumulate0, int accumulate1, void* stream) {
    FN2_CHECK_ARG(valid(bottom0) && d && state_dev && top_diff_dev, "l1loss_backward: null argument");
    FN2_CHECK_ARG(bottom0_diff || bottom1_diff, "l1loss_backward: no gradient requested");
    T4 a = view(bottom0), b = a, da = a, db = a;
    if (bottom1) { b = view(bottom1); FN2_CHECK_ARG(same_dims(a, b), "l1loss_backward: bottoms differ in shape"); }
    if (bottom0_diff) { da = view(bottom0_diff); FN2_CHECK_ARG(same_dims(a, da), "l1loss_backward: bottom0 diff shape"); }
    if (bottom1_diff) { FN2_CHECK_ARG(bottom1, "l1loss_backward: diff for a missing bottom"); db = view(bottom1_diff); FN2_CHECK_ARG(same_dims(a, db), "l1loss_backward: bottom1 diff shape"); }
    const L1P p = l1_params(d, a, bottom1);
    const int grid = loss_grid((long long)a.n * a.h * a.w);
    cudaStream_t st = (cudaStream_t)stream;
    if (p.l2_per_location)
        l1loss_bwd_kernel<true><<<grid, 256, 0, st>>>(a, b, p, state_dev, top_diff_dev, da, db, bottom0_diff ? 1 : 0, bottom1_diff ? 1 : 0, accumulate0, accumulate1);
    else
        l1loss_bwd_kernel<false><<<grid, 256, 0, st>>>(a, b, p, state_dev, top_diff_dev, da, db, bottom0_diff ? 1 : 0, bottom1_diff ? 1 : 0, accumulate0, accumulate1);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_lpqloss_workspace_bytes(int N, int H, int W, size_t* bytes) {
    FN2_CHECK_ARG(bytes && N > 0 && H > 0 && W > 0, "lpqloss_workspace_bytes: bad argument");
    *bytes = (size_t)loss_grid((long long)N * H * W) * 2 * sizeof(float);
    return FN2_OK;
}

int fn2_lpqloss_forward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_lpqloss_desc* d, float* state_dev,
                        float* loss_dev, void* workspace, size_t workspace_bytes, void* stream) {
    FN2_CHECK_ARG(valid(bottom0) && d && state_dev, "lpqloss_forward: null argument");
    T4 a = view(bottom0), b = a;
    if (bottom1) { FN2_CHECK_ARG(valid(bottom1), "lpqloss_forward: bad second bottom"); b = view(bottom1); FN2_CHECK_ARG(same_dims(a, b), "lpqloss_forward: bottoms differ in shape"); }
    const int grid = loss_grid((long long)a.n * a.h * a.w);
    if (!workspace || workspace_bytes < (size_t)grid * 2 * sizeof(float)) {
        set_error("lpqloss_forward: workspace too small (%zu < %zu)", workspace_bytes, (size_t)grid * 2 * sizeof(float));
        return FN2_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    lpqloss_fwd_kernel<<<grid, 256, 0, st>>>(a, b, lpq_params(d, a, bottom1), state_dev, (float*)workspace);
    FN2_LAUNCH_CHECK();
    l1loss_final_kernel<<<1, 32, 0, st>>>((const float*)workspace, grid, a.n, a.c, d->normalize_by_num_entries, state_dev, loss_dev);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_lpqloss_backward(const fn2_tensor* bottom0, const fn2_tensor* bottom1, const fn2_lpqloss_desc* d, const float* state_dev,
                         const float* top_diff_dev, const fn2_tensor* bottom0_diff, const fn2_tensor* bottom1_diff,
                         int accumulate0, int accumulate1, void* stream) {
    FN2_CHECK_ARG(valid(bottom0) && d && state_dev && top_diff_dev, "lpqloss_backward: null argument");
    FN2_CHECK_ARG(bottom0_diff || bottom1_diff, "lpqloss_backward: no gradient requested");
    T4 a = view(bottom0), b = a, da = a, db = a;
    if (bottom1) { b = view(bottom1); FN2_CHECK_ARG(same_dims(a, b), "lpqloss_backward: bottoms differ in shape"); }
    if (bottom0_diff) { da = view(bottom0_diff); FN2_CHECK_ARG(same_dims(a, da), "lpqloss_backward: bottom0 diff shape"); }
    if (bottom1_diff) { FN2_CHECK_ARG(bottom1, "lpqloss_backward: diff for a missing bottom"); db = view(bottom1_diff); FN2_CHECK_ARG(same_dims(a, db), "lpqloss_backward: bottom1 diff shape"); }
    const int grid = loss_grid((long long)a.n * a.h * a.w);
    lpqloss_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, b, lpq_params(d, a, bottom1), state_dev, top_diff_dev, da, db,
                                                                bottom0_diff ? 1 : 0, bottom1_diff ? 1 : 0, accumulate0, accumulate1);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_downsample_forward(const fn2_tensor* bottom, const fn2_tensor* top, void* stream) {
    FN2_CHECK_ARG(valid(bottom) && valid(top), "downsample: null argument");
    T4 s = view(bottom), t = view(top);
    FN2_CHECK_ARG(s.n == t.n && s.c == t.c, "downsample: num / channels differ");
    if (s.h == t.h && s.w == t.w) return fn2_copy(bottom, top, stream);            // downsample_layer.cpp:55-58 (shared data)
    const float wscale = (float)(s.w - 1) / (float)(t.w - 1), hscale = (float)(s.h - 1) / (float)(t.h - 1);
    const int wrad = (int)ceilf(wscale), hrad = (int)ceilf(hscale);
    if (!ds_wide(wrad, hrad, t.count())) return ew_launch(downsample_kernel, t.count(), stream, s, t, wscale, hscale, wrad, hrad);
    downsample_wide_kernel<<<(unsigned)t.count(), 256, 0, (cudaStream_t)stream>>>(s, t, wscale, hscale, wrad, hrad);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int fn2_flow_augmentation(const fn2_tensor* flow, const fn2_tensor* top, const float* mats1_dev, const float* mats2_inverse_dev, void* stream) {
    FN2_CHECK_ARG(valid(flow) && valid(top) && mats1_dev && mats2_inverse_dev, "flow_augmentation: null argument");
    T4 s = view(flow), t = view(top);
    FN2_CHECK_ARG(s.c == 2 && t.c == 2 && s.n == t.n, "flow_augmentation: flow blobs need 2 channels and equal num");
    return ew_launch(flow_aug_kernel, (long long)t.n * t.h * t.w, stream, s, t, mats1_dev, mats2_inverse_dev);
}

}  // extern "C"
