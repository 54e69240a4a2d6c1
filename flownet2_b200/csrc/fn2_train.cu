// Convolution and deconvolution gradients behind the C-ABI:
//   * gradients w.r.t. weights and bias (base_conv_layer.cpp:352-395 weight_gpu_gemm / backward_gpu_bias): on the tensor-core
//     engine where it takes the layer (fn2_conv_tc.cu), else an FP32 SIMT outer-product GEMM over the pixels, split over
//     pixel ranges with a fixed-order reduction (deterministic; the reference's cuBLAS order is unpinned);
//   * the descriptor and derived weights of the gradient w.r.t. the DATA, which reuses the forward engines
//     (fn2_conv_backward_data_desc: a stride-1 convolution's adjoint is a convolution with flipped, transposed weights; a
//     stride-2 convolution's adjoint is the deconvolution with the same weights and vice versa).
#include "fn2_common.cuh"

namespace fn2 {

// fn2_conv_tc.cu: weight gradient on the wgmma pipeline
int conv_tc_wgrad_takes(const fn2_conv_desc* d);
int conv_tc_wgrad_eligible(const fn2_conv_desc* d);
size_t conv_tc_wgrad_workspace_floats(const fn2_conv_desc* d, int N, int H, int W);
void conv_tc_wgrad_plan(const fn2_conv_desc* d, int N, int H, int W, int32_t* out8);
int conv_tc_wgrad(const fn2_conv_desc* d, const T4& bottom, const T4& top_diff, float* dw, float* db, int accumulate, float* ws,
                  size_t ws_floats, cudaStream_t st);

namespace {

// ---- bias gradient: db[c] = sum over (n, y, x) of dy, two stages, fixed order ---------------------------------------------
__global__ void bias_grad_partial_kernel(T4 dy, float* __restrict__ part, int chunks) {
    // block b sums pixels [b*per, (b+1)*per) for every channel.  Channel-fast maps: thread = channel (coalesced), the 256 / C
    // thread groups take interleaved pixels and are combined through shared memory in a fixed order.
    const long long P = (long long)dy.n * dy.h * dy.w;
    const long long per = (P + chunks - 1) / chunks;
    const long long p0 = blockIdx.x * per, p1 = min(P, p0 + per);
    __shared__ float sm[256];
    int lanes = 1;
    while (lanes < dy.c && lanes < 256) lanes *= 2;                 // channels per pass (power of two <= 256)
    const int groups = 256 / lanes, grp = threadIdx.x / lanes, cl = threadIdx.x % lanes;
    for (int c0 = 0; c0 < dy.c; c0 += lanes) {
        const int c = c0 + cl;
        float acc = 0.f;
        if (c < dy.c)
            for (long long p = p0 + grp; p < p1; p += groups) {
                const int w = (int)(p % dy.w);
                const long long r = p / dy.w;
                const int h = (int)(r % dy.h), n = (int)(r / dy.h);
                acc += dy.p[dy.off(n, c, h, w)];
            }
        sm[threadIdx.x] = acc;
        __syncthreads();
        if (grp == 0 && c < dy.c) {
            float t = 0.f;
            for (int g = 0; g < groups; g++) t += sm[g * lanes + cl];
            part[(long long)blockIdx.x * dy.c + c] = t;
        }
        __syncthreads();
    }
}
__global__ void bias_grad_final_kernel(const float* __restrict__ part, float* __restrict__ db, int C, int chunks, int accumulate) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float acc = 0.f;
    for (int k = 0; k < chunks; k++) acc += part[(long long)k * C + c];
    db[c] = accumulate ? db[c] + acc : acc;
}

// ---- weight gradient ---------------------------------------------------------------------------------------------------
// dW[a][b][r][s] = sum over (n, u, v) of S[n, u, v, a] * B[n, u*st + r - p, v*st + s - p, b]
//   convolution   : S = top diff (a = co), B = bottom data (b = ci), Caffe layout [co][ci][kh][kw]  = [a][b][r][s]
//   deconvolution : S = bottom data (a = ci), B = top diff (b = co), Caffe layout [ci][co][kh][kw]  = [a][b][r][s]
// CTA: 64 x 64 tile of (a, b) for one tap and one range of pixels; 256 threads x (4 x 4) accumulators; the pixel loop stages
// 16 pixels of both operands in shared memory (channel-fast rows, coalesced).  Partials go to ws[split][a][b][tap].
struct WgP {
    int A, Bc, kh, kw, st, ph, pw;
    int Hs, Ws, Hb, Wb, N;
    int splits;
    long long per;                                 // pixels of S per split
};
constexpr int WG_T = 64, WG_PX = 16;
constexpr int BIAS_CHUNKS = 296;                   // two blocks per SM

// pixel ranges of the SIMT weight gradient: about 4 CTAs per SM over the (a, b, tap) tiles, at most 64, >= 256 pixels each
int simt_wgrad_splits(const fn2_conv_desc* d, int N, int Hs, int Ws) {
    const long long P = (long long)N * Hs * Ws;
    const int A = d->deconv ? d->ci : d->co, Bc = d->deconv ? d->co : d->ci;
    const int tiles = ((A + WG_T - 1) / WG_T) * ((Bc + WG_T - 1) / WG_T) * d->kh * d->kw;
    int splits = (int)max(1LL, min((long long)64, (long long)(num_sms() * 4) / max(1, tiles)));
    splits = (int)min((long long)splits, (P + 255) / 256);
    return max(splits, 1);
}

__global__ void __launch_bounds__(256) weight_grad_kernel(T4 S, T4 B, float* __restrict__ ws, WgP p) {
    __shared__ float sS[WG_PX][WG_T + 4], sB[WG_PX][WG_T + 4];
    const int ta = blockIdx.x % ((p.A + WG_T - 1) / WG_T), tb = blockIdx.x / ((p.A + WG_T - 1) / WG_T);
    const int tap = blockIdx.y, r = tap / p.kw, s = tap % p.kw;
    const int split = blockIdx.z;
    const int a0 = ta * WG_T, b0 = tb * WG_T;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;         // thread computes a in [a0 + 4*ty, +4), b in [b0 + 4*tx, +4)
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
    const long long P = (long long)p.N * p.Hs * p.Ws;
    const long long q0 = split * p.per, q1 = min(P, q0 + p.per);
    for (long long q = q0; q < q1; q += WG_PX) {
        // stage 16 pixels: 16 x 64 channels of each operand = 1024 floats each, 4 per thread
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int e = tid + 256 * k;
            const int px = e >> 6, ch = e & 63;
            const long long qq = q + px;
            float vs = 0.f, vb = 0.f;
            if (qq < q1) {
                const int v = (int)(qq % p.Ws);
                const long long t = qq / p.Ws;
                const int u = (int)(t % p.Hs), n = (int)(t / p.Hs);
                if (a0 + ch < p.A) vs = S.p[S.off(n, a0 + ch, u, v)];
                const int yb = u * p.st + r - p.ph, xb = v * p.st + s - p.pw;
                if (b0 + ch < p.Bc && yb >= 0 && yb < p.Hb && xb >= 0 && xb < p.Wb) vb = B.p[B.off(n, b0 + ch, yb, xb)];
            }
            sS[px][ch] = vs;
            sB[px][ch] = vb;
        }
        __syncthreads();
#pragma unroll
        for (int px = 0; px < WG_PX; px++) {
            const float4 av = *reinterpret_cast<const float4*>(&sS[px][4 * ty]);
            const float4 bv = *reinterpret_cast<const float4*>(&sB[px][4 * tx]);
            const float a_[4] = {av.x, av.y, av.z, av.w}, b_[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a_[i], b_[j], acc[i][j]);
        }
        __syncthreads();
    }
    const int taps = p.kh * p.kw;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int a = a0 + 4 * ty + i, b = b0 + 4 * tx + j;
            if (a < p.A && b < p.Bc) ws[(((long long)split * p.A + a) * p.Bc + b) * taps + tap] = acc[i][j];
        }
}
__global__ void weight_grad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long count, int splits, int accumulate) {
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < count; idx += (long long)gridDim.x * blockDim.x) {
        float acc = 0.f;
        for (int k = 0; k < splits; k++) acc += ws[(long long)k * count + idx];
        dw[idx] = accumulate ? dw[idx] + acc : acc;
    }
}

// derived weights of the stride-1 data gradient: Wt[ci][co][r][s] = W[co][ci][kh-1-r][kw-1-s]  (conv layout with ci' = co, co' = ci)
__global__ void flip_transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int Co, int Ci, int kh, int kw) {
    const long long total = (long long)Co * Ci * kh * kw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(idx % kw);
        long long t = idx / kw;
        const int r = (int)(t % kh); t /= kh;
        const int co = (int)(t % Co);
        const int ci = (int)(t / Co);
        wt[idx] = w[(((long long)co * Ci + ci) * kh + (kh - 1 - r)) * kw + (kw - 1 - s)];
    }
}

}  // namespace
}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2_conv_backward_params_workspace_bytes(const fn2_conv_desc* d, int N, int H, int W, size_t* bytes) {
    FN2_CHECK_ARG(d && bytes, "conv_backward_params_workspace_bytes: null argument");
    int Ho, Wo;
    int rc = fn2_conv_out_shape(d, H, W, &Ho, &Wo);
    if (rc) return rc;
    const int splits = simt_wgrad_splits(d, N, d->deconv ? H : Ho, d->deconv ? W : Wo);
    size_t wfloats = (size_t)splits * d->ci * d->co * d->kh * d->kw;
    if (conv_tc_wgrad_eligible(d)) wfloats = max(wfloats, conv_tc_wgrad_workspace_floats(d, N, H, W));
    const size_t bfloats = (size_t)BIAS_CHUNKS * d->co;
    *bytes = (wfloats + bfloats + 64) * sizeof(float);
    return FN2_OK;
}

int fn2_conv_wgrad_plan(const fn2_conv_desc* d, int N, int H, int W, int32_t* plan8) {
    FN2_CHECK_ARG(d && plan8, "conv_wgrad_plan: null argument");
    int Ho, Wo;
    int rc = fn2_conv_out_shape(d, H, W, &Ho, &Wo);
    if (rc) return rc;
    for (int i = 0; i < 8; i++) plan8[i] = 0;
    if (conv_tc_wgrad_takes(d)) {
        conv_tc_wgrad_plan(d, N, H, W, plan8);
    } else {
        plan8[0] = 1;
        plan8[6] = simt_wgrad_splits(d, N, d->deconv ? H : Ho, d->deconv ? W : Wo);
        plan8[7] = d->has_bias ? BIAS_CHUNKS : 0;
    }
    return FN2_OK;
}

// Gradients w.r.t. weights (Caffe layout, conv [co][ci][kh][kw] / deconv [ci][co][kh][kw]) and bias.
int fn2_conv_backward_params(const fn2_conv_desc* d, const fn2_tensor* bottom, const fn2_tensor* top_diff, float* weight_diff_dev,
                             float* bias_diff_dev, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
    FN2_CHECK_ARG(d && valid(bottom) && valid(top_diff) && weight_diff_dev, "conv_backward_params: null argument");
    T4 x = view(bottom), dy = view(top_diff);
    FN2_CHECK_ARG(x.c == d->ci && dy.c == d->co && x.n == dy.n, "conv_backward_params: channel / batch mismatch");
    size_t need = 0;
    int rc = fn2_conv_backward_params_workspace_bytes(d, x.n, x.h, x.w, &need);
    if (rc) return rc;
    if (!workspace || workspace_bytes < need) { set_error("conv_backward_params: workspace too small (%zu < %zu)", workspace_bytes, need); return FN2_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    WgP p;
    const T4& S = d->deconv ? x : dy;
    const T4& B = d->deconv ? dy : x;
    p.A = d->deconv ? d->ci : d->co; p.Bc = d->deconv ? d->co : d->ci;
    p.kh = d->kh; p.kw = d->kw; p.st = d->stride_h; p.ph = d->pad_h; p.pw = d->pad_w;
    FN2_CHECK_ARG(d->stride_h == d->stride_w, "conv_backward_params: anisotropic stride");
    p.Hs = S.h; p.Ws = S.w; p.Hb = B.h; p.Wb = B.w; p.N = x.n;
    const long long P = (long long)p.N * p.Hs * p.Ws;
    const int tiles = ((p.A + WG_T - 1) / WG_T) * ((p.Bc + WG_T - 1) / WG_T);
    const int splits = simt_wgrad_splits(d, p.N, p.Hs, p.Ws);
    p.splits = splits;
    p.per = ((P + splits - 1) / splits + WG_PX - 1) / WG_PX * WG_PX;
    float* ws = (float*)workspace;
    const long long count = (long long)d->ci * d->co * d->kh * d->kw;
    const size_t bias_floats = (size_t)BIAS_CHUNKS * d->co + 64;
    if (conv_tc_wgrad_eligible(d)) {
        // (the bias gradient comes out of the top diff's transposition pass)
        return conv_tc_wgrad(d, x, dy, weight_diff_dev, d->has_bias ? bias_diff_dev : nullptr, accumulate, ws,
                             workspace_bytes / sizeof(float) - bias_floats, st);
    } else {
        dim3 grid((unsigned)tiles, (unsigned)(d->kh * d->kw), (unsigned)splits);
        weight_grad_kernel<<<grid, 256, 0, st>>>(S, B, ws, p);
        FN2_LAUNCH_CHECK();
        weight_grad_reduce_kernel<<<ew_grid(count, 256), 256, 0, st>>>(ws, weight_diff_dev, count, splits, accumulate);
        FN2_LAUNCH_CHECK();
    }
    if (d->has_bias && bias_diff_dev) {
        float* part = ws + (workspace_bytes / sizeof(float) - bias_floats);
        const int chunks = BIAS_CHUNKS;
        bias_grad_partial_kernel<<<chunks, 256, 0, st>>>(dy, part, chunks);
        FN2_LAUNCH_CHECK();
        bias_grad_final_kernel<<<(d->co + 127) / 128, 128, 0, st>>>(part, bias_diff_dev, d->co, chunks, accumulate);
        FN2_LAUNCH_CHECK();
    }
    return FN2_OK;
}

// Descriptor + Caffe-layout weights of the forward operator that computes the gradient w.r.t. the bottom data
// (see the header comment).  derived_weights_dev: count(weights) floats (only written for stride-1 convolutions).
int fn2_conv_backward_data_desc(const fn2_conv_desc* d, int bottom_h, int bottom_w, fn2_conv_desc* out, int* needs_flip) {
    FN2_CHECK_ARG(d && out && needs_flip, "conv_backward_data_desc: null argument");
    *out = *d;
    out->out_pad_h = out->out_pad_w = 0;
    out->ci = d->co; out->co = d->ci;
    out->has_bias = 0; out->relu = 0; out->negative_slope = 0.f; out->input_guard_bytes = 0;
    *needs_flip = 0;
    if (!d->deconv && d->stride_h == 1 && d->stride_w == 1) {
        out->deconv = 0;
        out->pad_h = d->kh - 1 - d->pad_h; out->pad_w = d->kw - 1 - d->pad_w;
        FN2_CHECK_ARG(out->pad_h >= 0 && out->pad_w >= 0, "conv_backward_data: pad larger than kernel - 1");
        *needs_flip = 1;
    } else if (!d->deconv) {
        out->deconv = 1;                           // adjoint of a strided convolution = deconvolution with the same weights
        FN2_CHECK_ARG(bottom_h + 2 * d->pad_h >= d->kh && bottom_w + 2 * d->pad_w >= d->kw, "conv_backward_data_desc: bottom smaller than the kernel");
        out->out_pad_h = (bottom_h + 2 * d->pad_h - d->kh) % d->stride_h;
        out->out_pad_w = (bottom_w + 2 * d->pad_w - d->kw) % d->stride_w;
    } else {
        out->deconv = 0;                           // adjoint of a deconvolution = convolution with the same weights
    }
    return FN2_OK;
}

int fn2_conv_flip_transpose_weights(const fn2_conv_desc* d, const float* caffe_weights_dev, float* derived_dev, void* stream) {
    FN2_CHECK_ARG(d && caffe_weights_dev && derived_dev, "conv_flip_transpose_weights: null argument");
    const long long total = (long long)d->co * d->ci * d->kh * d->kw;
    flip_transpose_kernel<<<ew_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(caffe_weights_dev, derived_dev, d->co, d->ci, d->kh, d->kw);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // extern "C"
