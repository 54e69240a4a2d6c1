// FP32 SIMT implicit-GEMM convolution / deconvolution for channel-fastest (NHWC) activations -- the
// exact-FP32 engine of the FlowNet2 conv stacks (see fn2_conv.cu for the reference citations).
//
// One kernel serves conv and deconv through a tap table:
//   * the launch enumerates a sub-grid (n, u, v) of output pixels: out(y, x) = (u*ou + oy0, v*ov + ox0)
//   * tap t reads in(u*su + dy[t], v*sv + dx[t]) and the packed weight rows of kernel position widx[t]
// Convolution: sub-grid = all outputs, su/sv = stride, dy = r - pad.  Deconvolution (gather form of col2im,
// util/im2col.cpp:158-190): one launch per output parity class (oy mod s, ox mod s) with only the kernel
// taps that hit that class (4 of 16 for the FlowNet 4x4/stride-2 upsamplers), so no multiply is wasted.
//
// CTA: 256 threads, tile 128 pixels x BN outputs (BN = 128/64/32 picked from Co), K step 16 channels of one tap,
// double-buffered shared memory, 128-bit global loads along the channel dimension, fused bias + leaky ReLU,
// 128-bit stores.  Small spatial maps (conv6: 7x16) are split over the taps (grid.z) into a workspace that a
// fixed-order reduction kernel sums (deterministic, no atomics).
#include "fn2_common.cuh"

namespace fn2 {

struct NhwcConv {
    int N, Hu, Wu, su, sv, ou, ov, oy0, ox0;
    int H, W, Ci, Co;
    long long in_sn, in_sh, in_sw, out_sn, out_sh, out_sw;
    int relu, has_bias;
    float slope;
    int vec_in, vec_out;        // 128-bit access allowed (alignment)
    int ntaps;
    int splits;                 // split-K: blockIdx.z handles steps [z*S/splits, (z+1)*S/splits), S = ntaps*cblocks
    short dy[49], dx[49], widx[49];
};

constexpr int NB_M = 128, NB_K = 16;

template <int BN>
__global__ void __launch_bounds__(256, 2) conv_nhwc_kernel(const float* __restrict__ in, const float* __restrict__ wp,
                                                           const float* __restrict__ bias, float* __restrict__ out,
                                                           float* __restrict__ partial, const NhwcConv p) {
    constexpr int TN = BN / 16;                       // outputs per thread along N (8, 4, 2)
    __shared__ __align__(16) float As[2][NB_K][NB_M + 4];
    __shared__ __align__(16) float Bs[2][NB_K][BN];
    const int tid = threadIdx.x;
    const long long M = (long long)p.N * p.Hu * p.Wu;
    const long long m0 = (long long)blockIdx.x * NB_M;
    const int n0 = blockIdx.y * BN;

    // ---- A loader state: two pixels per thread, one 4-channel chunk -------------------------------------
    const int a_chunk = tid & 3;
    int a_n[2], a_u[2], a_v[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const long long m = m0 + (tid >> 2) + 64 * i;
        if (m < M) {
            a_v[i] = (int)(m % p.Wu);
            a_u[i] = (int)((m / p.Wu) % p.Hu);
            a_n[i] = (int)(m / ((long long)p.Wu * p.Hu));
        } else { a_n[i] = -1; a_u[i] = 0; a_v[i] = 0; }
    }
    // ---- B loader: 16 rows x BN columns -------------------------------------------------------------------
    constexpr int B_F4 = NB_K * BN / 4;               // float4 per tile
    constexpr int B_PER_THREAD = (B_F4 + 255) / 256;  // 2, 1, 1
    constexpr int B_COLS4 = BN / 4;

    float4 a_reg[2];
    float4 b_reg[B_PER_THREAD];
    const float* a_ptr[2];
    bool a_ok[2];

    auto set_tap = [&](int t) {
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int iy = a_u[i] * p.su + p.dy[t], ix = a_v[i] * p.sv + p.dx[t];
            a_ok[i] = a_n[i] >= 0 && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
            a_ptr[i] = in + (a_ok[i] ? a_n[i] * p.in_sn + iy * p.in_sh + ix * p.in_sw : 0);
        }
    };
    auto load_tiles = [&](int t, int ci0) {
        const int c = ci0 + 4 * a_chunk;
#pragma unroll
        for (int i = 0; i < 2; i++) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (a_ok[i] && c < p.Ci) {
                const float* s = a_ptr[i] + c;
                if (p.vec_in) {
                    v = __ldg(reinterpret_cast<const float4*>(s));
                    if (c + 1 >= p.Ci) v.y = 0.f;
                    if (c + 2 >= p.Ci) v.z = 0.f;
                    if (c + 3 >= p.Ci) v.w = 0.f;
                } else {
                    v.x = __ldg(s);
                    if (c + 1 < p.Ci) v.y = __ldg(s + 1);
                    if (c + 2 < p.Ci) v.z = __ldg(s + 2);
                    if (c + 3 < p.Ci) v.w = __ldg(s + 3);
                }
            }
            a_reg[i] = v;
        }
        const float* wt = wp + (long long)p.widx[t] * p.Ci * p.Co;
#pragma unroll
        for (int i = 0; i < B_PER_THREAD; i++) {
            const int f = tid + 256 * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (f < B_F4) {
                const int row = f / B_COLS4, col = (f % B_COLS4) * 4;
                const int ci = ci0 + row;
                if (ci < p.Ci && n0 + col < p.Co)       // Co % 4 == 0 is a launch precondition
                    v = __ldg(reinterpret_cast<const float4*>(wt + (long long)ci * p.Co + n0 + col));
            }
            b_reg[i] = v;
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int mrow = (tid >> 2) + 64 * i;
            As[buf][4 * a_chunk + 0][mrow] = a_reg[i].x;
            As[buf][4 * a_chunk + 1][mrow] = a_reg[i].y;
            As[buf][4 * a_chunk + 2][mrow] = a_reg[i].z;
            As[buf][4 * a_chunk + 3][mrow] = a_reg[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_PER_THREAD; i++) {
            const int f = tid + 256 * i;
            if (f < B_F4) *reinterpret_cast<float4*>(&Bs[buf][f / B_COLS4][(f % B_COLS4) * 4]) = b_reg[i];
        }
    };

    const int tx = tid & 15, ty = tid >> 4;
    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

    const int cblocks = (p.Ci + NB_K - 1) / NB_K;
    const int all_steps = p.ntaps * cblocks;
    const int step_begin = (int)((long long)all_steps * blockIdx.z / p.splits);
    const int steps = (int)((long long)all_steps * (blockIdx.z + 1) / p.splits) - step_begin;
    int t = step_begin / cblocks, cb = step_begin % cblocks;
    if (steps > 0) {
        set_tap(t);
        load_tiles(t, cb * NB_K);
        store_tiles(0);
    }
    __syncthreads();
    for (int st = 0; st < steps; st++) {
        const int buf = st & 1;
        // advance (t, cb) to the next step and prefetch it into registers
        int nt = t, ncb = cb + 1;
        if (ncb == cblocks) { ncb = 0; nt = t + 1; }
        const bool more = st + 1 < steps;
        if (more) {
            if (nt != t) set_tap(nt);
            load_tiles(nt, ncb * NB_K);
        }
#pragma unroll
        for (int kk = 0; kk < NB_K; kk++) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4 + 64]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bv[TN];
            if constexpr (TN == 8) {
                const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4 + 64]);
                bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
                bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
            } else if constexpr (TN == 4) {
                const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
                bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
            } else {
                const float2 b0 = *reinterpret_cast<const float2*>(&Bs[buf][kk][tx * 2]);
                bv[0] = b0.x; bv[1] = b0.y;
            }
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < TN; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (more) {
            store_tiles(buf ^ 1);
            __syncthreads();
        }
        t = nt; cb = ncb;
    }

    // ---- epilogue ---------------------------------------------------------------------------------------------
    const bool split = partial != nullptr;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const long long m = m0 + ty * 4 + (i & 3) + (i >> 2) * 64;
        if (m >= M) continue;
        float* orow;
        if (split) {
            orow = partial + ((long long)blockIdx.z * M + m) * p.Co;
        } else {
            const int v = (int)(m % p.Wu);
            const int u = (int)((m / p.Wu) % p.Hu);
            const int n = (int)(m / ((long long)p.Wu * p.Hu));
            orow = out + n * p.out_sn + (u * p.ou + p.oy0) * p.out_sh + (v * p.ov + p.ox0) * p.out_sw;
        }
#pragma unroll
        for (int g = 0; g < (TN + 3) / 4; g++) {
            constexpr int GW = TN >= 4 ? 4 : TN;
            const int co = n0 + (TN == 2 ? tx * 2 : tx * 4 + g * 64);
            float v[GW];
#pragma unroll
            for (int e = 0; e < GW; e++) {
                float x = acc[i][g * 4 + e];
                if (!split) {
                    if (p.has_bias && co + e < p.Co) x += __ldg(bias + co + e);
                    if (p.relu) x = x > 0 ? x : x * p.slope;
                }
                v[e] = x;
            }
            bool vec = false;
            if constexpr (GW == 4) {
                vec = co + 3 < p.Co && (split || p.vec_out);
                if (vec) *reinterpret_cast<float4*>(orow + co) = make_float4(v[0], v[1], v[2], v[3]);
            }
            if (!vec) {
#pragma unroll
                for (int e = 0; e < GW; e++)
                    if (co + e < p.Co) orow[co + e] = v[e];
            }
        }
    }
}

// Fixed-order reduction of the split-K partials + bias + ReLU.
__global__ void conv_nhwc_reduce_kernel(const float* __restrict__ partial, const float* __restrict__ bias,
                                        float* __restrict__ out, int splits, const NhwcConv p) {
    const long long M = (long long)p.N * p.Hu * p.Wu;
    const long long total = M * p.Co;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(idx % p.Co);
        const long long m = idx / p.Co;
        float x = 0.f;
        for (int z = 0; z < splits; z++) x += partial[((long long)z * M + m) * p.Co + co];
        if (p.has_bias) x += __ldg(bias + co);
        if (p.relu) x = x > 0 ? x : x * p.slope;
        const int v = (int)(m % p.Wu);
        const int u = (int)((m / p.Wu) % p.Hu);
        const int n = (int)(m / ((long long)p.Wu * p.Hu));
        out[n * p.out_sn + (u * p.ou + p.oy0) * p.out_sh + (v * p.ov + p.ox0) * p.out_sw + co] = x;
    }
}

int conv_nhwc_eligible(const fn2_conv_desc* d, const T4& in, const T4& out) {
    if (in.sc != 1 || out.sc != 1) return 0;
    if (d->co % 4 || d->co < 8) return 0;
    if (d->kh * d->kw > 49) return 0;
    if (d->deconv && d->stride_h * d->stride_w > 16) return 0;
    return 1;
}

static int pick_bn(int co) { return co >= 96 ? 128 : (co >= 48 ? 64 : 32); }

// Split-K plan: when the (pixel tile x output tile) grid cannot fill the GPU, the K loop (taps x channel
// blocks) is cut into `splits` ranges whose partial tiles go to a workspace and are summed in fixed order.
static int plan_splits(long long M, int co, int ci, int ntaps) {
    const int bn = pick_bn(co);
    const long long ctas = ((M + NB_M - 1) / NB_M) * ((co + bn - 1) / bn);
    const int steps = ntaps * ((ci + NB_K - 1) / NB_K);
    const long long target = 2LL * num_sms();
    if (ctas >= target / 2 || steps < 16) return 1;
    long long z = (target + ctas - 1) / ctas;
    if (z > steps / 8) z = steps / 8;
    if (z > 32) z = 32;
    return z < 2 ? 1 : (int)z;
}

// Workspace (floats) the split-K path may need for this shape; 0 = never splits.
// The partials are written as float4: a caller's workspace may start anywhere 4-byte aligned, and the 4 floats of slack on top
// of them are the room to move it to a 16-byte boundary.
constexpr size_t NHWC_WS_SLACK = 4;

size_t conv_nhwc_workspace_floats(const fn2_conv_desc* d, int N, int Ho, int Wo) {
    if (!d->deconv) {
        const long long M = (long long)N * Ho * Wo;
        const int z = plan_splits(M, d->co, d->ci, d->kh * d->kw);
        return z > 1 ? (size_t)z * M * d->co + NHWC_WS_SLACK : 0;
    }
    // deconvolution: per parity class; the largest class decides
    const int sh = d->stride_h, sw = d->stride_w;
    const long long M = (long long)N * ((Ho + sh - 1) / sh) * ((Wo + sw - 1) / sw);
    const int taps = ((d->kh + sh - 1) / sh) * ((d->kw + sw - 1) / sw);
    const int z = plan_splits(M, d->co, d->ci, taps);
    return z > 1 ? (size_t)(z + 1) * M * d->co + NHWC_WS_SLACK : 0;
}

int conv_nhwc_forward(const fn2_conv_desc* d, const T4& in, const float* wp, const float* bias, const T4& out,
                      float* ws, size_t ws_floats, cudaStream_t st) {
    NhwcConv p;
    p.N = in.n; p.H = in.h; p.W = in.w; p.Ci = d->ci; p.Co = d->co;
    p.in_sn = in.sn; p.in_sh = in.sh; p.in_sw = in.sw;
    p.out_sn = out.sn; p.out_sh = out.sh; p.out_sw = out.sw;
    p.relu = d->relu; p.has_bias = d->has_bias; p.slope = d->negative_slope;
    p.vec_in = in.px_float4();          // both views are channel-fast (conv_nhwc_eligible)
    p.vec_out = out.px_float4();
    ws_floats = ws && ws_floats > NHWC_WS_SLACK ? ws_floats - NHWC_WS_SLACK : 0;
    ws = reinterpret_cast<float*>(((uintptr_t)ws + 15) & ~(uintptr_t)15);
    const int bn = pick_bn(d->co);
    auto launch = [&](dim3 grid, float* partial) {
        if (bn == 128) conv_nhwc_kernel<128><<<grid, 256, 0, st>>>(in.p, wp, bias, out.p, partial, p);
        else if (bn == 64) conv_nhwc_kernel<64><<<grid, 256, 0, st>>>(in.p, wp, bias, out.p, partial, p);
        else conv_nhwc_kernel<32><<<grid, 256, 0, st>>>(in.p, wp, bias, out.p, partial, p);
    };
    ConvTaps tp;
    conv_taps(d, out.h, out.w, &tp);
    p.su = d->deconv ? 1 : d->stride_h; p.sv = d->deconv ? 1 : d->stride_w; p.ou = tp.ou; p.ov = tp.ov;
    // one launch per output parity class (a convolution has one)
    for (int c = 0; c < tp.ncls; c++) {
        p.Hu = tp.Hu[c]; p.Wu = tp.Wu[c]; p.oy0 = tp.oy0[c]; p.ox0 = tp.ox0[c];
        p.ntaps = tp.ntaps[c];
        for (int t = 0; t < p.ntaps; t++) {
            p.dy[t] = tp.dy[tp.tap0[c] + t]; p.dx[t] = tp.dx[tp.tap0[c] + t]; p.widx[t] = tp.widx[tp.tap0[c] + t];
        }
        const long long M = (long long)p.N * p.Hu * p.Wu;
        dim3 grid((unsigned)((M + NB_M - 1) / NB_M), (unsigned)((d->co + bn - 1) / bn), 1);
        p.splits = p.ntaps > 0 ? plan_splits(M, d->co, d->ci, p.ntaps) : 1;
        if (p.splits > 1 && ws && ws_floats >= (size_t)p.splits * M * d->co) {
            grid.z = p.splits;
            launch(grid, ws);
            FN2_LAUNCH_CHECK();
            conv_nhwc_reduce_kernel<<<ew_grid(M * p.Co, 256), 256, 0, st>>>(ws, bias, out.p, p.splits, p);
        } else {
            p.splits = 1;
            launch(grid, nullptr);     // a class without taps still gets bias (+ReLU)
        }
        FN2_LAUNCH_CHECK();
    }
    return FN2_OK;
}

}  // namespace fn2
