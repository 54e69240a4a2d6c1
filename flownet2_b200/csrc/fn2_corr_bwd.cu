// Correlation backward (2-D and 1-D, MULTIPLY and SUBTRACT), on the geometry of fn2_corr.cu (CorrGeo).
//
// Reference: CorrelateDataBackward0/1 (correlation_layer.cu:118-249), ...Subtract (:298-427), correlation_layer1d.cu:48-420.
// The reference launches one thread per bottom element that walks all displacements and, inside, the range of top positions
// whose patch covers the element.  Here the adjoint is FACTORISED instead (the patch walk does not depend on the channel):
//
//   G[n, d, q]   = sum over the k x k patch taps (j, i) with (q - tap - (md - pad)) divisible by stride_1 and inside the top
//                  of topdiff[n, d, y, x]                                  -- "patch sum", bottom resolution, channel-free
//   d bottom0[q] = 1/(k*k*C) * sum_d G[d, q]          * M[q + disp(d)]     M = bottom1            (MULTIPLY)
//   d bottom1[q] = 1/(k*k*C) * sum_d G[d, q - disp(d)] * M'[q - disp(d)]   M' = bottom0           (MULTIPLY)
//   SUBTRACT uses the reference's sign map in place of M / M': s(q) = (bottom0[q] >= bottom1[q]) ? +1 : -1 evaluated AT THE
//   DISPLACED position for both gradients (:327-329, :397-399), +s for bottom0 and -s for bottom1, and +-1 (not 0) outside
//   the image, because the reference compares its two zero-padded copies there.
// When k = 1, stride_1 = 1 and pad = md, G is topdiff itself (identity G); otherwise corr_patchsum_kernel forms it first.
// Routes (corr_bwd_plan, corr_backward):
//   * fast  -- FlowNet2-C's layer (MULTIPLY, identity G, 21 x 21 displacements, stride_2 <= 2, C % 32 == 0) on channel-fast
//              maps with 16-byte aligned pixels: corr_bwd_fast_kernel on the stride_2 parity planes.  Workspace N*H*W*D.
//   * tiled -- everything else: one shared-memory tiled apply kernel.  An 8 x 8 pixel tile keeps its G rows (64 x D floats)
//              resident and streams the (8 + 2*reach)^2 halo of M in 8-channel chunks; thread = (pixel, 2 channels), D fused
//              multiply-adds per chunk and channel, fixed summation order (no atomics).  Workspace: N*H*W*D for the patch sum
//              unless G is the identity, plus N*H*W*C for the SUBTRACT sign map.
#include "fn2_common.cuh"

namespace fn2 {

namespace {

constexpr int CB_TILE = 8;                 // tile edge (pixels)
constexpr int CB_CH = 8;                   // channels per chunk

struct CbP {
    int N, C, H, W;                        // bottom shape
    int D;                                 // displacements (top channels)
    int topH, topW;
    int k, s1, md, pad;                    // patch walk
    int ypatch_off;                        // (md - pad) vertically; 0 for Correlation1D rows (no vertical displacement border)
    int reach_y, reach_x;                  // max |dy|, |dx| over the displacement table
    int identity_g;                        // G == topdiff (k == 1, s1 == 1, offsets 0, top size == bottom size)
    float scale, oob;                      // 1 / (k*k*C); value of M outside the image
    short dy[441], dx[441];
};

// patch sum: G[n][q][d] (d fastest) = sum of topdiff[n][d][y][x] over the top positions whose patch covers q
__global__ void corr_patchsum_kernel(T4 td, float* __restrict__ g, CbP p) {
    const long long total = (long long)p.N * p.H * p.W * p.D;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(idx % p.D);
        long long r = idx / p.D;
        const int xx = (int)(r % p.W); r /= p.W;
        const int yy = (int)(r % p.H);
        const int n = (int)(r / p.H);
        float acc = 0.f;
        for (int j = 0; j < p.k; j++) {
            const int ty = yy - j - p.ypatch_off;                      // = y * s1
            if (ty < 0 || ty % p.s1) continue;
            const int y = ty / p.s1;
            if (y >= p.topH) continue;
            for (int i = 0; i < p.k; i++) {
                const int tx = xx - i - (p.md - p.pad);
                if (tx < 0 || tx % p.s1) continue;
                const int x = tx / p.s1;
                if (x >= p.topW) continue;
                acc += td.p[td.off(n, d, y, x)];
            }
        }
        g[idx] = acc;
    }
}

// sign map of the SUBTRACT gradients
__global__ void corr_sign_kernel(T4 a, T4 b, float* __restrict__ s) {
    const long long total = a.count();
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % a.c);
        long long r = idx / a.c;
        const int x = (int)(r % a.w); r /= a.w;
        const int y = (int)(r % a.h);
        const int n = (int)(r / a.h);
        s[idx] = a.p[a.off(n, c, y, x)] >= b.p[b.off(n, c, y, x)] ? 1.f : -1.f;
    }
}

// MODE 0: out[q] = scale * sum_d G[q][d] * M[q + disp(d)]        (gradient w.r.t. bottom0)
// MODE 1: out[q] = scale * sum_d G[q - disp(d)][d] * M[q - disp(d)]   (gradient w.r.t. bottom1), M already carries its sign
// G: dense [N][H][W][D] or (identity_g) the top diff tensor itself; M: strided view, channel-fast or not.
template <int MODE>
__global__ void __launch_bounds__(256) corr_apply_kernel(const float* __restrict__ gdense, T4 td, T4 m, T4 out, CbP p, float msign) {
    extern __shared__ float sm[];
    const int hw = CB_TILE + 2 * p.reach_x, hh = CB_TILE + 2 * p.reach_y;
    float* gs = sm;                                        // [64][D]
    float* hs = sm + 64 * p.D;                             // [hh][hw][CB_CH]
    const int tiles_x = (p.W + CB_TILE - 1) / CB_TILE, tiles_y = (p.H + CB_TILE - 1) / CB_TILE;
    const int tid = threadIdx.x;
    const int px = tid >> 2, cg = tid & 3;                 // pixel 0..63, channel pair 0..3
    const int ty_ = px >> 3, tx_ = px & 7;
    for (int tile = blockIdx.x; tile < p.N * tiles_y * tiles_x; tile += gridDim.x) {
        const int n = tile / (tiles_y * tiles_x);
        const int t2 = tile - n * tiles_y * tiles_x;
        const int y0 = (t2 / tiles_x) * CB_TILE, x0 = (t2 % tiles_x) * CB_TILE;
        __syncthreads();
        // G rows of the tile: gs[pixel][d]
        for (int idx = tid; idx < 64 * p.D; idx += 256) {
            const int q = idx / p.D, d = idx - q * p.D;
            int y = y0 + (q >> 3), x = x0 + (q & 7);
            if (MODE == 1) { y -= p.dy[d]; x -= p.dx[d]; }
            float v = 0.f;
            if (y >= 0 && y < p.H && x >= 0 && x < p.W) {
                if (y0 + (q >> 3) < p.H && x0 + (q & 7) < p.W)
                    v = p.identity_g ? td.p[td.off(n, d, y, x)] : gdense[(((long long)n * p.H + y) * p.W + x) * p.D + d];
            }
            gs[idx] = v;
        }
        const int y = y0 + ty_, x = x0 + tx_;
        for (int c0 = 0; c0 < p.C; c0 += CB_CH) {
            __syncthreads();
            for (int idx = tid; idx < hh * hw * CB_CH; idx += 256) {
                const int c = idx % CB_CH, hpix = idx / CB_CH;
                const int hy = hpix / hw, hx = hpix - hy * hw;
                const int yy = y0 - p.reach_y + hy, xx = x0 - p.reach_x + hx;
                float v = 0.f;
                if (c0 + c < p.C) v = (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) ? msign * m.p[m.off(n, c0 + c, yy, xx)] : p.oob * msign;
                hs[idx] = v;
            }
            __syncthreads();
            float a0 = 0.f, a1 = 0.f;
            const float* grow = gs + px * p.D;
            const float* hbase = hs + ((ty_ + p.reach_y) * hw + (tx_ + p.reach_x)) * CB_CH + 2 * cg;
#pragma unroll 4
            for (int d = 0; d < p.D; d++) {
                const int off = (MODE == 0 ? 1 : -1) * ((int)p.dy[d] * hw + (int)p.dx[d]) * CB_CH;
                const float g = grow[d];
                const float2 v = *reinterpret_cast<const float2*>(hbase + off);
                a0 = fmaf(g, v.x, a0);
                a1 = fmaf(g, v.y, a1);
            }
            if (y < p.H && x < p.W) {
                const int c = c0 + 2 * cg;
                if (c < p.C) out.p[out.off(n, c, y, x)] = a0 * p.scale;
                if (c + 1 < p.C) out.p[out.off(n, c + 1, y, x)] = a1 * p.scale;
            }
        }
    }
}

// ---- fast path: FlowNet2-C's layer (MULTIPLY, k = 1, stride_1 = 1, pad = md, R = md / stride_2 = 10, C % 32 == 0) ----------------
// out[q][c] = scale * sum over (dj, di) of Gx[q][dj][di] * M[q + SGN * (dj - R, di - R) * stride_2][c]
//   bottom0 gradient: Gx = top diff, M = bottom1, SGN = +1
//   bottom1 gradient: Gx = the top diff SHIFTED per displacement (corr_shift_kernel: Gx[q][d] = topdiff[q - disp(d)][d]), M = bottom0, SGN = -1
// A displacement only connects pixels of the same stride_2 parity class, so a work unit is (sample, parity class, 8 x 16 tile of
// that class's plane, 32 channels): the (8 + 2R) x (16 + 2R) plane-pixel halo of M sits in shared memory (129 KB), the tile's Gx
// values of one displacement row (128 x 21) are re-staged per dj.  Thread = 4 consecutive pixels x 4 channels: a halo float4 is
// loaded once and feeds up to 4 pixels (pixel i meets it with di = t - i), the pixel's 21 Gx values of the row live in registers:
// 336 FMAs per 24 + 24 128-bit shared loads.  Fixed summation order (dj, then the halo column), no atomics.
constexpr int CF_R = 10, CF_DW = 2 * CF_R + 1, CF_TH = 8, CF_TW = 16, CF_HH = CF_TH + 2 * CF_R, CF_HW = CF_TW + 2 * CF_R, CF_GROW = 24;
constexpr int CF_GB = 3;                                  // displacement rows staged per step (Gx values prefetched one step ahead)
constexpr int CF_GSTAGE = CF_GB * CF_TH * CF_TW * CF_GROW; // floats per stage
constexpr int CF_SMEM = (CF_HH * CF_HW * 32 + CF_GSTAGE) * (int)sizeof(float);
static_assert(CF_DW % CF_GB == 0 && CF_GSTAGE % 256 == 0, "stage shape");

struct CfP { int N, C, H, W, S, tiles_x, tiles_y, cchunks; float scale; };

template <int SGN>
__global__ void __launch_bounds__(256, 1) corr_bwd_fast_kernel(T4 g, T4 m, T4 out, CfP p) {
    extern __shared__ __align__(16) float cfsm[];
    float* halo = cfsm;                                   // [HH * HW][32]
    float* gs = cfsm + CF_HH * CF_HW * 32;                // [128][GROW]
    const int tid = threadIdx.x;
    const int cg = tid & 7, pg = tid >> 3;                // channel float4 0..7, pixel group 0..31
    const int row = pg >> 2, xg = pg & 3;                 // tile row 0..7, group of 4 pixels 0..3
    const int units = p.N * p.S * p.S * p.tiles_y * p.tiles_x * p.cchunks;
    for (int unit = blockIdx.x; unit < units; unit += gridDim.x) {
        int r = unit;
        const int cc = r % p.cchunks; r /= p.cchunks;
        const int tx = r % p.tiles_x; r /= p.tiles_x;
        const int ty = r % p.tiles_y; r /= p.tiles_y;
        const int cls = r % (p.S * p.S), n = r / (p.S * p.S);
        const int py = cls / p.S, px = cls % p.S;
        const int u0 = ty * CF_TH, v0 = tx * CF_TW, c0 = cc * 32;
        __syncthreads();
        for (int idx = tid; idx < CF_HH * CF_HW * 8; idx += 256) {
            const int hp = idx >> 3, c4 = idx & 7;
            const int hy = hp / CF_HW, hx = hp - hy * CF_HW;
            const int y = (u0 - CF_R + hy) * p.S + py, x = (v0 - CF_R + hx) * p.S + px;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (y >= 0 && y < p.H && x >= 0 && x < p.W) v = *reinterpret_cast<const float4*>(m.p + m.off(n, c0 + 4 * c4, y, x));
            *reinterpret_cast<float4*>(halo + hp * 32 + 4 * c4) = v;
        }
        float4 acc[4];
#pragma unroll
        for (int i = 0; i < 4; i++) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        // Gx values of CF_GB displacement rows per step; the next step's values are fetched into registers while this one computes
        float pre[CF_GSTAGE / 256];
        auto gfetch = [&](int dj0) {
#pragma unroll
            for (int j = 0; j < CF_GSTAGE / 256; j++) {
                const int idx = tid + 256 * j;
                const int b = idx / (CF_TH * CF_TW * CF_GROW), rem = idx - b * (CF_TH * CF_TW * CF_GROW);
                const int q = rem / CF_GROW, di = rem - q * CF_GROW;
                const int y = (u0 + (q >> 4)) * p.S + py, x = (v0 + (q & 15)) * p.S + px;
                pre[j] = (di < CF_DW && y < p.H && x < p.W) ? g.p[g.off(n, (dj0 + b) * CF_DW + di, y, x)] : 0.f;
            }
        };
        gfetch(0);
#pragma unroll 1
        for (int dj = 0; dj < CF_DW; dj++) {
            if (dj % CF_GB == 0) {
                __syncthreads();
#pragma unroll
                for (int j = 0; j < CF_GSTAGE / 256; j++) gs[tid + 256 * j] = pre[j];
                __syncthreads();
                if (dj + CF_GB < CF_DW) gfetch(dj + CF_GB);
            }
            const float* gsr = gs + (dj % CF_GB) * (CF_TH * CF_TW * CF_GROW);
            float gr[4][CF_GROW];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int k4 = 0; k4 < CF_GROW / 4; k4++) {
                    const float4 t = *reinterpret_cast<const float4*>(gsr + (row * CF_TW + xg * 4 + i) * CF_GROW + 4 * k4);
                    gr[i][4 * k4] = t.x; gr[i][4 * k4 + 1] = t.y; gr[i][4 * k4 + 2] = t.z; gr[i][4 * k4 + 3] = t.w;
                }
            // halo row / first halo column of this thread for displacement row dj
            const int hrow = SGN > 0 ? row + dj : row + 2 * CF_R - dj;
            const float* hb = halo + (hrow * CF_HW + xg * 4) * 32 + 4 * cg;
#pragma unroll
            for (int t = 0; t < CF_DW + 3; t++) {
                const float4 mv = *reinterpret_cast<const float4*>(hb + t * 32);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    // halo column xg*4 + t is pixel i's column + di (SGN > 0) resp. + 2R - di (SGN < 0)
                    const int e = t - i;
                    if (e >= 0 && e < CF_DW) {
                        const float gv = gr[i][SGN > 0 ? e : 2 * CF_R - e];
                        acc[i].x = fmaf(gv, mv.x, acc[i].x); acc[i].y = fmaf(gv, mv.y, acc[i].y);
                        acc[i].z = fmaf(gv, mv.z, acc[i].z); acc[i].w = fmaf(gv, mv.w, acc[i].w);
                    }
                }
            }
        }
        const int y = (u0 + row) * p.S + py;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int x = (v0 + xg * 4 + i) * p.S + px;
            if (y < p.H && x < p.W)
                *reinterpret_cast<float4*>(out.p + out.off(n, c0 + 4 * cg, y, x)) =
                    make_float4(acc[i].x * p.scale, acc[i].y * p.scale, acc[i].z * p.scale, acc[i].w * p.scale);
        }
    }
}

// Gx[n][y][x][d] = topdiff[n][d][y - dy(d)][x - dx(d)] (0 outside): the bottom1 gradient then has the bottom0 gradient's form
__global__ void corr_shift_kernel(T4 td, float* __restrict__ gx, int R, int S) {
    const int Dw = 2 * R + 1, D = Dw * Dw;
    const long long total = (long long)td.n * td.h * td.w * D;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(idx % D);
        long long r = idx / D;
        const int x = (int)(r % td.w); r /= td.w;
        const int y = (int)(r % td.h);
        const int n = (int)(r / td.h);
        const int yy = y - (d / Dw - R) * S, xx = x - (d % Dw - R) * S;
        gx[idx] = (yy >= 0 && yy < td.h && xx >= 0 && xx < td.w) ? td.p[td.off(n, d, yy, xx)] : 0.f;
    }
}


// Backward route of a layer, from its shape.  G is the top diff itself when the patch walk is the identity (k 1, stride_1 1,
// pad = md); otherwise the tiled route first forms the patch sum.  FlowNet2-C's class -- MULTIPLY, G = top diff, the 21 x 21
// displacement grid, stride_2 <= 2, C % 32 == 0 -- takes the fast kernel when the four bottom maps are channel-fast with
// 16-byte aligned pixels too (corr_backward); it stages the shifted top diff in the workspace.
struct CorrBwdPlan {
    bool fast;              // shape of the fast route
    bool patch_sum;         // the tiled route needs the patch sum
    size_t g_floats;        // N*H*W*D: the fast route's shifted top diff, or the patch sum
    size_t s_floats;        // SUBTRACT: the sign map, N*H*W*C
    size_t tiled_floats() const { return (patch_sum ? g_floats : 0) + s_floats; }
};

CorrBwdPlan corr_bwd_plan(const CorrGeo& g, int N, int C, int H, int W, int corr_type) {
    CorrBwdPlan pl;
    pl.patch_sum = !(g.k == 1 && g.s1 == 1 && g.pad == g.md && g.topH == H && g.topW == W);
    pl.fast = corr_type == 0 && !pl.patch_sum && g.topC == CF_DW * CF_DW && g.Dx == CF_DW && g.xs == -CF_R && g.ys == -CF_R &&
              g.s2 <= 2 && C % 32 == 0;
    pl.g_floats = (size_t)N * H * W * g.topC;
    pl.s_floats = corr_type == 1 ? (size_t)N * H * W * C : 0;
    return pl;
}

int corr_fast_run(const T4& b0, const T4& b1, const T4& td, const T4& d0, const T4& d1, const CbP& p, int s2, float* ws, cudaStream_t st) {
    CfP f;
    f.N = p.N; f.C = p.C; f.H = p.H; f.W = p.W; f.S = s2; f.scale = p.scale; f.cchunks = p.C / 32;
    const int Hp = (p.H + s2 - 1) / s2, Wp = (p.W + s2 - 1) / s2;
    f.tiles_y = (Hp + CF_TH - 1) / CF_TH; f.tiles_x = (Wp + CF_TW - 1) / CF_TW;
    const int units = f.N * s2 * s2 * f.tiles_y * f.tiles_x * f.cchunks;
    const int grid = min(units, num_sms());
    FN2_CUDA(cudaFuncSetAttribute(corr_bwd_fast_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, CF_SMEM));
    corr_bwd_fast_kernel<1><<<grid, 256, CF_SMEM, st>>>(td, b1, d0, f);
    FN2_LAUNCH_CHECK();
    corr_shift_kernel<<<ew_grid((long long)p.N * p.H * p.W * p.D, 256), 256, 0, st>>>(td, ws, CF_R, s2);
    FN2_LAUNCH_CHECK();
    T4 gx;
    gx.p = ws; gx.n = p.N; gx.c = p.D; gx.h = p.H; gx.w = p.W;
    gx.sc = 1; gx.sw = p.D; gx.sh = (long long)p.W * p.D; gx.sn = (long long)p.H * p.W * p.D;
    FN2_CUDA(cudaFuncSetAttribute(corr_bwd_fast_kernel<-1>, cudaFuncAttributeMaxDynamicSharedMemorySize, CF_SMEM));
    corr_bwd_fast_kernel<-1><<<grid, 256, CF_SMEM, st>>>(gx, b0, d1, f);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int corr_tiled_run(const T4& b0, const T4& b1, const T4& td, const T4& d0, const T4& d1, CbP& p, int corr_type, float* g,
                   float* sgn, cudaStream_t st) {
    if (!p.identity_g) {
        corr_patchsum_kernel<<<ew_grid((long long)p.N * p.H * p.W * p.D, 256), 256, 0, st>>>(td, g, p);
        FN2_LAUNCH_CHECK();
    }
    T4 m0 = b1, m1 = b0;
    float s0 = 1.f, s1 = 1.f;
    p.oob = 0.f;
    if (corr_type == 1) {
        corr_sign_kernel<<<ew_grid(b0.count(), 256), 256, 0, st>>>(b0, b1, sgn);
        FN2_LAUNCH_CHECK();
        T4 sv; sv.p = sgn; sv.n = p.N; sv.c = p.C; sv.h = p.H; sv.w = p.W;
        sv.sc = 1; sv.sw = p.C; sv.sh = (long long)p.W * p.C; sv.sn = (long long)p.H * p.W * p.C;
        m0 = sv; m1 = sv; s0 = 1.f; s1 = -1.f; p.oob = 1.f;
    }
    const int hw = CB_TILE + 2 * p.reach_x, hh = CB_TILE + 2 * p.reach_y;
    const size_t smem = ((size_t)64 * p.D + (size_t)hh * hw * CB_CH) * sizeof(float);
    if (smem > 220 * 1024) { set_error("correlation_backward: displacement window too large for the tiled kernel (%zu B)", smem); return FN2_ERR_INVALID; }
    const int tiles = p.N * ((p.H + CB_TILE - 1) / CB_TILE) * ((p.W + CB_TILE - 1) / CB_TILE);
    const int grid = min(tiles, num_sms());
    if (smem > 48 * 1024) FN2_CUDA(cudaFuncSetAttribute(corr_apply_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_apply_kernel<0><<<grid, 256, smem, st>>>(g, td, m0, d0, p, s0);
    FN2_LAUNCH_CHECK();
    if (smem > 48 * 1024) FN2_CUDA(cudaFuncSetAttribute(corr_apply_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_apply_kernel<1><<<grid, 256, smem, st>>>(g, td, m1, d1, p, s1);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // namespace

size_t corr_bwd_workspace_floats(const CorrGeo& g, int N, int C, int H, int W, int corr_type) {
    const CorrBwdPlan pl = corr_bwd_plan(g, N, C, H, W, corr_type);
    return pl.fast ? pl.g_floats : pl.tiled_floats();
}

int corr_backward(const CorrGeo& g, const T4& b0, const T4& b1, const T4& td, const T4& d0, const T4& d1, int corr_type,
                  float* ws, size_t ws_floats, cudaStream_t st) {
    const CorrBwdPlan pl = corr_bwd_plan(g, b0.n, b0.c, b0.h, b0.w, corr_type);
    if (g.topC > 441) { set_error("correlation_backward: more than 441 displacements"); return FN2_ERR_INVALID; }
    CbP p;
    memset(&p, 0, sizeof(p));
    p.N = b0.n; p.C = b0.c; p.H = b0.h; p.W = b0.w;
    p.D = g.topC;
    p.topH = g.topH; p.topW = g.topW; p.k = g.k; p.s1 = g.s1; p.md = g.md; p.pad = g.pad; p.ypatch_off = g.y0;
    for (int tc = 0; tc < p.D; tc++) {
        p.dy[tc] = (short)((tc / g.Dx + g.ys) * g.s2);
        p.dx[tc] = (short)((tc % g.Dx + g.xs) * g.s2);
    }
    p.reach_x = max(-g.xs, g.Dx - 1 + g.xs) * g.s2;
    p.reach_y = max(-g.ys, g.topC / g.Dx - 1 + g.ys) * g.s2;
    p.identity_g = pl.patch_sum ? 0 : 1;
    p.scale = 1.f / (float)(g.k * g.k * p.C);
    if (pl.fast && b0.px_float4() && b1.px_float4() && d0.px_float4() && d1.px_float4()) {
        if (!ws || ws_floats < pl.g_floats) { set_error("correlation_backward: workspace too small"); return FN2_ERR_WORKSPACE; }
        return corr_fast_run(b0, b1, td, d0, d1, p, g.s2, ws, st);
    }
    const size_t need = pl.tiled_floats();
    if (need > ws_floats || (!ws && need)) { set_error("correlation_backward: workspace too small (%zu floats needed)", need); return FN2_ERR_WORKSPACE; }
    return corr_tiled_run(b0, b1, td, d0, d1, p, corr_type, ws, ws + (pl.patch_sum ? pl.g_floats : 0), st);
}

}  // namespace fn2
