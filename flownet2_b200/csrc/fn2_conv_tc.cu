// wgmma implicit-GEMM convolution + deconvolution engine (sm_90a), FP32-faithful.
//
// GEMM view per CTA: D[128 pixels x NT outputs] = sum over (kernel tap, 32-channel block) A_tap[128 x 32] * W_tap[NT x 32]^T
//   * A (activations, NHWC) : one TMA box per step straight from the activation tensor -- {32 ch, tw, th} with element
//     strides = conv stride and out-of-bounds zero fill, so padding, stride and the channel tail cost nothing and no
//     im2col buffer exists.  Lands as a K-major SWIZZLE_128B tile of raw FP32.
//   * W (weights) : packed once as [hi|lo][tap][Co][Ci32] (TF32 split), TMA boxes {32, NT}, K-major SWIZZLE_128B.
//   * 3xTF32: a = a_hi + a_lo, w = w_hi + w_lo (each rounded to TF32), D = a_hi*w_hi + a_hi*w_lo + a_lo*w_hi.
//     The activation split is done by the MMA warpgroups themselves: each thread reads its elements of the raw tile
//     straight into the wgmma A register fragment and splits them there (RS form: A from registers, W from shared memory).
//   * FP16 route (NT == 128, plain K blocks: three quarters of FlowNet2's flops): FP16 has TF32's 11-bit significand at half
//     the tensor-pipe cost, and a power-of-two scale covers its narrow exponent range exactly.  Per K step and pixel row,
//     a 2^-e = hi + lo'' (e from the row's largest |a|); per layer, w 2^-f = w_hi + 2^-11 w_lo' (f from the largest |w|),
//     packed as W_A = 2^11 w_hi, W_B = w_lo' (and W_C = w_hi, which no kernel reads).  Per 16-channel half,
//     lo'' W_A + hi W_B + hi W_A = 2^(11-e-f) a w (m64n128k16 f16 MMAs, two weight tiles per K step) into the chunk
//     accumulator, scaled back exactly when it is folded.
//   * Accumulation: the tensor core truncates its FP32 accumulator, which over K up to 9216 and ~60 layers would shrink
//     the flow.  Therefore the MMAs only chain over short chunks (kd K steps) in a register accumulator that is then added
//     into a second, FP32 register accumulator with round-to-nearest, applying the mean truncation loss of a chain of that
//     length as a correction.  Within a step the two cross terms (2^-11 smaller) are issued before a_hi*w_hi, so they
//     enter the chunk accumulator while it is still small.
//   * Epilogue: the accumulator fragments go through shared memory to 128-bit stores, consecutive threads along a pixel's
//     channels (each warp stores whole pixels): + bias, leaky ReLU, strided NHWC output view (or raw partials into the
//     workspace when the K loop is split over SMs).
// Persistent kernel, one CTA per SM walking the tile list (pixel tile x Co tile x deconv parity class x K split).
// Warp roles (384 threads, setmaxnreg re-balances registers): warp 0 TMA producer, warpgroups 1 and 2 the MMAs and the
// epilogue of tile rows 0-63 and 64-127.  Small-Ci inputs use kernel-row or tap-group packing of the K blocks
// (tc_weights).  DESIGN.md section 3 has the reasoning behind each of these choices.
#include <cuda.h>
#include <cuda_fp16.h>
#include <mutex>
#include <type_traits>

#include "fn2_common.cuh"
#include "fn2_tc_ptx.cuh"

namespace fn2 {

namespace {

constexpr int TC_THREADS = 384;
constexpr int A_TILE_BYTES = 128 * 128;          // 128 pixels x 32 fp32

struct TcParams {
    int N, su, sv, ou, ov;                        // sub-grid / mapping (see fn2_conv_nhwc.cu)
    int ncls;                                     // output parity classes handled by this launch (grid.z)
    int cls_Hu[4], cls_Wu[4], cls_oy0[4], cls_ox0[4], cls_tap0[4], cls_ntaps[4];
    int cblocks;                                  // ceil(Ci / 32)
    long long out_sn, out_sh, out_sw;
    int relu, has_bias;
    float slope;
    int tw, th, tiles_x, tiles_y;
    int kd;                                       // channel blocks per tensor-core accumulation chain
    int Ho, Wo;                                   // output size
    // K split (tc_split_plan): the tiles [split_first, ntotal) are cut into split_z K ranges each, which run on different SMs
    // as consecutive tile units; their raw partial tiles go to the workspace and tc_split_reduce_kernel sums them.
    // split_z = 1: unsplit (split_first = ntotal).
    int split_first, split_z, ntotal;
    FastDiv d_ntiles, d_cotiles, d_tiles_x, d_tiles_y, d_split_z;
    // Correlation on the same pipeline (corr_tc_forward): a unit = (sample, parity plane, 128-pixel tile of map 0, block of
    // cbw x cbh halo pixels of map 1); D[pixel][halo pixel] = <a, b> over C channels; the epilogue keeps the band that
    // lies inside the (2R+1)^2 displacement window.  W tiles are halo-pixel tiles of the pre-split map 1.
    int cR, cS, cD, cbw, cbh, cnt;
    float cscale;
    int ntiles, cotiles, total;                   // pixel tiles, Co tiles, all tiles
    int gcs;                                      // tap-group packing for Ci <= 16: padded channels per tap (4/8/12/16), 0 = off
    // kernel-row packing for Ci <= 16 on a dense input (pixel stride == rcs floats, guard band around the blob): the kw taps
    // of one kernel row are CONTIGUOUS in memory for every output pixel, so one K block = 32 consecutive floats of that run.
    int rowmode, rcs, rblocks, rsteps, rkw, rpad, rW;   // rblocks = ceil(kw*rcs/32) K blocks per kernel row, rsteps = kh*rblocks
    // Weight gradient on the same pipeline (conv_tc_wgrad): a unit = (kernel tap, 128 channels of the shifted map, NT channels of
    // the unshifted map, range of 32-pixel K segments); D[big channel][small channel] = sum over the segments' pixels.
    // Maps with few channels (wg_G = 8 .. 64 rows per tap) put 128 / wg_G taps side by side in one 128-row tile (wg_TPT).
    int wg_S, wg_ST, wg_BT, wg_segs, wg_segs_x, wg_sx, wg_G, wg_TPT, wg_taps;
    short dy[49], dx[49], widx[49];
    const uint32_t* wmax;                         // FP16 route: bits of the layer's largest |w|, behind the packed tiles
};

// W stage = two tiles: TF32 hi and lo [NT][32 floats], or on the FP16 route (NT == 128, plain K blocks) W_A and W_B
// [NT][32 halves].  The packed FP16 layout still holds a third tile, W_C, after them (tc_pack_f16_kernel); no kernel reads it,
// and it stays only because the packed format and its size are pinned: the stage box takes the first two.
template <int NT, bool F16 = false> struct TcGeo {
    static constexpr int B_TILE_BYTES = F16 ? NT * 64 : NT * 128;
    static constexpr int STAGE_BYTES = A_TILE_BYTES + 2 * B_TILE_BYTES;
    // ring of R shared-memory stages (raw A tile + W tiles), then the epilogue's staging buffer [128 pixels][STG]
    // (FP16: 5 stages of 32 KB would fit, and measured no faster than 4: the two-tile stage's gain is its bytes, DESIGN.md section 6)
    static constexpr int R = F16 ? 4 : (NT == 128 ? 3 : (NT == 64 ? 4 : 6));
    static constexpr int STG = NT + 4;                                             // floats per staged pixel row
    static constexpr int STG_BYTES = 128 * STG * 4;
    static constexpr int SMEM = R * STAGE_BYTES + STG_BYTES + 1024;
    // NT <= 64 (WIDE): the W stage holds [w_hi rows ; w_lo rows] back to back, so ONE MMA with N = 2*NT computes
    //   a_hi*[w_hi|w_lo] into two column blocks and a second one (N = NT, an accumulator of its own: MMAs of different
    //   shapes are not ordered on shared accumulator registers) computes a_lo*w_hi.  NT == 128: all three products chain into one accumulator, cross terms first in every step.
    static constexpr bool WIDE = NT <= 64;
    static constexpr int MMAS_PER_STEP = F16 ? 2 : 4;                             // a_hi*w_hi MMAs per step (the chain that truncates)
    static constexpr float TRUNC_LOSS = F16 ? TRUNC_LOSS_PER_MMA_F16 : TRUNC_LOSS_PER_MMA;
    static_assert(SMEM <= 227 * 1024, "shared memory overflow");
};

// one output tile: 128 pixels (th x tw) of one sample and parity class, NT output channels
struct TcTile {
    int n, u0, v0, co0, cls, tap0, ntaps, steps;
    int k0;                                       // first K step of this unit
    int slot;                                     // >= 0: raw partial sums go to workspace slot `slot` (K split)
    bool valid;
};
// MODE (compile time, so that each instantiation's role loops stay small -- the all-in-one kernel had ~1900 SASS instructions in
// the converter loop and stalled on instruction fetch): 0 plain K blocks, 1 tap groups, 2 kernel rows, 3 correlation
enum { TC_PLAIN = 0, TC_GROUP = 1, TC_ROW = 2, TC_CORR = 3, TC_WGRAD = 4 };
// the instantiations that take the FP16 route: the forward of the NT = 128 layers in plain K-block mode
__host__ __device__ constexpr bool tc_f16(int NT, int MODE) { return NT == 128 && MODE == TC_PLAIN; }

// FP16 route, weights: one exponent f per layer from its largest |w| (the float bits `maxbits` that tc_absmax_kernel leaves
// behind the packed tiles) puts the largest scaled weight in [8, 16), so that W_A = 2^11 w_hi stays below 2^15.  0 for a
// non-finite maximum; clamped to [-100, 100], the range in which the kernels' power-of-two factors stay normal floats.
__host__ __device__ __forceinline__ int tc_f16_wexp(uint32_t maxbits) {
    const int E = (int)(maxbits >> 23);
    return E >= 255 ? 0 : min(max(E - 130, -100), 100);
}
__device__ __forceinline__ float tc_pow2(int k) { return __int_as_float((127 + k) << 23); }     // 2^k, -126 <= k <= 127
// K slot s (0..31) of a 32-channel block <-> channel of the block: the FP16 A fragment of thread t (t = lane % 4) takes K slots
// {2t, 2t+1, 2t+8, 2t+9} of each 16-slot half h, which this order maps to channels 8t + 4h + {0, 1, 2, 3} -- one 16-byte chunk
// of the raw tile row per half, read with one conflict-free 128-bit load.  The weights are packed in the same order.
__host__ __device__ __forceinline__ int tc_f16_channel(int s) {
    const int h = s >> 4, j = s & 15;
    return 8 * ((j & 7) >> 1) + 4 * h + 2 * (j >> 3) + (j & 1);
}

// whole tile `tile` of the plain, tap-group and kernel-row modes: sample, pixel origin, Co tile, parity class and its taps
template <int NT>
__device__ __forceinline__ void tc_whole_tile(const TcParams& p, int tile, TcTile& t) {
    int pix, r, cot = 0;
    p.d_ntiles.divmod(tile, r, pix);
    t.cls = 0;
    if (r) p.d_cotiles.divmod(r, t.cls, cot);
    int tx, ty, q2;
    p.d_tiles_x.divmod(pix, q2, tx);
    p.d_tiles_y.divmod(q2, t.n, ty);
    t.u0 = ty * p.th; t.v0 = tx * p.tw;
    t.co0 = cot * NT;
    t.tap0 = p.cls_tap0[t.cls]; t.ntaps = p.cls_ntaps[t.cls];
    t.valid = t.u0 < p.cls_Hu[t.cls] && t.v0 < p.cls_Wu[t.cls];                   // false: tile outside this (smaller) parity class
}

template <int NT, int MODE>
__device__ __forceinline__ TcTile tc_decode_tile(const TcParams& p, int tile) {
    TcTile t;
    t.slot = -1;
    if constexpr (MODE == TC_CORR) {
        // unit -> (halo block, tile x, tile y, plane, sample); co0 carries the halo block, cls the parity plane
        int r = tile / p.cnt;
        t.co0 = tile - r * p.cnt;
        int q = r / p.tiles_x;
        const int tx = r - q * p.tiles_x;
        r = q / p.tiles_y;
        const int ty = q - r * p.tiles_y;
        const int planes = p.cS * p.cS;
        t.n = r / planes;
        t.cls = r - t.n * planes;
        t.u0 = ty * p.th; t.v0 = tx * p.tw;
        t.tap0 = 0; t.ntaps = 1; t.k0 = 0;
        t.steps = p.cblocks;
        const int py = t.cls / p.cS, px = t.cls % p.cS;
        t.valid = t.u0 * p.cS + py < p.Ho && t.v0 * p.cS + px < p.Wo;
        return t;
    }
    if constexpr (MODE == TC_WGRAD) {
        // unit -> (K range, small-channel tile, big-channel tile, tap); u0 carries the first big channel, slot the unit itself
        int q = tile / p.wg_S;
        const int split = tile - q * p.wg_S;
        const int q2 = q / p.wg_ST;
        t.co0 = (q - q2 * p.wg_ST) * NT;
        t.tap0 = q2 / p.wg_BT;
        t.u0 = (q2 - t.tap0 * p.wg_BT) * 128;
        t.tap0 *= p.wg_TPT;                                        // first tap of the group
        t.n = 0; t.v0 = 0; t.cls = 0; t.ntaps = 1; t.slot = tile; t.valid = true;
        const int per = (p.wg_segs + p.wg_S - 1) / p.wg_S;
        t.k0 = min(p.wg_segs, split * per);
        t.steps = min(p.wg_segs, t.k0 + per) - t.k0;
        return t;
    }
    int seg = 0;
    if (p.split_z > 1 && tile >= p.split_first) {              // the K ranges of a split tile run side by side (shared A tiles in L2)
        t.slot = tile - p.split_first;
        int q;
        p.d_split_z.divmod(t.slot, q, seg);
        tile = p.split_first + q;
    }
    tc_whole_tile<NT>(p, tile, t);
    const int gsz = MODE == TC_GROUP ? 32 / p.gcs : 1;
    t.steps = MODE == TC_ROW ? p.rsteps : (MODE == TC_GROUP ? (t.ntaps + gsz - 1) / gsz : t.ntaps * p.cblocks);
    t.k0 = 0;
    if (t.slot >= 0) {
        const int per = (t.steps + p.split_z - 1) / p.split_z;
        t.k0 = min(t.steps, seg * per);
        t.steps = min(t.steps, t.k0 + per) - t.k0;
    }
    return t;
}

// Tap-group packing (Ci <= 16): the stage holds up to 32/CS dense boxes [128 pixels][CS floats] (one per kernel tap);
// row m of the K block = concatenation of its CS-channel slices, zero beyond the taps present.
template <int CS>
__device__ __forceinline__ void gather_taps(const unsigned char* base, int r0, int r1, int t, int nt, uint32_t* hi, uint32_t* lo) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const int k = 8 * (i >> 2) + t + 4 * ((i >> 1) & 1);
        const int r = (i & 1) ? r1 : r0;
        const int j = k / CS, c = k - j * CS;
        const float f = j < nt ? *reinterpret_cast<const float*>(base + (size_t)j * (128 * CS * 4) + (size_t)r * (CS * 4) + c * 4) : 0.f;
        split_store(f, hi[i], lo[i]);
    }
}

// Persistent kernel: gridDim.x CTAs (one per SM) walk the tile list with stride gridDim.x; the barrier ring runs straight
// through tile boundaries, so the producer loads the next tile's first stages while the MMA warpgroups finish the current one.
template <int NT, int MODE>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW, const float* __restrict__ bias,
               float* __restrict__ out, float* __restrict__ ws, const TcParams p) {
    constexpr bool F16 = tc_f16(NT, MODE);
    using G = TcGeo<NT, F16>;
    // MMA N: the correlation's halo block has cbw * cbh = 112 pixels (corr_tc_forward)
    constexpr int NM = MODE == TC_CORR ? 112 : NT;
    extern __shared__ __align__(1024) unsigned char smem[];
    float* stg = reinterpret_cast<float*>(smem + G::R * G::STAGE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + G::R * G::STAGE_BYTES + G::STG_BYTES);
    uint64_t* full = bars;                         // [R]  TMA bytes of the stage have landed
    uint64_t* done = bars + G::R;                  // [R]  MMAs of the step have retired: the stage is free

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // Programmatic dependent launch: let the next kernel of the stream be scheduled as soon as every CTA of this one is
    // running, so that its CTAs take over SMs the moment ours exit and run their prologue (barrier init) there; it blocks
    // in griddepcontrol.wait (below, before its first global access) until this grid has completed.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int gsz = MODE == TC_GROUP ? 32 / p.gcs : 1;   // taps per K block when packing

    if (tid == 0) {
        // done[s]: one arrival per MMA warp (8)
        for (int s = 0; s < G::R; s++) { mbar_init(&full[s], 1); mbar_init(&done[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");      // no-op unless launched with programmatic stream serialization

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 0 && lane == 0) {
            // ===== TMA producer (running counters instead of per-step divisions: this single thread's instruction chain
            // paces the whole pipeline) =====
            const int cblocks = p.cblocks, gcs = p.gcs;
            int s = 0; uint32_t ph = 1u;                // ph: parity to wait on done[s]
            for (int tile = blockIdx.x; tile < p.total; tile += gridDim.x) {
                const TcTile T = tc_decode_tile<NT, MODE>(p, tile);
                if (!T.valid) continue;
                const int cx0 = T.v0 * p.su, cy0 = T.u0 * p.sv;
                auto load_w = [&](unsigned char* st, uint64_t* bar, int c0, int blk) {
                    if constexpr (F16) {
                        // one box {32 halves, NT, 2 tiles: W_A | W_B} of K block (tap blk, channel block c0 / 32)
                        tma_load_4d(st + A_TILE_BYTES, &mapW, bar, 0, T.co0, 0, blk * cblocks + c0 / 32);
                    } else {
                        tma_load_4d(st + A_TILE_BYTES, &mapW, bar, c0, T.co0, blk, 0);
                        tma_load_4d(st + A_TILE_BYTES + G::B_TILE_BYTES, &mapW, bar, c0, T.co0, blk, 1);
                    }
                };
                if constexpr (MODE == TC_CORR) {
                    const int py = T.cls / p.cS, px = T.cls % p.cS;
                    const int ax = T.v0 * p.cS + px, ay = T.u0 * p.cS + py;
                    const int bx = (T.v0 - p.cR) * p.cS + px, by = (T.u0 - p.cR + T.co0 * p.cbh) * p.cS + py;
                    const uint32_t bbytes = (uint32_t)(p.cbw * p.cbh * 128);
#pragma unroll 1
                    for (int i = 0; i < T.steps; i++) {
                        mbar_wait(&done[s], ph);
                        unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                        mbar_expect_tx(&full[s], (uint32_t)A_TILE_BYTES + 2u * bbytes);
                        tma_load_4d(st, &mapA, &full[s], i * 32, ax, ay, T.n);
                        tma_load_4d(st + A_TILE_BYTES, &mapW, &full[s], i * 32, bx, by, T.n);
                        tma_load_4d(st + A_TILE_BYTES + G::B_TILE_BYTES, &mapW, &full[s], i * 32, bx, by, p.N + T.n);
                        if (++s == G::R) { s = 0; ph ^= 1u; }
                    }
                } else if constexpr (MODE == TC_WGRAD) {
                    // K segment = 32 consecutive output columns of one output row of one sample.  A: the tap's shifted window of
                    // the big map, 128 channel rows x 32 pixels (column-parity plane widx[tap], so that a strided convolution
                    // still reads consecutive floats); B: the same 32 pixels of the small map's hi and lo planes.
                    // (TMA needs the innermost coordinate on a 16-byte boundary: the big map is stored in 4 copies delayed by 0..3
                    // columns, widx[tap] >> 4 picks the copy that makes the tap's column shift a multiple of 4.)
                    int xs = T.k0 % p.wg_segs_x, r = T.k0 / p.wg_segs_x;
                    int oy = r % p.Ho, n = r / p.Ho;
                    const int tpt = p.wg_TPT, gbytes = p.wg_G * 128;
#pragma unroll 1
                    for (int i = 0; i < T.steps; i++) {
                        mbar_wait(&done[s], ph);
                        unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                        mbar_expect_tx(&full[s], (uint32_t)G::STAGE_BYTES);
                        for (int j = 0; j < tpt; j++) {
                            // a group past the last tap repeats tap 0 (its rows are never read back)
                            const int tap = T.tap0 + j < p.wg_taps ? T.tap0 + j : 0;
                            tma_load_4d(st + j * gbytes, &mapA, &full[s], xs * 32 + p.dx[tap], (oy * p.sv + p.dy[tap]) * p.wg_sx + (p.widx[tap] & 15),
                                        T.u0, (p.widx[tap] >> 4) * p.N + n);
                        }
                        tma_load_4d(st + A_TILE_BYTES, &mapW, &full[s], xs * 32, oy, T.co0, n);
                        tma_load_4d(st + A_TILE_BYTES + G::B_TILE_BYTES, &mapW, &full[s], xs * 32, oy, T.co0, p.N + n);
                        if (++xs == p.wg_segs_x) { xs = 0; if (++oy == p.Ho) { oy = 0; ++n; } }
                        if (++s == G::R) { s = 0; ph ^= 1u; }
                    }
                } else if constexpr (MODE == TC_ROW) {
                    // one box per step: {32 floats of the kernel-row run, tw output pixels (stride su pixels), th rows}
                    int r = 0, kb = 0;
#pragma unroll 1
                    for (int i = 0; i < T.steps; i++) {
                        mbar_wait(&done[s], ph);
                        unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                        mbar_expect_tx(&full[s], (uint32_t)G::STAGE_BYTES);
                        tma_load_4d(st, &mapA, &full[s], kb * 32, T.v0, cy0 + p.dy[r * p.rkw], T.n);
                        load_w(st, &full[s], 0, i);
                        if (++kb == p.rblocks) { kb = 0; ++r; }
                        if (++s == G::R) { s = 0; ph ^= 1u; }
                    }
                } else if constexpr (MODE == TC_GROUP) {
                    // several taps share one 32-wide K block: one small box {gcs channels, tw, th} per tap
                    const int box_bytes = 128 * gcs * 4;
                    for (int i = 0, t0 = 0; i < T.steps; i++, t0 += gsz) {
                        mbar_wait(&done[s], ph);
                        unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                        const int nt = min(gsz, T.ntaps - t0);
                        mbar_expect_tx(&full[s], (uint32_t)(nt * box_bytes + 2 * G::B_TILE_BYTES));
                        for (int j = 0; j < nt; j++) {
                            const int t = T.tap0 + t0 + j;
                            tma_load_4d(st + j * box_bytes, &mapA, &full[s], 0, cx0 + p.dx[t], cy0 + p.dy[t], T.n);
                        }
                        load_w(st, &full[s], 0, i);
                        if (++s == G::R) { s = 0; ph ^= 1u; }
                    }
                } else {
                    int t = T.tap0 + T.k0 / cblocks, cb = T.k0 % cblocks;
                    int cx = cx0 + p.dx[t], cy = cy0 + p.dy[t], wi = p.widx[t];
#pragma unroll 1
                    for (int i = 0; i < T.steps; i++) {
                        mbar_wait(&done[s], ph);
                        unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                        mbar_expect_tx(&full[s], (uint32_t)G::STAGE_BYTES);
                        tma_load_4d(st, &mapA, &full[s], cb * 32, cx, cy, T.n);
                        load_w(st, &full[s], cb * 32, wi);
                        if (++cb == cblocks && i + 1 < T.steps) { cb = 0; ++t; cx = cx0 + p.dx[t]; cy = cy0 + p.dy[t]; wi = p.widx[t]; }
                        if (++s == G::R) { s = 0; ph ^= 1u; }
                    }
                }
            }
        }
    } else {
        // ===== MMA warpgroups: raw FP32 tile (smem) -> a_hi / a_lo fragments -> wgmma -> FP32 registers -> epilogue =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
        const int ct = tid - 128;                  // 0..255
        const int wg = ct >> 7, wi = (ct >> 5) & 3;
        const int g = lane >> 2, t = lane & 3;
        const int r0 = 64 * wg + 16 * wi + g, r1 = r0 + 8;      // tile rows of this thread's fragment elements
        const int m = ct & 127, hf = ct >> 7;      // epilogue: pixel row m, column half hf
        constexpr int NH = NT / 2;
        const int tws = __ffs(p.tw) - 1;           // epilogue: log2 of the tile width (a power of two)
        // FP16 route: the layer's weight exponent f and the range of the row exponents e that keeps 2^-e, 2^(11-e) and
        // 2^(e+f-11) normal floats
        int fw = 0, elo = 0, ehi = 0;
        if constexpr (F16) {
            fw = tc_f16_wexp(*p.wmax);
            elo = max(-116, -115 - fw); ehi = min(126, 138 - fw);
        }
        int s = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < p.total; tile += gridDim.x) {
            const TcTile T = tc_decode_tile<NT, MODE>(p, tile);
            if (!T.valid) continue;
            float acc[NH];
#pragma unroll
            for (int j = 0; j < NH; j++) acc[j] = 0.f;
            float c[G::WIDE ? NT : NM / 2];        // chunk accumulator (WIDE: [a_hi*w_hi | a_hi*w_lo])
            float cx[G::WIDE ? NH : 1];            // WIDE: a_lo*w_hi, an MMA shape of its own
            int in_chunk = 0;
#pragma unroll 1
            for (int i = 0; i < T.steps; i++) {
                mbar_wait(&full[s], ph);
                const unsigned char* st = smem + (size_t)s * G::STAGE_BYTES;
                uint32_t ah[16], al[16];
                float rs[2];                       // FP16 route: 2^(e+f-11) of rows r0, r1
                if constexpr (F16) {
                    // per row: e from the largest |a| of the row's 32 channels (8 per quad lane), so that |a| 2^-e < 2^15;
                    // a 2^-e = hi + lo'', both FP16 (a_hi / a_lo'' in the fragments of the two 16-slot halves).  The
                    // subtraction is exact; lo'' meets W_A = 2^11 w_hi, so no third weight tile is needed (DESIGN.md section 3)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int r = e ? r1 : r0;
                        const float4 v0 = *reinterpret_cast<const float4*>(st + r * 128 + (((2 * t) ^ (r & 7)) << 4));
                        const float4 v1 = *reinterpret_cast<const float4*>(st + r * 128 + (((2 * t + 1) ^ (r & 7)) << 4));
                        float mx = fmaxf(fmaxf(fmaxf(fabsf(v0.x), fabsf(v0.y)), fmaxf(fabsf(v0.z), fabsf(v0.w))),
                                         fmaxf(fmaxf(fabsf(v1.x), fabsf(v1.y)), fmaxf(fabsf(v1.z), fabsf(v1.w))));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                        const int E = (int)(__float_as_uint(mx) >> 23);
                        const int ex = E == 255 ? 0 : min(max(E - 141, elo), ehi);          // E = 255: no finite max
                        const float up = tc_pow2(-ex);
                        rs[e] = tc_pow2(ex + fw - 11);
                        const float4 vh[2] = {v0, v1};
#pragma unroll
                        for (int hh = 0; hh < 2; hh++) {
                            const float x[4] = {vh[hh].x * up, vh[hh].y * up, vh[hh].z * up, vh[hh].w * up};
#pragma unroll
                            for (int q = 0; q < 2; q++) {
                                const __half2 h = __floats2half2_rn(x[2 * q], x[2 * q + 1]);
                                const float2 hf = __half22float2(h);
                                const __half2 l = __floats2half2_rn(__fsub_rn(x[2 * q], hf.x), __fsub_rn(x[2 * q + 1], hf.y));
                                ah[4 * hh + 2 * q + e] = *reinterpret_cast<const uint32_t*>(&h);
                                al[4 * hh + 2 * q + e] = *reinterpret_cast<const uint32_t*>(&l);
                            }
                        }
                    }
                } else if constexpr (MODE == TC_GROUP) {
                    const int nt = min(gsz, T.ntaps - i * gsz);
                    if (p.gcs == 4) gather_taps<4>(st, r0, r1, t, nt, ah, al);
                    else if (p.gcs == 8) gather_taps<8>(st, r0, r1, t, nt, ah, al);
                    else if (p.gcs == 12) gather_taps<12>(st, r0, r1, t, nt, ah, al);
                    else gather_taps<16>(st, r0, r1, t, nt, ah, al);
                } else if constexpr (MODE == TC_ROW) {
                    // row mode: taps that fall outside the image row (and the K padding) hold whatever follows in memory; the
                    // padding channels of the pixels inside the row meet zero weights (fn2.h: they must be finite)
                    const int kb32 = (i % p.rblocks) * 32;
                    int klo[2], khi[2];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int x0 = (T.v0 + (e ? r1 : r0) % p.tw) * p.su - p.rpad;     // input column of tap 0
                        klo[e] = max(0, -x0) * p.rcs - kb32;
                        khi[e] = min(p.rkw, p.rW - x0) * p.rcs - kb32;
                    }
#pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const int e = q & 1, chunk = 2 * (q >> 2) + ((q >> 1) & 1);
                        const bool keep = 4 * chunk >= klo[e] && 4 * chunk < khi[e];
                        const float f = raw_at(st, e ? r1 : r0, chunk, t);
                        split_store(keep ? f : 0.f, ah[q], al[q]);
                    }
                } else {
#pragma unroll
                    for (int q = 0; q < 16; q++)
                        split_store<MODE == TC_CORR>(raw_at(st, (q & 1) ? r1 : r0, 2 * (q >> 2) + ((q >> 1) & 1), t), ah[q], al[q]);
                }
                const uint32_t bh = su32(st + A_TILE_BYTES);
                const uint64_t dbh0 = make_desc_sw128(bh), dbl0 = make_desc_sw128(bh + G::B_TILE_BYTES);
                const bool chunk_end = (in_chunk == p.kd - 1) || (i == T.steps - 1);
#pragma unroll
                for (int j = 0; j < (int)(sizeof(c) / sizeof(float)); j++) reg_fence(c[j]);
#pragma unroll
                for (int j = 0; j < (int)(sizeof(cx) / sizeof(float)); j++) reg_fence(cx[j]);
                wgmma_fence();
                if constexpr (F16) {
                    // per 16-slot half: a_lo'' * W_A and a_hi * W_B (2^-11 smaller) first, then a_hi * W_A
                    const uint64_t dA = make_desc_sw64(bh), dB = make_desc_sw64(bh + G::B_TILE_BYTES);
                    const int acc0 = in_chunk != 0;
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        WgmmaF16<NT>::mma(c, al + 4 * hh, dA + (uint64_t)(2 * hh), acc0 | hh);
                        WgmmaF16<NT>::mma(c, ah + 4 * hh, dB + (uint64_t)(2 * hh), 1);
                    }
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) WgmmaF16<NT>::mma(c, ah + 4 * hh, dA + (uint64_t)(2 * hh), 1);
                } else {
                    const int acc0 = in_chunk != 0;
#pragma unroll
                    for (int kk = 0; kk < 4; kk++) {
                        // +2 in the start-address field = +32 bytes = the next 8 TF32 columns of the swizzled tile
                        if constexpr (G::WIDE) {
                            Wgmma<2 * NT>::mma(c, ah + 4 * kk, dbh0 + (uint64_t)(2 * kk), acc0 | kk);
                            Wgmma<NT>::mma(cx, al + 4 * kk, dbh0 + (uint64_t)(2 * kk), acc0 | kk);
                        } else {
                            Wgmma<NM>::mma(c, al + 4 * kk, dbh0 + (uint64_t)(2 * kk), acc0 | kk);
                            Wgmma<NM>::mma(c, ah + 4 * kk, dbl0 + (uint64_t)(2 * kk), 1);
                        }
                    }
                    if constexpr (!G::WIDE) {
#pragma unroll
                        for (int kk = 0; kk < 4; kk++) Wgmma<NM>::mma(c, ah + 4 * kk, dbh0 + (uint64_t)(2 * kk), 1);
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
#pragma unroll
                for (int j = 0; j < (int)(sizeof(c) / sizeof(float)); j++) reg_fence(c[j]);
#pragma unroll
                for (int j = 0; j < (int)(sizeof(cx) / sizeof(float)); j++) reg_fence(cx[j]);
                // this warp's MMAs of the step have retired: release the stage
                __syncwarp();
                if (lane == 0) mbar_arrive(&done[s]);
                if (chunk_end) {
                    // mean truncation loss of the a_hi*w_hi chain of this chunk
                    const float comp = G::TRUNC_LOSS * (float)(G::MMAS_PER_STEP * (in_chunk + 1));
                    if constexpr (F16) {
                        // the chunk holds 2^(11-e-f) sum a w (one K step: kd == 1); scaling back is exact
#pragma unroll
                        for (int j = 0; j < NM / 2; j++) acc[j] = fmaf(fmaf(c[j], comp, c[j]), rs[(j >> 1) & 1], acc[j]);
                    } else if constexpr (G::WIDE) {
#pragma unroll
                        for (int j = 0; j < NH; j++) acc[j] += fmaf(c[j], comp, c[j]) + (c[NH + j] + cx[j]);
                    } else {
#pragma unroll
                        for (int j = 0; j < NM / 2; j++) acc[j] += fmaf(c[j], comp, c[j]);
                    }
                    in_chunk = 0;
                } else {
                    ++in_chunk;
                }
                if (++s == G::R) { s = 0; ph ^= 1u; }
            }
            // fragments -> staging buffer [128 pixels][STG]; bar.sync 1 = the 256 MMA threads
            asm volatile("bar.sync 1, 256;" ::: "memory");             // the previous tile's epilogue has read the buffer
#pragma unroll
            for (int j = 0; j < NH; j += 2) {
                const int row = (j & 2) ? r1 : r0, col = 8 * (j >> 2) + 2 * t;
                if (MODE != TC_CORR || col < NM) *reinterpret_cast<float2*>(stg + row * G::STG + col) = make_float2(acc[j], acc[j + 1]);
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // epilogue
            if constexpr (MODE == TC_CORR) {
                // A halo block = cbh full halo rows (cbw = tw + 2R pixels each): for every tile pixel it holds cbh
                // displacement rows dy with all D = 2R+1 values of dx, i.e. runs of D consecutive output channels.  The
                // block is written from the staging buffer with lanes = channels: one coalesced run per (pixel, dy).
                const int py = T.cls / p.cS, px = T.cls % p.cS;
                const int cw = ct >> 5;
                const bool lane_on = lane < p.cD;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    // warp cw stores tile rows qy = cw, cw+8: 8 pixels x 2 displacement rows each, lanes = dx
                    const int dy_base = T.co0 * 4 + h * 2 - p.cR;
#pragma unroll
                    for (int k = 0; k < 2; k++) {
                        const int qy = cw + 8 * k;
                        const int y = (T.u0 + qy) * p.cS + py;
                        const int dy0 = dy_base - qy, dy1 = dy0 + 1;
                        const bool ok0 = lane_on && y < p.Ho && dy0 >= -p.cR && dy0 <= p.cR;
                        const bool ok1 = lane_on && y < p.Ho && dy1 >= -p.cR && dy1 <= p.cR;
                        float* o = out + T.n * p.out_sn + (long long)y * p.out_sh + (long long)(T.v0 * p.cS + px) * p.out_sw + lane;
                        const float* tr = stg + (qy * 8) * G::STG + h * 56 + lane;
                        const int c0 = (dy0 + p.cR) * p.cD, c1 = (dy1 + p.cR) * p.cD;
#pragma unroll
                        for (int qx = 0; qx < 8; qx++) {
                            const bool inx = (T.v0 + qx) * p.cS + px < p.Wo;
                            const float v0 = lane_on ? tr[qx * G::STG + qx] * p.cscale : 0.f, v1 = lane_on ? tr[qx * G::STG + 28 + qx] * p.cscale : 0.f;
                            if (ok0 && inx) o[(long long)qx * p.cS * p.out_sw + c0] = v0;
                            if (ok1 && inx) o[(long long)qx * p.cS * p.out_sw + c1] = v1;
                        }
                    }
                }
                continue;
            }
            float* srow = stg + m * G::STG + hf * NH;                  // this thread's half row
            if constexpr (MODE == TC_WGRAD) {
                // raw partial sums of this unit, [unit][128 big channels][NT small channels]; conv_tc_wgrad's reduction sums the
                // K ranges in a fixed order and scatters into the Caffe weight layout
                float* o = ws + ((long long)T.slot * 128 + m) * NT + hf * NH;
#pragma unroll
                for (int j = 0; j < NH; j += 4) *reinterpret_cast<float4*>(o + j) = *reinterpret_cast<const float4*>(srow + j);
                continue;
            }
            // one float4 of the tile per thread and pass, consecutive threads along a pixel's NT channels: every warp stores
            // whole pixels (full 32-byte sectors, where a thread per pixel left half of each sector of a store to the next
            // one), and a thread keeps its 4 channels -- and their bias -- in every pass
            constexpr int CG = NT / 4, PX = 256 / CG;                  // float4 groups per pixel, pixels per pass
            const int cg = ct % CG;
            float bv[4] = {0.f, 0.f, 0.f, 0.f};
            if (T.slot < 0 && p.has_bias) {
#pragma unroll
                for (int e = 0; e < 4; e++) bv[e] = __ldg(bias + T.co0 + 4 * cg + e);
            }
#pragma unroll
            for (int k = 0; k < 128 / PX; k++) {
                const int px = k * PX + ct / CG;                       // tile pixel
                const int u = T.u0 + (px >> tws), v = T.v0 + (px & (p.tw - 1));
                if (u >= p.cls_Hu[T.cls] || v >= p.cls_Wu[T.cls]) continue;
                const float4 a = *reinterpret_cast<const float4*>(stg + px * G::STG + 4 * cg);
                if (T.slot >= 0) {
                    // K split: raw partial sums of this K range, [slot][128 pixels][NT]
                    *reinterpret_cast<float4*>(ws + ((long long)T.slot * 128 + px) * NT + 4 * cg) = a;
                    continue;
                }
                const int oy = u * p.ou + p.cls_oy0[T.cls], ox = v * p.ov + p.cls_ox0[T.cls];
                float r[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    if (p.has_bias) r[e] += bv[e];
                    if (p.relu) r[e] = r[e] > 0 ? r[e] : r[e] * p.slope;
                }
                *reinterpret_cast<float4*>(out + T.n * p.out_sn + (long long)oy * p.out_sh + (long long)ox * p.out_sw + T.co0 + 4 * cg) =
                    make_float4(r[0], r[1], r[2], r[3]);
            }
        }
    }
    __syncthreads();
}

__global__ void tc_pack_kernel(const float* __restrict__ w, float* __restrict__ wp, int Ci, int Co, int kh, int kw, int cip, int deconv) {
    const long long per = (long long)kh * kw * Co * cip;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < per; idx += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(idx % cip);
        long long r_ = idx / cip;
        const int co = (int)(r_ % Co);
        const int t = (int)(r_ / Co);
        const int r = t / kw, s = t % kw;
        float v = 0.f;
        if (ci < Ci) v = deconv ? w[(((long long)ci * Co + co) * kh + r) * kw + s] : w[(((long long)co * Ci + ci) * kh + r) * kw + s];
        store_tf32_split(wp, per, idx, v);
    }
}

// FP16 route: bits of the layer's largest |w| into *out (zeroed before; the bits of non-negative floats order like their values,
// and a NaN's lie above infinity's)
__global__ void tc_absmax_kernel(const float* __restrict__ w, long long n, uint32_t* __restrict__ out) {
    uint32_t m = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = max(m, __float_as_uint(w[i]) & 0x7fffffffu);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// FP16 route: [tap][channel block][W_A | W_B | W_C][Co][32 K slots] halves (K slot order tc_f16_channel).  With f from the
// layer's largest |w| (*wmax) and w_hi = fp16(w 2^-f): W_A = 2^11 w_hi, W_B = fp16(2^11 (w 2^-f - w_hi)), W_C = w_hi (all but
// the rounding of W_B exact).  The forward reads only W_A and W_B (conv_tc_kernel multiplies the activations' low half by W_A);
// W_C is still written because the packed format and its size are pinned, so that it can be dropped in one change with them.
__global__ void tc_pack_f16_kernel(const float* __restrict__ w, __half* __restrict__ wp, int Ci, int Co, int kh, int kw, int cblocks,
                                   int deconv, const uint32_t* __restrict__ wmax) {
    const long long per = (long long)kh * kw * cblocks * 3 * Co * 32;
    const float down = tc_pow2(-tc_f16_wexp(*wmax));
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < per; idx += (long long)gridDim.x * blockDim.x) {
        const int sl = (int)(idx % 32);
        long long r_ = idx / 32;
        const int co = (int)(r_ % Co);
        r_ /= Co;
        const int part = (int)(r_ % 3), blk = (int)(r_ / 3);
        const int t = blk / cblocks, ci = (blk % cblocks) * 32 + tc_f16_channel(sl);
        const int r = t / kw, s = t % kw;
        float v = 0.f;
        if (ci < Ci) v = deconv ? w[(((long long)ci * Co + co) * kh + r) * kw + s] : w[(((long long)co * Ci + ci) * kh + r) * kw + s];
        const float x = v * down;
        const __half hi = __float2half_rn(x);
        const float hf = __half2float(hi);
        wp[idx] = part == 0 ? __float2half_rn(2048.f * hf) : (part == 1 ? __float2half_rn((x - hf) * 2048.f) : hi);
    }
}

// group-packed weights for Ci <= 16: [hi|lo][group][Co][32], K index = j*CS + ci for tap = group*(32/CS) + j
__global__ void tc_pack_group_kernel(const float* __restrict__ w, float* __restrict__ wp, int Ci, int Co, int kh, int kw, int cs, int ngroups) {
    const long long per = (long long)ngroups * Co * 32;
    const int gs = 32 / cs;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < per; idx += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(idx % 32);
        long long r_ = idx / 32;
        const int co = (int)(r_ % Co);
        const int g = (int)(r_ / Co);
        const int j = k / cs, ci = k % cs;
        const int t = g * gs + j;
        float v = 0.f;
        if (j < gs && t < kh * kw && ci < Ci) v = w[(((long long)co * Ci + ci) * kh + t / kw) * kw + t % kw];
        store_tf32_split(wp, per, idx, v);
    }
}

// row-packed weights for Ci <= 16: [hi|lo][r*rblocks + kb][Co][32], K index kb*32 + k = s*cs + ci of kernel row r
__global__ void tc_pack_row_kernel(const float* __restrict__ w, float* __restrict__ wp, int Ci, int Co, int kh, int kw, int cs, int rblocks) {
    const long long per = (long long)kh * rblocks * Co * 32;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < per; idx += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(idx % 32);
        long long r_ = idx / 32;
        const int co = (int)(r_ % Co);
        const int blk = (int)(r_ / Co);
        const int r = blk / rblocks, kk = (blk % rblocks) * 32 + k;
        const int sx = kk / cs, ci = kk % cs;
        float v = 0.f;
        if (sx < kw && ci < Ci) v = w[(((long long)co * Ci + ci) * kh + r) * kw + sx];
        store_tf32_split(wp, per, idx, v);
    }
}

// fix-up of a K-split layer: fixed-order sum of the split_z partial tiles of every split tile + bias + ReLU, one thread per
// (tile row, 4 channels)
template <int NT>
__global__ void tc_split_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ bias, float* __restrict__ out, const TcParams p) {
    const int nsplit = p.ntotal - p.split_first;
    const long long per = (long long)nsplit * 128 * (NT / 4);
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < per; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % (NT / 4)) * 4;
        const int m = (int)((idx / (NT / 4)) % 128);
        const int t = (int)(idx / ((NT / 4) * 128));
        TcTile T;
        tc_whole_tile<NT>(p, p.split_first + t, T);
        const int u = T.u0 + m / p.tw, v = T.v0 + m % p.tw;
        if (!T.valid || u >= p.cls_Hu[T.cls] || v >= p.cls_Wu[T.cls]) continue;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int z = 0; z < p.split_z; z++) {
            const float4 x = *reinterpret_cast<const float4*>(ws + (((long long)t * p.split_z + z) * 128 + m) * NT + c);
            a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
        }
        const int co = T.co0 + c;
        if (p.has_bias) { a.x += __ldg(bias + co); a.y += __ldg(bias + co + 1); a.z += __ldg(bias + co + 2); a.w += __ldg(bias + co + 3); }
        if (p.relu) {
            a.x = a.x > 0 ? a.x : a.x * p.slope; a.y = a.y > 0 ? a.y : a.y * p.slope;
            a.z = a.z > 0 ? a.z : a.z * p.slope; a.w = a.w > 0 ? a.w : a.w * p.slope;
        }
        const int oy = u * p.ou + p.cls_oy0[T.cls], ox = v * p.ov + p.cls_ox0[T.cls];
        *reinterpret_cast<float4*>(out + T.n * p.out_sn + (long long)oy * p.out_sh + (long long)ox * p.out_sw + co) = a;
    }
}

// The driver's cuTensorMapEncodeTiled, looked up once; nullptr if the driver does not provide it.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tc_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

// f(std::integral_constant<int, NT>()) for the tile width nt (128, 64, 32, else 16)
template <class F>
int tc_with_nt(int nt, const F& f) {
    if (nt == 128) return f(std::integral_constant<int, 128>());
    if (nt == 64) return f(std::integral_constant<int, 64>());
    if (nt == 32) return f(std::integral_constant<int, 32>());
    return f(std::integral_constant<int, 16>());
}

// conv_tc_kernel<nt, MODE> over p.total tile units; the forward modes with programmatic stream serialization, the weight gradient
// without
template <int MODE>
int tc_run(int nt, cudaStream_t st, const CUtensorMap& mapA, const CUtensorMap& mapW, const float* bias, float* out, float* ws,
           const TcParams& p) {
    return tc_with_nt(nt, [&](auto c) {
        constexpr int NT = decltype(c)::value;
        return tc_launch<conv_tc_kernel<NT, MODE>>(p.total, TC_THREADS, TcGeo<NT, tc_f16(NT, MODE)>::SMEM, MODE != TC_WGRAD, st,
                                                   mapA, mapW, bias, out, ws, p);
    });
}

}  // namespace

int tc_tensor_map(CUtensorMap* map, const char* what, CUtensorMapDataType dtype, const void* base, const cuuint64_t* dims,
                  const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* es, CUtensorMapSwizzle swizzle,
                  CUtensorMapL2promotion l2) {
    EncodeTiledFn enc = tc_encode_fn();
    if (!enc) { set_error("%s tensor map: cuTensorMapEncodeTiled unavailable", what); return FN2_ERR_CUDA; }
    const CUresult r = enc(map, dtype, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("%s tensor map failed (%d)", what, (int)r); return FN2_ERR_CUDA; }
    return FN2_OK;
}

// output channels per tile (MMA N) of a layer with `co` output channels
static int tc_nt(int co) { return (co % 128 == 0) ? 128 : (co % 64 == 0 ? 64 : (co % 32 == 0 ? 32 : 16)); }
// K steps per accumulation chunk: NT == 128 chains the cross terms into the chunk accumulator too, so its chunks are one step
static int tc_chunk_steps(int NT) { return NT == 128 ? 1 : 4; }

// The per-tap engine's packed weights of a layer read through an input of pixel stride ci_stride: its route and layout.
//   TF32, plain K blocks:  [hi|lo][tap][Co][cip]                   blocks = taps, width = cip = 32 * cblocks floats
//   TF32, tap groups:      [hi|lo][group][Co][32]                  K index j*cs + ci for tap group*(32/cs) + j
//   TF32, kernel rows:     [hi|lo][r*rblocks + kb][Co][32]         K index kb*32 + k = s*cs + ci of kernel row r
//   FP16:                  [tap*cblocks + cb][W_A|W_B|W_C][Co][32 halves] (tc_pack_f16_kernel), then 4 floats holding the bits
//                          of the largest |w| (tc_absmax_kernel).  The forward reads W_A and W_B only; W_C is no longer read
//                          by any kernel and stays packed because the packed format and its size are pinned
// Small-Ci packing (plain convolutions with at most 16 input channels): tap groups (several taps share a 32-wide K block, one small
// TMA box per tap), or kernel rows where they take no more K blocks (needs a dense input whose pixel stride equals the padded
// channel count, and a guard band around the tensor because the row runs of the edge pixels reach a little outside it).  The
// NT = 128 layers in plain K-block mode run on FP16 operands (three FP16 products per K step from two weight tiles, with a
// power-of-two scale per pixel row and per layer), every other layer on TF32 (3xTF32).
struct TcWeights {
    int mode;                 // TC_PLAIN, TC_GROUP or TC_ROW
    bool f16;                 // FP16 operands (three tiles per K block, of which the forward reads two), else TF32 hi and lo tiles
    int cs, rblocks;          // small-Ci packing: channels per tap padded to a multiple of 4, K blocks per kernel row
    int blocks, width, tiles; // K blocks, elements per output channel of a block, tiles per block
    size_t tile_floats;       // floats of the tiles
    size_t floats;            // all floats; 0 for a layer without whole 16-channel output tiles
};
static TcWeights tc_weights(const fn2_conv_desc* d, int ci_stride) {
    TcWeights w = {};
    if (d->co % 16) return w;
    const int taps = d->kh * d->kw, cblocks = (d->ci + 31) / 32;
    w.width = 32; w.tiles = 2;
    if (!d->deconv && d->ci <= 16 && taps >= 2) {
        w.cs = (d->ci + 3) / 4 * 4;
        const int gs = 32 / w.cs, ngroups = (taps + gs - 1) / gs;
        w.rblocks = (d->kw * w.cs + 31) / 32;
        w.mode = d->input_guard_bytes >= 512 && ci_stride == w.cs && d->kh * w.rblocks <= ngroups ? TC_ROW : TC_GROUP;
        w.blocks = w.mode == TC_ROW ? d->kh * w.rblocks : ngroups;
    } else if (tc_nt(d->co) == 128) {
        w.f16 = true; w.blocks = taps * cblocks; w.tiles = 3;
    } else {
        w.blocks = taps; w.width = 32 * cblocks;
    }
    w.tile_floats = (size_t)w.blocks * d->co * w.width * w.tiles / (w.f16 ? 2 : 1);
    w.floats = w.tile_floats + (w.f16 ? 4 : 0);
    return w;
}

// K split of a layer with `tiles` tile units of `steps` K steps each (the fewest of any parity class): returns z (1 = unsplit)
// and the first split tile.
//  * Tile lists that cannot fill the GPU (the 7x16 .. 14x32 maps of conv5/conv6/deconv5 with K = 9 * 1024) split every tile.
//  * Otherwise the tiles of the last, partial wave are split so that they spread over all SMs (448 tiles on 132 SMs:
//    3 + 52/132 rounds instead of 4).
static int tc_split_plan(long long tiles, int steps, int NT, int* first) {
    const int nsm = num_sms();
    *first = 0;
    if (tiles * 2 <= nsm && steps >= 32) {
        const int z = min(min((int)(nsm / tiles), steps / 16), 8);
        if (z >= 2) return z;
    }
    *first = (int)tiles;
    if (steps < 16) return 1;                       // (tiles <= nsm: everything is "tail" -- 112 tiles become 560 fifths on 132 SMs)
    const long long full = tiles / nsm * nsm, r = tiles - full;
    if (r == 0) return 1;
    // cost model in units of one tile's time: rounds of whole tiles + rounds of 1/z tiles + the fix-up kernel reading r*z
    // partial tiles (128 x NT floats each at ~3 TB/s; a tile takes ~1400 cycles per K step at 1.9 GHz)
    const double tile_s = steps * 1400.0 / 1.9e9, part_s = 128.0 * NT * 4 / 3e12 + 2e-9;
    const double now = (double)((tiles + nsm - 1) / nsm);
    double best = now * 0.94;
    int bz = 1;
    for (int z = 2; z <= min(8, steps / 8); z++) {
        const double then = (double)(full / nsm) + (double)((r * z + nsm - 1) / nsm) / z + (r * z * part_s + 4e-6) / tile_s;
        if (then < best) { best = then; bz = z; }
    }
    if (bz < 2) return 1;
    *first = (int)full;
    return bz;
}

// layer shapes the engine takes: whole 16-channel output tiles, at most 49 taps, convolution stride <= 2, deconvolution
// stride 1 or 2 (at most 4 parity classes)
static bool tc_takes(const fn2_conv_desc* d) {
    if (d->co % 16 || d->kh * d->kw > 49 || d->stride_h > 2 || d->stride_w > 2) return false;
    return !d->deconv || d->stride_h == d->stride_w;
}

// The engine's plan of one layer: every TcParams field of a forward launch except the output view, and the packed weights.
struct TcPlan {
    TcParams p;
    TcWeights w;
    int NT, steps;                                // output channels per tile, K steps per tile (the fewest of any parity class)
};
// W: input width (kernel-row packing), ci_stride: input pixel stride, ws_floats: workspace available for a K split (a K split
// that does not fit runs unsplit).  Returns false for a layer the engine does not take, including a deconvolution with a
// parity class that no tap reaches.
static bool tc_plan(const fn2_conv_desc* d, int N, int W, int Ho, int Wo, int ci_stride, size_t ws_floats, TcPlan* pl) {
    if (!tc_takes(d)) return false;
    ConvTaps tp;
    conv_taps(d, Ho, Wo, &tp);
    TcParams* p = &pl->p;
    const TcWeights& w = pl->w = tc_weights(d, ci_stride);
    memset(p, 0, sizeof(*p));
    const int NT = pl->NT = tc_nt(d->co);
    p->N = N; p->cblocks = (d->ci + 31) / 32;
    p->Ho = Ho; p->Wo = Wo;
    p->relu = d->relu; p->has_bias = d->has_bias; p->slope = d->negative_slope;
    // the kernel adds back the mean truncation loss of each chunk: TRUNC_LOSS_PER_MMA per a_hi*w_hi MMA chained into the
    // chunk accumulator (4 per step; with NT == 128 the 8 cross-term MMAs of a step precede them while it is still small; the
    // FP16 route: TRUNC_LOSS_PER_MMA_F16 per a_hi*W_A MMA, 2 per step after 4 cross-term MMAs, and its row scale needs kd == 1)
    p->kd = tc_chunk_steps(NT);
    p->gcs = w.mode == TC_GROUP ? w.cs : 0;
    p->rowmode = w.mode == TC_ROW; p->rcs = w.cs; p->rblocks = w.rblocks; p->rsteps = d->kh * w.rblocks;
    p->rkw = d->kw; p->rpad = d->pad_w; p->rW = W;
    // A box element strides: the convolution stride (x, y); a deconvolution's classes are stride-1 convolutions
    p->su = d->deconv ? 1 : d->stride_w; p->sv = d->deconv ? 1 : d->stride_h;
    p->ou = tp.ou; p->ov = tp.ov; p->ncls = tp.ncls;
    int steps = 1 << 30, Wmax = 0, Hmax = 0;
    for (int c = 0; c < tp.ncls; c++) {
        if (!tp.ntaps[c]) return false;
        p->cls_Hu[c] = tp.Hu[c]; p->cls_Wu[c] = tp.Wu[c]; p->cls_oy0[c] = tp.oy0[c]; p->cls_ox0[c] = tp.ox0[c];
        p->cls_tap0[c] = tp.tap0[c]; p->cls_ntaps[c] = tp.ntaps[c];
        steps = min(steps, tp.ntaps[c] * p->cblocks);
        Wmax = max(Wmax, tp.Wu[c]); Hmax = max(Hmax, tp.Hu[c]);
    }
    memcpy(p->dy, tp.dy, sizeof(p->dy)); memcpy(p->dx, tp.dx, sizeof(p->dx)); memcpy(p->widx, tp.widx, sizeof(p->widx));
    if (w.mode) steps = w.blocks;                 // small-Ci packing: one K step per tap group or kernel-row block
    pl->steps = steps;
    // tile shape: widest power of two covering the (largest) row, 128 pixels per tile
    int tw = 8;
    while (tw < Wmax && tw < 128) tw *= 2;
    p->tw = tw; p->th = 128 / tw;
    p->tiles_x = (Wmax + p->tw - 1) / p->tw; p->tiles_y = (Hmax + p->th - 1) / p->th;
    p->ntiles = N * p->tiles_x * p->tiles_y;
    p->cotiles = d->co / NT;
    p->ntotal = p->ntiles * p->cotiles * p->ncls;
    int first = p->ntotal, z = 1;
    if (!w.mode) z = tc_split_plan(p->ntotal, steps, NT, &first);             // small-Ci packing modes do not split
    if (z > 1 && ws_floats < (size_t)(p->ntotal - first) * z * 128 * NT) { z = 1; first = p->ntotal; }
    p->split_first = first; p->split_z = z;
    p->total = first + (p->ntotal - first) * z;
    p->d_ntiles.init(p->ntiles); p->d_cotiles.init(p->cotiles); p->d_tiles_x.init(p->tiles_x); p->d_tiles_y.init(p->tiles_y);
    p->d_split_z.init(z);
    return true;
}

// The partial tiles of a K split are written as float4: a caller's workspace may start anywhere 4-byte aligned, and the 4 floats
// of slack on top of the partials are the room to move it to a 16-byte boundary.
constexpr size_t TC_WS_SLACK = 4;

// ---------------------------------------------------------------------------------------------------------------------
// The tensor-core convolution engines behind fn2_conv.cu: eligibility, packed weights, plan, workspace and forward of a layer.
// The taps-on-N engine (fn2_conv_tn.cu) owns the layers it takes, the per-tap engine every other layer.
// ---------------------------------------------------------------------------------------------------------------------
int conv_tn_applicable(const fn2_conv_desc* d);
size_t conv_tn_packed_floats(const fn2_conv_desc* d);
int conv_tn_pack(const fn2_conv_desc* d, const float* w, float* wp, cudaStream_t st);
int conv_tn_plan(const fn2_conv_desc* d, int N, int Ho, int Wo, int* out8);
int conv_tn_forward(const fn2_conv_desc* d, const T4& in, const float* wp, const float* bias, const T4& out, cudaStream_t st);

// Which engine owns a layer: taps-on-N (few output channels at high resolution) wherever it applies.
static bool tc_taps_on_n(const fn2_conv_desc* d) { return conv_tn_applicable(d); }

// workspace of the layer's K split; the pixel stride does not matter: only the small-Ci modes depend on it, and they never split
size_t conv_tc_workspace_floats(const fn2_conv_desc* d, int N, int W, int Ho, int Wo) {
    TcPlan pl;
    if (tc_taps_on_n(d) || !tc_plan(d, N, W, Ho, Wo, d->ci, SIZE_MAX, &pl) || pl.p.split_z == 1) return 0;
    return (size_t)(pl.p.ntotal - pl.p.split_first) * pl.p.split_z * 128 * pl.NT + TC_WS_SLACK;
}

// plan8 (fn2_conv_plan), per-tap engine: {NT, tile units, K steps per tile, small-Ci mode (0 plain, 1 tap groups, 2 kernel rows),
// first split tile, K ranges per split tile, 0, 0}; taps-on-N: conv_tn_plan; left 0 for a layer neither engine takes
void conv_tc_plan(const fn2_conv_desc* d, int N, int W, int Ho, int Wo, int ci_stride, int* out8) {
    if (tc_taps_on_n(d)) { conv_tn_plan(d, N, Ho, Wo, out8); return; }
    TcPlan pl;
    if (!tc_plan(d, N, W, Ho, Wo, ci_stride, SIZE_MAX, &pl)) return;
    out8[0] = pl.NT; out8[1] = pl.p.ntotal; out8[2] = pl.steps; out8[3] = pl.w.mode;
    out8[4] = pl.p.split_first; out8[5] = pl.p.split_z;
}

int conv_tc_eligible(const fn2_conv_desc* d, const T4& in, const T4& out) {
    if (in.sc != 1 || out.sc != 1) return 0;
    if (!tc_takes(d)) return 0;
    if (((uintptr_t)in.p & 15) || (in.sw & 3) || (in.sh & 3) || (in.sn & 3)) return 0;
    if (((uintptr_t)out.p & 15) || (out.sw & 3) || (out.sh & 3) || (out.sn & 3)) return 0;
    if (!tc_encode_fn()) return 0;
    // the per-tap engine refuses a deconvolution whose kernel is shorter than its stride (parity classes without taps); the
    // taps-on-N engine takes its own shapes whole
    TcPlan pl;
    return tc_taps_on_n(d) || tc_plan(d, in.n, in.w, out.h, out.w, (int)in.sw, 0, &pl) ? 1 : 0;
}

size_t conv_tc_packed_floats(const fn2_conv_desc* d, int ci_stride) {
    return tc_taps_on_n(d) ? conv_tn_packed_floats(d) : tc_weights(d, ci_stride).floats;
}

int conv_tc_pack(const fn2_conv_desc* d, int ci_stride, const float* w, float* wp, cudaStream_t st) {
    if (tc_taps_on_n(d)) return conv_tn_pack(d, w, wp, st);
    const TcWeights L = tc_weights(d, ci_stride);
    if (!L.floats) return FN2_OK;
    if (L.f16) {
        uint32_t* wmax = reinterpret_cast<uint32_t*>(wp + L.tile_floats);
        const long long n = (long long)d->kh * d->kw * d->ci * d->co;
        FN2_CUDA(cudaMemsetAsync(wmax, 0, sizeof(uint32_t), st));
        const int rc = ew_launch(tc_absmax_kernel, n, st, w, n, wmax);
        if (rc) return rc;
        return ew_launch(tc_pack_f16_kernel, (long long)L.tile_floats * 2, st, w, reinterpret_cast<__half*>(wp), d->ci, d->co, d->kh,
                         d->kw, (d->ci + 31) / 32, d->deconv, wmax);
    }
    const long long per = (long long)L.tile_floats / 2;
    if (L.mode == TC_ROW) return ew_launch(tc_pack_row_kernel, per, st, w, wp, d->ci, d->co, d->kh, d->kw, L.cs, L.rblocks);
    if (L.mode == TC_GROUP) return ew_launch(tc_pack_group_kernel, per, st, w, wp, d->ci, d->co, d->kh, d->kw, L.cs, L.blocks);
    return ew_launch(tc_pack_kernel, per, st, w, wp, d->ci, d->co, d->kh, d->kw, L.width, d->deconv);
}

int conv_tc_forward(const fn2_conv_desc* d, const T4& in, const float* wp, const float* bias, const T4& out, float* ws, size_t ws_floats,
                    cudaStream_t st) {
    if (tc_taps_on_n(d)) return conv_tn_forward(d, in, wp, bias, out, st);
    TcPlan pl;
    const size_t avail = ws && ws_floats > TC_WS_SLACK ? ws_floats - TC_WS_SLACK : 0;
    if (!tc_plan(d, in.n, in.w, out.h, out.w, (int)in.sw, avail, &pl)) {
        set_error("conv_tc: layer not supported (deconvolution parity class without taps)"); return FN2_ERR_INVALID;
    }
    ws = reinterpret_cast<float*>(((uintptr_t)ws + 15) & ~(uintptr_t)15);
    TcParams& p = pl.p;
    const TcWeights& L = pl.w;
    const int NT = pl.NT, su = p.su, sv = p.sv;
    p.out_sn = out.sn; p.out_sh = out.sh; p.out_sw = out.sw;
    // weights (tc_weights): TF32 {width, Co, blocks, hi|lo} read as boxes {32, NT}, one tile at a time; FP16 {32 halves, Co,
    // W_A|W_B|W_C, blocks} read as one box {32, NT, 2} per K block: W_A | W_B, contiguous in each block (W_C is not read)
    CUtensorMap mapW;
    {
        const cuuint64_t row = (cuuint64_t)L.width * (L.f16 ? 2 : 4), tile = row * d->co;
        const int inner = L.f16 ? L.tiles : L.blocks, outer = L.f16 ? L.blocks : L.tiles;
        const cuuint64_t dims[4] = {(cuuint64_t)L.width, (cuuint64_t)d->co, (cuuint64_t)inner, (cuuint64_t)outer};
        const cuuint64_t strides[3] = {row, tile, tile * inner};
        const cuuint32_t box[4] = {32, (cuuint32_t)NT, L.f16 ? 2u : 1u, 1};
        const cuuint32_t es[4] = {1, 1, 1, 1};
        const int rc = tc_tensor_map(&mapW, "conv_tc: weight", L.f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                                     wp, dims, strides, box, es, L.f16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
        if (L.f16) p.wmax = reinterpret_cast<const uint32_t*>(wp + L.tile_floats);
    }
    CUtensorMap mapA;
    {
        cuuint64_t dims[4] = {(cuuint64_t)in.c, (cuuint64_t)in.w, (cuuint64_t)in.h, (cuuint64_t)in.n};
        cuuint64_t strides[3] = {(cuuint64_t)in.sw * 4, (cuuint64_t)in.sh * 4, (cuuint64_t)in.sn * 4};
        cuuint32_t box[4] = {(cuuint32_t)(p.gcs ? p.gcs : 32), (cuuint32_t)(p.tw * su), (cuuint32_t)(p.th * sv), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)su, (cuuint32_t)sv, 1};
        const float* baseA = in.p;
        if (p.rowmode) {
            // dim0: the run of kw*cs floats that starts pad_w pixels left of the output pixel's first tap column;
            // dim1: output column (consecutive runs overlap: stride = su pixels); dim2: input row; dim3: sample
            dims[0] = (cuuint64_t)p.rblocks * 32; dims[1] = (cuuint64_t)p.cls_Wu[0];
            strides[0] = (cuuint64_t)su * p.rcs * 4;
            box[1] = (cuuint32_t)p.tw; es[1] = 1;
            baseA = in.p - (long long)p.rpad * p.rcs;
        }
        const int rc = tc_tensor_map(&mapA, "conv_tc: activation", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, baseA, dims, strides, box, es,
                                     p.gcs ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    const int rc = L.mode == TC_ROW     ? tc_run<TC_ROW>(NT, st, mapA, mapW, bias, out.p, ws, p)
                   : L.mode == TC_GROUP ? tc_run<TC_GROUP>(NT, st, mapA, mapW, bias, out.p, ws, p)
                                        : tc_run<TC_PLAIN>(NT, st, mapA, mapW, bias, out.p, ws, p);
    if (rc || p.split_z == 1) return rc;
    const long long work = (long long)(p.ntotal - p.split_first) * 128 * (NT / 4);
    return tc_with_nt(NT, [&](auto c) { return ew_launch(tc_split_reduce_kernel<decltype(c)::value>, work, st, ws, bias, out.p, p); });
}

// ---------------------------------------------------------------------------------------------------------------------
// Correlation (MULTIPLY, kernel 1, stride_1 1, pad == max_displacement) on the tensor cores.
// stride_2 = S samples displacements that are multiples of S, so a pixel only meets map-1 pixels of its own parity plane;
// within a plane the op is "every pixel against its (2R+1)^2 neighbours", R = md / S.  Per 8x16-pixel tile the neighbours are
// the (8+2R) x (16+2R) halo; the kernel computes ALL tile-pixel x halo-pixel dot products as 3xTF32 GEMMs
// D[128 x 112] = A[128 x C] * B[112 x C]^T (one unit per block of 4 full halo rows: 9 blocks for R = 10) and keeps the 441 of the
// 1008 that lie in the window (2.3x redundant MMA work, which still beats the FP32 FMA pipe by a wide margin).
// Map 1 is split into TF32 hi / lo once per call (workspace [2][N][H][W][C]); both maps are read through element-strided
// TMA boxes, so the parity planes are never materialised and out-of-image neighbours are zero fill.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void corr_split_kernel(const float* __restrict__ b, long long sn, long long sh, long long sw, int N, int H, int W, int C,
                                  float* __restrict__ hi, float* __restrict__ lo) {
    const long long total = (long long)N * H * W * (C / 4);
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % (C / 4)) * 4;
        long long r = idx / (C / 4);
        const int x = (int)(r % W); r /= W;
        const int y = (int)(r % H);
        const int n = (int)(r / H);
        const float4 v = *reinterpret_cast<const float4*>(b + n * sn + y * sh + x * sw + c);
        const float f[4] = {v.x, v.y, v.z, v.w};
        float h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint32_t hb = to_tf32_nan(f[e]);
            h[e] = __uint_as_float(hb);
            l[e] = __uint_as_float(to_tf32(f[e] - h[e]));
        }
        const long long o = (((long long)n * H + y) * W + x) * C + c;
        *reinterpret_cast<float4*>(hi + o) = make_float4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<float4*>(lo + o) = make_float4(l[0], l[1], l[2], l[3]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient of Convolution / Deconvolution on the tensor cores (base_conv_layer.cpp:352-372 weight_gpu_gemm).
//   dW[a][b][ky][kx] = sum over (n, u, v) small[n, a, u, v] * big[n, b, u*s + ky - pad, v*s + kx - pad]
// with (small, big) = (top diff, bottom) for a convolution and (bottom, top diff) for a deconvolution: in both cases the Caffe
// blob is [small channels][big channels][kh][kw].  Per kernel tap this is a GEMM D[big ch x small ch] over K = pixels, and with
// both maps transposed to channel-major planes (pixels contiguous) its operands are K-major tiles exactly like the forward
// engine's: A = 128 channel rows x 32 consecutive pixels of the big map (raw FP32, split into TF32 hi/lo by the MMA warpgroups),
// B = NT channel rows x the same 32 pixels of the small map, pre-split once by the transposition pass.  The tap's shift is a TMA
// coordinate offset (zero fill = the convolution's padding); a strided layer reads the column-parity plane the tap falls into.
// Same FP32-faithful accumulation as the forward pass (short RZ chains drained to FP32 registers).
// ---------------------------------------------------------------------------------------------------------------------
struct WgPlan {
    int Cb, Cs, Hb, Wb, Hs, Ws, N, sx, sy;
    int NT, BT, ST, S, segs_x, segs, taps, G, TPT, TG;   // G rows per tap, TPT taps per 128-row tile, TG tap groups
    int Wq, Wq_p, Ws_p;                           // columns per parity plane (and its padded pitch), padded pitch of the small map
    size_t big_floats, small_floats, part_floats; // workspace pieces (each a multiple of 64 floats)
    size_t bias_floats;                           // per-block channel sums of the top diff (bias gradient, fused into its transposition)
    int bias_blocks;
};
static size_t up64(size_t x) { return (x + 63) / 64 * 64; }

static WgPlan wg_plan(const fn2_conv_desc* d, int N, int H, int W) {
    WgPlan g;
    int Ho = 0, Wo = 0;
    fn2_conv_out_shape(d, H, W, &Ho, &Wo);
    g.N = N; g.sx = d->stride_w; g.sy = d->stride_h; g.taps = d->kh * d->kw;
    if (!d->deconv) { g.Cb = d->ci; g.Cs = d->co; g.Hb = H; g.Wb = W; g.Hs = Ho; g.Ws = Wo; }
    else            { g.Cb = d->co; g.Cs = d->ci; g.Hb = Ho; g.Wb = Wo; g.Hs = H; g.Ws = W; }
    g.NT = g.Cs >= 128 ? 128 : (g.Cs >= 64 ? 64 : (g.Cs >= 32 ? 32 : 16));
    g.BT = (g.Cb + 127) / 128; g.ST = (g.Cs + g.NT - 1) / g.NT;
    g.G = 128;
    if (g.Cb <= 64) { g.G = 8; while (g.G < g.Cb) g.G *= 2; }
    g.TPT = 128 / g.G; g.TG = (g.taps + g.TPT - 1) / g.TPT;
    g.segs_x = (g.Ws + 31) / 32; g.segs = N * g.Hs * g.segs_x;
    const int base = g.TG * g.BT * g.ST;
    g.S = max(1, min((3 * num_sms() + base - 1) / base, g.segs / 8));
    g.Wq = (g.Wb + g.sx - 1) / g.sx + 3;          // + 3: room for the column delay of the 4 copies
    g.Wq_p = (g.Wq + 3) / 4 * 4; g.Ws_p = (g.Ws + 3) / 4 * 4;
    g.big_floats = up64((size_t)4 * N * g.Cb * g.Hb * g.sx * g.Wq_p);          // 4 copies, delayed by 0..3 columns
    g.small_floats = up64((size_t)2 * N * g.Cs * g.Hs * g.Ws_p);
    g.part_floats = up64((size_t)base * g.S * 128 * g.NT);
    // the top diff is the small map of a convolution and the big map of a deconvolution
    g.bias_blocks = d->deconv ? ((g.Wq_p + 127) / 128) * (N * g.Hb * g.sx) : ((g.Ws_p + 127) / 128) * (N * g.Hs);
    g.bias_floats = d->has_bias ? up64((size_t)g.bias_blocks * d->co) : 0;
    return g;
}

// channel-major planes: dst[dl][((n*C + c)*H + h)*sx + par][j] = src[n, c, h, (j - dl)*sx + par] (zero outside the row) for
// dl < nadv column delays; SPLIT writes the TF32 hi plane there and the lo plane `lo_off` floats further
// `dlmask`: which of the 4 delays are written (bit dl); the source is read once per block: 32 channels x (WG_TW + 3) columns.
// bias_part != nullptr: also the per-block channel sums of src, [block (x, z)][C] (the bias gradient when src is the top diff).
constexpr int WG_TW = 128;                        // columns per block (4 x the 32 threads of a row)
template <bool SPLIT>
__global__ void __launch_bounds__(256) wg_transpose_kernel(T4 src, float* __restrict__ dst, int sx, int Wq, int Wq_p, long long lo_off, int dlmask,
                                                           float* __restrict__ bias_part) {
    __shared__ float tile[WG_TW + 3][33];
    __shared__ float red[8][33];
    // grid: x = (sample, row, parity) -- the long dimension --, y = channel tile, z = column tile
    const int wq0 = blockIdx.z * WG_TW, c0 = blockIdx.y * 32;
    const int rp = blockIdx.x % (src.h * sx), n = blockIdx.x / (src.h * sx);
    const int h = rp / sx, par = rp % sx;
    const int halo = SPLIT ? 0 : 3;
    const int cols = min(WG_TW, Wq_p - wq0);                         // columns of this block that exist in the destination row
    for (int j = threadIdx.y; j < cols + halo; j += 8) {
        const int wq = wq0 + j - halo, w = wq * sx + par, c = c0 + threadIdx.x;       // tile row j = column wq0 + j - halo
        tile[j][threadIdx.x] = (c < src.c && wq >= 0 && w < src.w) ? src.p[src.off(n, c, h, w)] : 0.f;
    }
    __syncthreads();
    if (bias_part) {
        float a = 0.f;
        for (int j = threadIdx.y; j < cols; j += 8) a += tile[j + halo][threadIdx.x];           // the core columns, fixed order
        red[threadIdx.y][threadIdx.x] = a;
        __syncthreads();
        if (threadIdx.y == 0 && c0 + threadIdx.x < src.c) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 8; k++) t += red[k][threadIdx.x];
            bias_part[((long long)blockIdx.z * gridDim.x + blockIdx.x) * src.c + c0 + threadIdx.x] = t;
        }
    }
    const long long copy = (long long)src.n * src.c * src.h * sx * Wq_p;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int c = c0 + j;
        if (c >= src.c) continue;
        float* row = dst + (((long long)n * src.c + c) * src.h * sx + rp) * Wq_p + wq0;
        for (int x = threadIdx.x; x < cols; x += 32) {
            if (SPLIT) {
                const float v = tile[x][j];
                const float hi = __uint_as_float(to_tf32(v));
                row[x] = hi;
                row[x + lo_off] = __uint_as_float(to_tf32(v - hi));
            } else {
#pragma unroll
                for (int dl = 0; dl < 4; dl++)
                    if (dlmask >> dl & 1) row[x + dl * copy] = tile[x + 3 - dl][j];       // index wq holds column wq - dl
            }
        }
    }
}

// db[c] (+)= sum over the blocks' partial sums, fixed order: 8 strided groups per channel, then the 8 group sums
__global__ void wg_bias_final_kernel(const float* __restrict__ part, float* __restrict__ db, int C, int blocks, int accumulate) {
    __shared__ float red[32][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float a = 0.f;
    if (c < C)
        for (int k = threadIdx.y; k < blocks; k += 32) a += part[(long long)k * C + c];
    red[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 32; k++) t += red[k][threadIdx.x];
        db[c] = accumulate ? db[c] + t : t;
    }
}

// dW[a][b][tap] (+)= sum over the K ranges of part[unit][row = (tap % TPT) * G + b % 128][col = a % NT]; threads run along the
// Caffe layout (coalesced read-modify-write of the diff; the strided partial reads hit L2).  A variant with coalesced partial reads
// and scattered diff updates measured 2.3x slower.
__global__ void wg_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, WgPlan g, int accumulate) {
    const long long total = (long long)g.Cs * g.Cb * g.taps;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int tap = (int)(idx % g.taps);
        const long long r = idx / g.taps;
        const int b = (int)(r % g.Cb), a = (int)(r / g.Cb);
        const long long unit0 = ((long long)((tap / g.TPT) * g.BT + b / 128) * g.ST + a / g.NT) * g.S;
        const float* src = part + (unit0 * 128 + (tap % g.TPT) * g.G + (b % 128)) * g.NT + (a % g.NT);
        float acc = 0.f;
        for (int k = 0; k < g.S; k++) acc += src[(long long)k * 128 * g.NT];
        dw[idx] = accumulate ? dw[idx] + acc : acc;
    }
}

// the layer shapes the weight-gradient engine takes (engine 1 = `engine: CAFFE`: exact-FP32 SIMT everywhere)
int conv_tc_wgrad_takes(const fn2_conv_desc* d) {
    return d->engine != 1 && d->kh * d->kw <= 49 && d->stride_w <= 8 && d->stride_h <= 8;
}
int conv_tc_wgrad_eligible(const fn2_conv_desc* d) {
    return conv_tc_wgrad_takes(d) && tc_encode_fn() ? 1 : 0;
}
size_t conv_tc_wgrad_workspace_floats(const fn2_conv_desc* d, int N, int H, int W) {
    const WgPlan g = wg_plan(d, N, H, W);
    return g.big_floats + g.small_floats + g.part_floats + g.bias_floats + 64;
}
// plan8 of fn2_conv_wgrad_plan for the tensor-core route: {2, NT, G, TG, BT, ST, S, bias blocks (0 without a bias)}
void conv_tc_wgrad_plan(const fn2_conv_desc* d, int N, int H, int W, int32_t* out8) {
    const WgPlan g = wg_plan(d, N, H, W);
    out8[0] = 2; out8[1] = g.NT; out8[2] = g.G; out8[3] = g.TG; out8[4] = g.BT; out8[5] = g.ST; out8[6] = g.S;
    out8[7] = d->has_bias ? g.bias_blocks : 0;
}

int conv_tc_wgrad(const fn2_conv_desc* d, const T4& bottom, const T4& top_diff, float* dw, float* db, int accumulate, float* ws,
                  size_t ws_floats, cudaStream_t st) {
    const WgPlan g = wg_plan(d, bottom.n, bottom.h, bottom.w);
    if (!ws || ws_floats < conv_tc_wgrad_workspace_floats(d, bottom.n, bottom.h, bottom.w)) { set_error("conv_tc_wgrad: workspace too small"); return FN2_ERR_WORKSPACE; }
    const T4& big = d->deconv ? top_diff : bottom;
    const T4& small = d->deconv ? bottom : top_diff;
    if (big.h != g.Hb || big.w != g.Wb || small.h != g.Hs || small.w != g.Ws || big.c != g.Cb || small.c != g.Cs) {
        set_error("conv_tc_wgrad: tensor shapes do not match the descriptor"); return FN2_ERR_INVALID;
    }
    ws = reinterpret_cast<float*>(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    float* bigT = ws; float* smallT = ws + g.big_floats; float* part = smallT + g.small_floats;
    float* bias_part = (d->has_bias && db) ? part + g.part_floats : nullptr;
    {
        dim3 blk(32, 8);
        int dlmask = 0;                                     // column delays the layer's taps actually use
        for (int kx = 0; kx < d->kw; kx++) {
            const int q = kx - d->pad_w, par = ((q % g.sx) + g.sx) % g.sx, shift = (q - par) / g.sx;
            dlmask |= 1 << ((((-shift) % 4) + 4) % 4);
        }
        dim3 gb((unsigned)(g.N * g.Hb * g.sx), (unsigned)((g.Cb + 31) / 32), (unsigned)((g.Wq_p + WG_TW - 1) / WG_TW));
        wg_transpose_kernel<false><<<gb, blk, 0, st>>>(big, bigT, g.sx, g.Wq, g.Wq_p, 0, dlmask, d->deconv ? bias_part : nullptr);
        FN2_LAUNCH_CHECK();
        dim3 gs((unsigned)(g.N * g.Hs), (unsigned)((g.Cs + 31) / 32), (unsigned)((g.Ws_p + WG_TW - 1) / WG_TW));
        wg_transpose_kernel<true><<<gs, blk, 0, st>>>(small, smallT, 1, g.Ws, g.Ws_p, (long long)g.N * g.Cs * g.Hs * g.Ws_p, 1,
                                                      d->deconv ? nullptr : bias_part);
        FN2_LAUNCH_CHECK();
        if (bias_part) {
            wg_bias_final_kernel<<<(unsigned)((d->co + 31) / 32), dim3(32, 32), 0, st>>>(bias_part, db, d->co, g.bias_blocks, accumulate);
            FN2_LAUNCH_CHECK();
        }
    }
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.N = g.N; p.cblocks = 1;
    p.Ho = g.Hs; p.Wo = g.Ws;
    p.split_z = 1; p.su = g.sx; p.sv = g.sy; p.ou = p.ov = 1; p.ncls = 1;
    p.tw = 128; p.th = 1; p.tiles_x = p.tiles_y = 1;
    p.wg_S = g.S; p.wg_ST = g.ST; p.wg_BT = g.BT; p.wg_segs = g.segs; p.wg_segs_x = g.segs_x; p.wg_sx = g.sx;
    p.wg_G = g.G; p.wg_TPT = g.TPT; p.wg_taps = g.taps;
    p.kd = tc_chunk_steps(g.NT);
    for (int ky = 0; ky < d->kh; ky++)
        for (int kx = 0; kx < d->kw; kx++) {
            const int t = ky * d->kw + kx, q = kx - d->pad_w;
            const int par = ((q % g.sx) + g.sx) % g.sx;
            const int shift = (q - par) / g.sx, dl = (((-shift) % 4) + 4) % 4;    // copy `dl` holds column j - dl at index j
            p.dy[t] = (short)(ky - d->pad_h); p.dx[t] = (short)(shift + dl); p.widx[t] = (short)(par | (dl << 4));
        }
    p.total = g.TG * g.BT * g.ST * g.S;
    p.ntotal = p.total; p.split_first = p.total;
    CUtensorMap mapA, mapB;
    {
        cuuint64_t dims[4] = {(cuuint64_t)g.Wq, (cuuint64_t)g.Hb * g.sx, (cuuint64_t)g.Cb, (cuuint64_t)4 * g.N};
        cuuint64_t strides[3] = {(cuuint64_t)g.Wq_p * 4, (cuuint64_t)g.Hb * g.sx * g.Wq_p * 4, (cuuint64_t)g.Cb * g.Hb * g.sx * g.Wq_p * 4};
        cuuint32_t box[4] = {32, 1, (cuuint32_t)g.G, 1};
        cuuint32_t es[4] = {1, 1, 1, 1};
        const int rc = tc_tensor_map(&mapA, "conv_tc_wgrad: big-map", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, bigT, dims, strides, box, es,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    {
        cuuint64_t dims[4] = {(cuuint64_t)g.Ws, (cuuint64_t)g.Hs, (cuuint64_t)g.Cs, (cuuint64_t)2 * g.N};
        cuuint64_t strides[3] = {(cuuint64_t)g.Ws_p * 4, (cuuint64_t)g.Hs * g.Ws_p * 4, (cuuint64_t)g.Cs * g.Hs * g.Ws_p * 4};
        cuuint32_t box[4] = {32, 1, (cuuint32_t)g.NT, 1};
        cuuint32_t es[4] = {1, 1, 1, 1};
        const int rc = tc_tensor_map(&mapB, "conv_tc_wgrad: small-map", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, smallT, dims, strides, box, es,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    const int rc = tc_run<TC_WGRAD>(g.NT, st, mapA, mapB, nullptr, nullptr, part, p);
    if (rc) return rc;
    wg_reduce_kernel<<<ew_grid((long long)g.Cs * g.Cb * g.taps, 256), 256, 0, st>>>(part, dw, g, accumulate);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

// The correlation route itself is chosen in fn2_corr.cu (corr_fwd_route); this says whether the tensor cores may take it.
bool corr_tc_available() { return tc_encode_fn() != nullptr; }
size_t corr_tc_workspace_floats(int N, int C, int H, int W) { return (size_t)2 * N * H * W * C; }

// R = 10, s2 <= 2, C % 32 == 0, channel-fast maps with 16-byte aligned pixels; ws holds corr_tc_workspace_floats
int corr_tc_forward(const T4& b0, const T4& b1, const T4& top, int R, int s2, float* ws, cudaStream_t st) {
    const int N = b0.n, C = b0.c, H = b0.h, W = b0.w, S = s2;
    float* hi = ws; float* lo = ws + (size_t)N * H * W * C;
    corr_split_kernel<<<ew_grid((long long)N * H * W * (C / 4), 256), 256, 0, st>>>(b1.p, b1.sn, b1.sh, b1.sw, N, H, W, C, hi, lo);
    FN2_LAUNCH_CHECK();
    constexpr int NT = 128;
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.cR = R; p.cS = S; p.cD = 2 * R + 1;
    p.tw = 8; p.th = 16;                                                   // halo 28 x 36
    p.cbw = p.tw + 2 * R; p.cbh = 4;                                       // block = 4 full halo rows = 112 pixels (MMA N = 112)
    p.cnt = (p.th + 2 * R) / p.cbh;                             // 9 blocks
    p.cscale = 1.0f / (float)C;                                           // sumelems = k*k*C (correlation_layer.cu:108)
    p.N = N; p.cblocks = C / 32;
    p.Ho = H; p.Wo = W;
    p.out_sn = top.sn; p.out_sh = top.sh; p.out_sw = top.sw;
    p.split_z = 1; p.su = S; p.sv = S; p.ou = p.ov = 1; p.ncls = 1;
    p.kd = tc_chunk_steps(NT);
    const int Ws = (W + S - 1) / S, Hs = (H + S - 1) / S;
    p.tiles_x = (Ws + p.tw - 1) / p.tw; p.tiles_y = (Hs + p.th - 1) / p.th;
    p.total = N * S * S * p.tiles_x * p.tiles_y * p.cnt;
    p.ntotal = p.total; p.split_first = p.total;
    CUtensorMap mapA, mapB;
    {
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
        cuuint64_t strides[3] = {(cuuint64_t)b0.sw * 4, (cuuint64_t)b0.sh * 4, (cuuint64_t)b0.sn * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)(p.tw * S), (cuuint32_t)(p.th * S), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)S, (cuuint32_t)S, 1};
        const int rc = tc_tensor_map(&mapA, "corr_tc: map-0", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, b0.p, dims, strides, box, es,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    {
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)2 * N};
        cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)(p.cbw * S), (cuuint32_t)(p.cbh * S), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)S, (cuuint32_t)S, 1};
        const int rc = tc_tensor_map(&mapB, "corr_tc: map-1", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, hi, dims, strides, box, es,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    return tc_launch<conv_tc_kernel<NT, TC_CORR>>(p.total, TC_THREADS, TcGeo<NT>::SMEM, false, st, mapA, mapB, (const float*)nullptr,
                                                 top.p, (float*)nullptr, p);
}

}  // namespace fn2
