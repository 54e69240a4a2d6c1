// The solver's parameter update: SGDSolver::ApplyUpdate (reference: src/caffe/solvers/sgd_solver.cpp:102-116) as one pass over
// the parameter arena.  Per element of every trainable parameter blob, in the reference's order:
//   ClipGradients   g *= scale                              (:81-99; scale from solver_clip_scale below)
//   Normalize       g *= 1 / iter_size                      (:119-142)
//   Regularize      g += local_decay * w   or   * sign(w)   (:145-204, L2 / L1)
//   SGD             h = fma(momentum, h, local_rate * g); g = h                       (sgd_solver.cu:6-12)
//   Adam            m = fma(1 - b1, g, m * b1); v = fma(1 - b2, g * g, v * b2);
//                   g = local_rate * correction * m / (sqrt(v) + delta)             (adam_solver.cu:6-16)
//   Net::Update     w -= g                                  (blob.cpp:Update, net.cpp:957-964)
// The diff keeps the applied update value, as in the reference.  Compiled with -fmad=false, so the only fused multiply-adds are
// the three written out above: the ones the reference's own nvcc build (-fmad=true) makes of SGDUpdate and AdamUpdate (read off
// its SASS).  Given the same gradient, the SGD and Adam steps therefore equal the reference kernels' bit for bit, and the whole
// update equals a float32 restatement of these expressions (tests/solver_oracle.py) bit for bit.
//
// The pass is bound by HBM traffic (SGD reads w, g, h and writes all three; Adam adds m/v).  Work is cut into chunks of
// kChunkGroups float4 groups, each inside one parameter blob: the arena pads every blob to 64 floats.  When a blob's count is
// not a multiple of 4, its last float4 also loads up to 3 pad floats; they take no part in the update and are stored back
// with the values they had.  The chunk table is built once per solver.
#include "fn2_common.cuh"
#include "caffe/solver_update.hpp"

namespace fn2 {

namespace {

__device__ __forceinline__ float at(const float4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }
__device__ __forceinline__ void set(float4& v, int k, float x) {
    if (k == 0) v.x = x; else if (k == 1) v.y = x; else if (k == 2) v.z = x; else v.w = x;
}

template <bool ADAM>
__global__ void __launch_bounds__(kChunkGroups) solver_update_kernel(SolverUpdateArgs a) {
    const SolverChunk c = a.chunks[blockIdx.x];
    const SolverSegment s = a.segs[c.seg];
    const long long e0 = ((long long)c.group + threadIdx.x) * 4;       // first element of this thread's group in the blob
    if (e0 >= s.count) return;
    const int valid = (int)min(4LL, (long long)s.count - e0);
    float4* wp = reinterpret_cast<float4*>(a.data + s.offset + e0);
    float4* gp = reinterpret_cast<float4*>(a.diff + s.offset + e0);
    float4* hp = reinterpret_cast<float4*>(a.hist0 + s.hist_offset + e0);
    float4 w = *wp, g = *gp, h = *hp, v = make_float4(0.f, 0.f, 0.f, 0.f);
    float4* vp = nullptr;
    if (ADAM) { vp = reinterpret_cast<float4*>(a.hist1 + s.hist_offset + e0); v = *vp; }
    const float scale = a.clip_scale ? *a.clip_scale : 1.f;
    const float local_rate = a.rate * s.lr_mult;
    const float corrected_rate = local_rate * a.correction;
    for (int k = 0; k < valid; k++) {
        const float wk = at(w, k);
        float gk = at(g, k);
        if (a.clip_scale) gk = gk * scale;
        if (a.normalize) gk = gk * a.accum_normalization;
        if (s.local_decay != 0.f) {
            const float r = a.l1 ? (float)((0.f < wk) - (wk < 0.f)) : wk;
            gk = s.local_decay * r + gk;
        }
        if (ADAM) {
            const float mk = fmaf(1.f - a.momentum, gk, at(h, k) * a.momentum);
            const float vk = fmaf(1.f - a.momentum2, gk * gk, at(v, k) * a.momentum2);
            gk = corrected_rate * mk / (sqrtf(vk) + a.delta);
            set(h, k, mk);
            set(v, k, vk);
        } else {
            gk = fmaf(a.momentum, at(h, k), local_rate * gk);
            set(h, k, gk);
        }
        set(g, k, gk);
        set(w, k, wk - gk);
    }
    *wp = w; *gp = g; *hp = h;
    if (ADAM) *vp = v;
}

// Sum of squares of the trainable gradients: one double partial per chunk, then one block adds the partials in index order.
// The same inputs give the same scale on every run and every rank.
__global__ void __launch_bounds__(kChunkGroups) solver_sumsq_kernel(const float* diff, const SolverSegment* segs,
                                                                   const SolverChunk* chunks, double* partial) {
    const SolverChunk c = chunks[blockIdx.x];
    const SolverSegment s = segs[c.seg];
    const long long e0 = ((long long)c.group + threadIdx.x) * 4;
    double acc = 0;
    if (e0 < s.count) {
        const float4 g = *reinterpret_cast<const float4*>(diff + s.offset + e0);
        const int valid = (int)min(4LL, (long long)s.count - e0);
        for (int k = 0; k < valid; k++) acc += (double)at(g, k) * (double)at(g, k);
    }
    __shared__ double red[kChunkGroups];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int n = kChunkGroups / 2; n > 0; n >>= 1) {
        if ((int)threadIdx.x < n) red[threadIdx.x] += red[threadIdx.x + n];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

constexpr int kReduceThreads = 1024;

// ClipGradients' decision (sgd_solver.cpp:89-97) on the device: scale = clip / ||g|| when ||g|| > clip, else 1.
__global__ void __launch_bounds__(kReduceThreads) solver_clip_scale_kernel(const double* partial, int n, float clip, float* scale) {
    double acc = 0;
    for (int i = threadIdx.x; i < n; i += kReduceThreads) acc += partial[i];
    __shared__ double red[kReduceThreads];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int m = kReduceThreads / 2; m > 0; m >>= 1) {
        if ((int)threadIdx.x < m) red[threadIdx.x] += red[threadIdx.x + m];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float l2norm = (float)sqrt(red[0]);
        *scale = l2norm > clip ? clip / l2norm : 1.f;
    }
}

}  // namespace

int solver_clip_scale(const float* diff, const SolverSegment* segs, const SolverChunk* chunks, int nchunks, double* partial,
                      float clip, float* scale, cudaStream_t st) {
    FN2_CHECK_ARG(nchunks > 0, "solver_clip_scale: no trainable parameters");
    solver_sumsq_kernel<<<nchunks, kChunkGroups, 0, st>>>(diff, segs, chunks, partial);
    FN2_LAUNCH_CHECK();
    solver_clip_scale_kernel<<<1, kReduceThreads, 0, st>>>(partial, nchunks, clip, scale);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

int solver_update(const SolverUpdateArgs& a, int nchunks, bool adam, cudaStream_t st) {
    FN2_CHECK_ARG(nchunks > 0, "solver_update: no trainable parameters");
    if (adam) solver_update_kernel<true><<<nchunks, kChunkGroups, 0, st>>>(a);
    else solver_update_kernel<false><<<nchunks, kChunkGroups, 0, st>>>(a);
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

}  // namespace fn2
