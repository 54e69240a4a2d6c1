// Device side of the solver's update (fn2_solver.cu), as the host solver (solver.cpp) drives it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fn2 {

constexpr int kChunkGroups = 256;          // float4 groups per chunk = threads per block of the update pass

// One trainable parameter blob: where it lies in the parameter / gradient arenas and in the solver's history, and its
// ParamSpec multipliers (lr_mult != 0; local_decay = weight_decay * decay_mult).  Offsets are multiples of 64 floats.
struct SolverSegment {
    long long offset, hist_offset, count;
    float lr_mult, local_decay;
};
// kChunkGroups float4 groups of one segment, starting at float4 group `group` of the blob
struct SolverChunk {
    int seg, group;
};

struct SolverUpdateArgs {
    float* data;                           // parameter arena
    float* diff;                           // gradient arena
    float* hist0;                          // SGD history / Adam m
    float* hist1;                          // Adam v
    const SolverSegment* segs;
    const SolverChunk* chunks;
    const float* clip_scale;               // device scalar from solver_clip_scale, or nullptr without clipping
    float rate;                            // GetLearningRate
    float momentum, momentum2, delta;      // SGD momentum / Adam beta1, beta2, eps_hat
    float correction;                      // Adam's bias correction for this iteration
    float accum_normalization;             // 1 / iter_size
    int normalize;                         // iter_size != 1
    int l1;                                // regularization_type L1 (else L2)
};

int solver_clip_scale(const float* diff, const SolverSegment* segs, const SolverChunk* chunks, int nchunks, double* partial,
                      float clip, float* scale, cudaStream_t st);
int solver_update(const SolverUpdateArgs& a, int nchunks, bool adam, cudaStream_t st);

}  // namespace fn2
