// wgmma / TMA / mbarrier PTX wrappers and constants shared by the tensor-core engines (fn2_conv_tc.cu, fn2_conv_tn.cu) and the
// FP32 fast correlation (fn2_corr_fast.cu: mbarrier, TMA and the tensor-map helper), and the host helpers that encode their tensor
// maps and launch them; sm_90a.
#pragma once
#include <cuda.h>
#include "fn2_common.cuh"

namespace fn2 {

// Encodes a 4-D tiled tensor map of `base`: dims, byte strides of dims 1-3, box, element strides, no interleave, zero fill out of
// bounds (fn2_conv_tc.cu).  FN2_ERR_CUDA, with "<what> tensor map ..." as the last error, when the driver has no encoder or the
// encode fails.
int tc_tensor_map(CUtensorMap* map, const char* what, CUtensorMapDataType dtype, const void* base, const cuuint64_t* dims,
                  const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* es, CUtensorMapSwizzle swizzle,
                  CUtensorMapL2promotion l2);

// Launches a persistent tensor-core kernel: min(units, SM count) CTAs of `threads` threads with `smem` bytes of dynamic shared
// memory.  The kernel's shared-memory limit is raised when a launch needs more than the last one set; Kernel is a template
// argument so that this state is per kernel (the instantiations of one kernel template share a function type), and it is per
// process (one device per process, as num_sms assumes).  pdl: programmatic stream serialization, so that the kernel's CTAs may
// start on SMs the previous kernel of the stream leaves; the kernel then waits in griddepcontrol.wait before it reads anything.
template <auto Kernel, class... Args>
int tc_launch(int units, int threads, int smem, bool pdl, cudaStream_t st, const Args&... args) {
    static int smem_set = 0;
    if (smem > smem_set) {
        FN2_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        smem_set = smem;
    }
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)min(units, num_sms()));
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    FN2_CUDA(cudaLaunchKernelEx(&cfg, Kernel, args...));
    FN2_LAUNCH_CHECK();
    return FN2_OK;
}

// Mean relative loss of an FP32 accumulator per MMA that adds a non-zero product to it: the tensor core truncates (rounds
// toward zero) its accumulator, so a chain of n MMAs shrinks the result by about n times this, and both engines add that
// back.  H100: ~1.1e-8 .. 1.3e-8, from the mean signed errors of the tensor-core parity cases of tests/test_ops_gpu.py
// (per-tap engine, and the taps-on-N engine at Ci = 40 / 64 / 96: 1.1e-8 / 1.33e-8 / 1.3e-8), with no constant term.
// Recalibrating: build a side library with this set to 0, load it through FN2_LIB and run those tests; the mean signed error
// ("shrink") they compute, divided by the number of MMAs the engine's compensation counts per chain, is the new value.
constexpr float TRUNC_LOSS_PER_MMA = 1.3e-8f;
// The same loss per a_hi * W_A MMA (m64n128k16, FP16 operands) of the per-tap engine's FP16 route (NT = 128, plain K blocks; 2
// such MMAs per K step), calibrated the same way: with it set to 0 the NT = 128 forward and data-gradient cases of
// tests/test_conv_tc_routes_gpu.py shrink by 5.7e-8 .. 6.6e-8 (H100 80GB HBM3, 700 W), 6.2e-8 on average; with it, +2.0e-8.
constexpr float TRUNC_LOSS_PER_MMA_F16 = 3.1e-8f;

namespace {

// division by a launch constant without the ~40-instruction integer divide (the tile decode is on the critical path of the
// single-thread producer and MMA roles once per tile): q = (umulhi(n, mul) + n) >> shift for n < 2^31
struct FastDiv {
    uint32_t mul, shift, d;
    __host__ void init(int div) {
        d = (uint32_t)div;
        shift = 0;
        while ((1u << shift) < d) shift++;
        mul = (uint32_t)(((1ull << 32) * ((1ull << shift) - d)) / d + 1);
    }
    __device__ __forceinline__ int div(int n) const { return (int)(((uint32_t)__umulhi((uint32_t)n, mul) + (uint32_t)n) >> shift); }
    __device__ __forceinline__ void divmod(int n, int& q, int& r) const { q = div(n); r = n - q * (int)d; }
};

__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(su32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0, spins = 0;
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(su32(bar)), "r"(parity) : "memory");
        if (done) break;
        if (++spins > (1u << 24)) __trap();       // a lost arrival becomes a launch error, never a hang
    }
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(su32(dst)), "l"(map), "r"(su32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMAs
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
// x rounded half away from zero to TF32 (11 significant bits), as cvt.rna.tf32.f32 rounds a finite x.  A NaN does not survive
// it: the rounding add carries the payload of the device's own NaN (0x7fffffff) into the sign bit, giving -0, and turns a NaN
// with a small payload (0x7f800001) into Inf.  The convolution engines split with it in their MMA inner loop, where the NaN
// test of to_tf32_nan cost 1.5 % of the FlowNet2 deploy step (H100 80GB HBM3, 700 W).
__device__ __forceinline__ uint32_t to_tf32(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
// to_tf32 that keeps a NaN a NaN (the canonical one: the tensor cores read only the upper 19 bits).  The correlation splits
// both maps with it, so that a NaN in either bottom reaches the products as in the reference's FP32 code.
__device__ __forceinline__ uint32_t to_tf32_nan(float x) { return x != x ? 0x7fffffffu : to_tf32(x); }
// weight packing: wp[idx] = v rounded to TF32, wp[per + idx] = the remainder rounded to TF32 (cvt.rna)
__device__ __forceinline__ void store_tf32_split(float* wp, long long per, long long idx, float v) {
    uint32_t h, l;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(v));
    const float hi = __uint_as_float(h);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(v - hi));
    wp[idx] = hi;
    wp[per + idx] = __uint_as_float(l);
}
// shared-memory matrix descriptor (sm_90 wgmma): K-major, SWIZZLE_128B, 8-row atoms of 1024 B, tile base 1024-byte aligned.
// Adding 2 to the start-address field (+32 bytes) selects the next 8 TF32 columns of the swizzled tile.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;                       // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset: next 8-row atom
    d |= (uint64_t)1 << 62;                       // layout: 128-byte swizzle
    return d;
}
// the same for K-major SWIZZLE_64B tiles of 32 halves per row (8-row atoms of 512 B, tile base 512-byte aligned); adding 2 to
// the start-address field (+32 bytes) selects the second 16 columns
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;                       // layout: 64-byte swizzle
    return d;
}

// A operand of one K step in wgmma register-fragment order: a[4*kk + q] = element (row rq = q&1 ? r1 : r0, column
// 8*kk + t + 4*(q>>1)) of the K block, split into hi / lo.  Plain layout: the raw tile is K-major SWIZZLE_128B (16-byte
// chunk c of row r at chunk position c ^ (r & 7)); the 32 lanes of a warp hit 32 different banks.
// KEEP_NAN: the high part keeps a NaN (to_tf32_nan); the remainder of a non-finite f needs no test, the high part already
// carries it into every product.
template <bool KEEP_NAN = false>
__device__ __forceinline__ void split_store(float f, uint32_t& hi, uint32_t& lo) {
    const uint32_t h = KEEP_NAN ? to_tf32_nan(f) : to_tf32(f);
    hi = h;
    lo = to_tf32(f - __uint_as_float(h));
}
__device__ __forceinline__ float raw_at(const unsigned char* st, int r, int chunk, int t) {
    return *reinterpret_cast<const float*>(st + r * 128 + ((chunk ^ (r & 7)) << 4) + t * 4);
}
// wgmma.mma_async m64nNk8 kind tf32, A from registers (RS form), B from a shared-memory descriptor, FP32 accumulator.
// d: the N/2 accumulator registers of this thread (column 8*(j/4) + 2*(lane%4) + (j%2), row lane/4 + 8*((j/2)%2) of the
// warp's 16 rows); a: {a(g, t), a(g+8, t), a(g, t+4), a(g+8, t+4)} of the warp's 16 x 8 A slice (g = lane/4, t = lane%4).
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<32> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<64> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<80> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %45, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, {%40,%41,%42,%43}, %44, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<96> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %53, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, {%48,%49,%50,%51}, %52, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<112> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %61, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n112k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, {%56,%57,%58,%59}, %60, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
template <> struct Wgmma<128> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};
// wgmma.mma_async m64nNk16 kind f16 (FP16 operands, FP32 accumulator), A from registers: the accumulator layout of Wgmma<N>;
// a: four f16x2 registers {row g, cols 2t..2t+1}, {row g+8, cols 2t..2t+1}, {row g, cols 2t+8..2t+9}, {row g+8, cols 2t+8..2t+9}
// of the warp's 16 x 16 A slice, the lower column in the low half.
template <int N> struct WgmmaF16;
template <> struct WgmmaF16<128> {
    __device__ __forceinline__ static void mma(float* d, const uint32_t* a, uint64_t desc, int scale_d) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
    }
};

}  // namespace
}  // namespace fn2
