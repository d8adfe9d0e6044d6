// common.cuh -- shared helpers: error plumbing, the lance f32 arithmetic restated for
// device code (same rounding order as oracle/oracle.c), key encodings.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <utility>

#include "../../include/lancedb_b200.h"

namespace lgpu {

// ---- error plumbing -------------------------------------------------------------
void set_error(const std::string &msg);
struct Failure { int status; };

#define LGPU_CUDA(expr)                                                                   \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::lgpu::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));        \
            throw ::lgpu::Failure{_e == cudaErrorMemoryAllocation ? LGPU_OOM : LGPU_RUNTIME}; \
        }                                                                                 \
    } while (0)

#define LGPU_REQUIRE(cond, msg)                                                           \
    do {                                                                                  \
        if (!(cond)) { ::lgpu::set_error(msg); throw ::lgpu::Failure{LGPU_INVALID_INPUT}; } \
    } while (0)

// kernels launched by this process through the library (bench.py reports the count of its timed region)
void count_launches(uint64_t n);
#define LGPU_COUNT_LAUNCH() ::lgpu::count_launches(1)

// ---- programmatic dependent launch (PDL) -----------------------------------------
// A search step is ~25 launches, most of them a few microseconds long, and every kernel boundary costs a drain + launch
// gap of its own.  launch_k() launches with the programmatic-stream-
// serialization attribute and the kernels it is used for begin with pdl_entry(): they tell the scheduler that the NEXT
// grid may be brought onto the SMs already, then wait until the PREVIOUS grid has completed and flushed before touching
// memory.  Correctness needs nothing else: every kernel waits for its predecessor, which waited for its own.
// LGPU_NO_PDL=1 launches without the attribute (the device-side wait is then a no-op).
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_entry()
{
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
template <class... KArgs, class... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&...args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
    if (e != cudaSuccess) { set_error(std::string("kernel launch: ") + cudaGetErrorString(e)); throw Failure{LGPU_RUNTIME}; }
}
#endif

static inline uint32_t ceil_div(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
static inline uint64_t round_up64(uint64_t a, uint64_t b) { return (a + b - 1) / b * b; }

// ---- ordered float <-> uint32 key (ascending float order == ascending uint order) --
__host__ __device__ __forceinline__ uint32_t f32_key(float f)
{
#ifdef __CUDA_ARCH__
    uint32_t b = __float_as_uint(f);
#else
    uint32_t b; memcpy(&b, &f, 4);
#endif
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float key_f32(uint32_t k)
{
    uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    float f; memcpy(&f, &b, 4); return f;
#endif
}

#ifdef __CUDACC__
// ---- lance-linalg f32 kernels, restated with explicit round-to-nearest ops so nvcc
// can neither contract (a*b+c -> fma) nor reassociate.  Same order as oracle.c. ------

// l2_scalar::<f32,f32,16>: 16 lane accumulators, remainder first, then sequential sum.
__device__ __forceinline__ float lance_l2(const float *__restrict__ x, const float *__restrict__ y, int d)
{
    int nch = d >> 4, rem0 = nch << 4;
    float s = 0.f;
    for (int i = rem0; i < d; i++) { float df = __fsub_rn(x[i], y[i]); s = __fadd_rn(s, __fmul_rn(df, df)); }
    float sums[16];
#pragma unroll
    for (int l = 0; l < 16; l++) sums[l] = 0.f;
    for (int c = 0; c < nch; c++) {
#pragma unroll
        for (int l = 0; l < 16; l++) {
            float df = __fsub_rn(x[c * 16 + l], y[c * 16 + l]);
            sums[l] = __fadd_rn(sums[l], __fmul_rn(df, df));
        }
    }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, sums[l]);
    return __fadd_rn(s, t);
}

__device__ __forceinline__ float lance_dot(const float *__restrict__ x, const float *__restrict__ y, int d)
{
    int nch = d >> 4, rem0 = nch << 4;
    float s = 0.f;
    for (int i = rem0; i < d; i++) s = __fadd_rn(s, __fmul_rn(x[i], y[i]));
    float sums[16];
#pragma unroll
    for (int l = 0; l < 16; l++) sums[l] = 0.f;
    for (int c = 0; c < nch; c++) {
#pragma unroll
        for (int l = 0; l < 16; l++) sums[l] = __fadd_rn(sums[l], __fmul_rn(x[c * 16 + l], y[c * 16 + l]));
    }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, sums[l]);
    return __fadd_rn(s, t);
}

// f32x8::reduce_sum (AVX2): ((s0+s4)+(s2+s6)) + ((s1+s5)+(s3+s7))
__device__ __forceinline__ float reduce_sum_x8(const float *s)
{
    float t0 = __fadd_rn(s[0], s[4]), t1 = __fadd_rn(s[1], s[5]);
    float t2 = __fadd_rn(s[2], s[6]), t3 = __fadd_rn(s[3], s[7]);
    return __fadd_rn(__fadd_rn(t0, t2), __fadd_rn(t1, t3));
}

// the PQ sub-vector L2 (oracle.c::orc_l2_subvec): DSUB 8 / 16 use the l2_once tree
template <int DSUB>
__device__ __forceinline__ float subvec_l2(const float *r, const float *c)
{
    if (DSUB == 8) {
        float s[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { float d = __fsub_rn(r[i], c[i]); s[i] = __fmul_rn(d, d); }
        return reduce_sum_x8(s);
    } else if (DSUB == 16) {
        float s[16], h[8];
#pragma unroll
        for (int i = 0; i < 16; i++) { float d = __fsub_rn(r[i], c[i]); s[i] = __fmul_rn(d, d); }
#pragma unroll
        for (int i = 0; i < 8; i++) h[i] = __fadd_rn(s[i], s[i + 8]);
        return reduce_sum_x8(h);
    } else {
        return lance_l2(r, c, DSUB);
    }
}
template <int DSUB>
__device__ __forceinline__ float subvec_dot_dist(const float *q, const float *c)
{
    return __fsub_rn(1.0f, lance_dot(q, c, DSUB));
}
#endif  // __CUDACC__

}  // namespace lgpu
