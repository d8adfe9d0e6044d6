// scan_common.cuh -- device helpers shared by the scan kernels (scan.cu, scan2.cu): named-barrier
// wrappers and the paired f32 arithmetic of the distance-table build.
#pragma once

#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int BAR_FULL = 1;    // named barriers 1..3: chunk buffer b is built
constexpr int BAR_EMPTY = 4;   // named barriers 4..6: chunk buffer b may be overwritten
constexpr int BAR_PROD = 7;    // named barrier 7: producer-only (residual chunk hand-over)

__device__ __forceinline__ void bar_sync(int id, int n)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int n)
{
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}

template <int DSUB>
__device__ __forceinline__ void load_vec(float *dst, const float *src)
{
    if constexpr (DSUB % 4 == 0) {
#pragma unroll
        for (int i = 0; i < DSUB / 4; i++) {
            float4 v = __ldg(reinterpret_cast<const float4 *>(src) + i);
            dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < DSUB; i++) dst[i] = __ldg(src + i);
    }
}

// ---- f32 pairs (even, odd) held in one 64-bit register pair.  sm_90 has no packed f32x2 arithmetic, so every
// op is two scalar IEEE round-to-nearest ops on the halves (the __f*_rn intrinsics are never contracted).  The
// square is fma(d, d, zero) with `zero` an opaque kernel argument: round(d*d + 0) == round(d*d), and nothing is
// left for the compiler to fold. ----
__device__ __forceinline__ uint64_t pk2(float a, float b)
{
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ void upk2(uint64_t v, float &a, float &b)
{
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ uint64_t sub2(uint64_t a, uint64_t b)
{
    float a0, a1, b0, b1;
    upk2(a, a0, a1); upk2(b, b0, b1);
    return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b)
{
    float a0, a1, b0, b1;
    upk2(a, a0, a1); upk2(b, b0, b1);
    return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t sq2(uint64_t d, uint64_t zero)
{
    float d0, d1, z0, z1;
    upk2(d, d0, d1); upk2(zero, z0, z1);
    return pk2(__fmaf_rn(d0, d0, z0), __fmaf_rn(d1, d1, z1));
}
// l2_once::<f32x8>: ((s0+s4)+(s2+s6)) + ((s1+s5)+(s3+s7)), s_k = (r_k-c_k)^2
__device__ __forceinline__ float l2_tree8_packed(const uint64_t r[4], const uint64_t c[4], uint64_t zero)
{
    uint64_t q01 = sq2(sub2(r[0], c[0]), zero), q23 = sq2(sub2(r[1], c[1]), zero);
    uint64_t q45 = sq2(sub2(r[2], c[2]), zero), q67 = sq2(sub2(r[3], c[3]), zero);
    uint64_t t01 = add2(q01, q45);     // (s0+s4, s1+s5)
    uint64_t t23 = add2(q23, q67);     // (s2+s6, s3+s7)
    uint64_t u = add2(t01, t23);       // ((s0+s4)+(s2+s6), (s1+s5)+(s3+s7))
    float u0, u1;
    upk2(u, u0, u1);
    return __fadd_rn(u0, u1);
}

// Four table entries (the 4 queries of a half against one codeword) level by level, so that every
// packed op has 3..15 independent neighbours instead of a 6-deep dependent chain per entry.
__device__ __forceinline__ float4 l2_tree8_packed_x4(const uint64_t (&r)[4][4], const uint64_t (&c)[4], uint64_t zero)
{
    uint64_t d[4][4];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) d[j][e] = sub2(r[j][e], c[e]);
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) d[j][e] = sq2(d[j][e], zero);
    uint64_t t[4][2];
#pragma unroll
    for (int j = 0; j < 4; j++) { t[j][0] = add2(d[j][0], d[j][2]); t[j][1] = add2(d[j][1], d[j][3]); }
    uint64_t u[4];
#pragma unroll
    for (int j = 0; j < 4; j++) u[j] = add2(t[j][0], t[j][1]);
    float lo[4], hi[4];
#pragma unroll
    for (int j = 0; j < 4; j++) upk2(u[j], lo[j], hi[j]);
    return make_float4(__fadd_rn(lo[0], hi[0]), __fadd_rn(lo[1], hi[1]), __fadd_rn(lo[2], hi[2]), __fadd_rn(lo[3], hi[3]));
}

}  // namespace

}  // namespace lgpu
