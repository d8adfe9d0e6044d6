// tables.cu -- the filter + verify form of the PQ scan: per-query tables, per-row constants, proof and re-score.
//
// The exact path (scan2.cu) builds one 96 KB distance table per (query, probed partition), because lance's table
// is on the *residual* q - c_p (SURVEY.md 8a rows a4-a5): 20 480 tables per 1024-query batch, 23 f32 ops per
// entry, and that table build -- not the scan -- bounds the kernel.  Algebraically
//     |(q_i - c_i) - b_i|^2 = |q_i - b_i|^2  +  (|c_i|^2 - 2 q_i.c_i)  +  2 b_i.c_i
// so the distance of row r of partition p is  S_q(r) + A(q,p) + R(r)  with
//     S_q(r) = sum_i T_q[i][code_i(r)],  T_q[i][c] = |q_i - codebook_i[c]|^2    one table per QUERY
//     A(q,p) = |q - c_p|^2 - |q|^2                                               from the coarse step
//     R(r)   = 2 * sum_i codebook_i[code_i(r)] . c_p,i                           one f32 per row, at open
// (dot: T_q[i][c] = 1 - q_i.codebook_i[c], A = R = 0, distance = S - (m - 1): lance's own table, no residual).
// The rounding differs from lance's, so this is only used as a FILTER.  T_q is quantised to 16 bits against a
// per-query step (launch_query_tables_q16): the scan kernel (scan3.cu) adds the m integers of a row exactly and
// turns the sum into a LOWER bound L(r) of the row's distance; with W = m step the real distance lies in
// [L - E, L + W + E] (E = floating-point slack, launch_band_check3).  The caller keeps the kp rows with the
// smallest L; if L[kp-1] > L[k-1] + W + 2E no other row can be among the exact top-k, `pq_rescore_kernel`
// recomputes the kp rows exactly as oracle.c does (residual, f32x8 tree entries, sequential sum) and the final
// top-k is selected on those; queries that cannot be proven are redone by the exact kernels.  Final ids and
// distances are bit-identical to the exact path.
#include "kernels.cuh"

#include <math_constants.h>

namespace lgpu {

namespace {

// ---- table entries for the FILTER.  Not lance's arithmetic (that is pq_rescore_kernel's job): the expansion
//     |q_i - b|^2 = |q_i|^2 + |b|^2 - 2 q_i.b      (1 - q_i.b for dot)
// with |b|^2 precomputed at open and the dot product accumulated in two chains over (even, odd) dimension pairs.  Its
// rounding error, <= ~12 u (|q_i| + |b|)^2 per entry, is part of the band (band_check3: the 2 (|q|^2 + CB2) term).
// Both table passes call this one function, so they see identical values.
__device__ __forceinline__ uint64_t pack2(float a, float b)
{
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float sum2(uint64_t v)
{
    float a, b;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
    return a + b;
}
// (even, odd) lanes: a * b + c, each one fused multiply-add
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c)
{
    float a0, a1, b0, b1, c0, c1;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(a));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(b0), "=f"(b1) : "l"(b));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(c0), "=f"(c1) : "l"(c));
    return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
template <int DSUB>
struct SubVec {
    static constexpr int NP = (DSUB + 1) / 2;
    uint64_t p[NP];             // (even, odd) dimension pairs; an odd DSUB pads with 0
    __device__ __forceinline__ void load(const float *src)
    {
        if constexpr (DSUB % 4 == 0) {
            if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
                for (int i = 0; i < DSUB / 4; i++) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(src) + i);
                    p[2 * i] = pack2(v.x, v.y); p[2 * i + 1] = pack2(v.z, v.w);
                }
            } else {                                    // caller-owned query buffer that is not 16-byte aligned
#pragma unroll
                for (int i = 0; i < DSUB / 2; i++) p[i] = pack2(__ldg(src + 2 * i), __ldg(src + 2 * i + 1));
            }
        } else if constexpr (DSUB == 2) {
            const float2 v = __ldg(reinterpret_cast<const float2 *>(src));
            p[0] = pack2(v.x, v.y);
        } else {
            p[0] = pack2(__ldg(src), 0.f);
        }
    }
    __device__ __forceinline__ float dot(const SubVec &o) const
    {
        uint64_t acc = 0ull;
#pragma unroll
        for (int i = 0; i < NP; i++) acc = fma2(p[i], o.p[i], acc);
        return sum2(acc);
    }
};
template <int DSUB, bool DOT>
__device__ __forceinline__ float filter_entry(const SubVec<DSUB> &q, float qi2, const SubVec<DSUB> &cb, float cbn2)
{
    const float d = q.dot(cb);
    return DOT ? 1.0f - d : fmaf(-2.0f, d, qi2 + cbn2);
}

// thread mapping of both table passes: grid (ceil(B/32), nch), 256 threads; warp g = the 4 queries 32 bx + 4 g + j;
// lane = (s = lane & 7, cq = lane >> 3); step t handles code c = 4 t + cq.  The CTA first stages its codebook chunk
// (256 codes x 8 sub-spaces x DSUB floats, 64 KB at DSUB = 8) and the |b|^2 in shared memory -- read once from L2
// instead of once per warp, which was the kernels' bound (L1 sector throughput) -- and the quantiser collects 32 codes
// per query in a per-warp scratch so that its output leaves as full 16-byte stores.
constexpr int QT_NQ = 4;
template <int DSUB> struct QtSmem {
    static constexpr bool STAGE = DSUB <= 16;                       // DSUB = 32 would need 256 KB: read from L2 instead
    static constexpr size_t CB = STAGE ? (size_t)2048 * DSUB * 4 : 0;
    static constexpr size_t N2 = CB, SCRATCH = N2 + (STAGE ? 2048 * 4 : 0);
    static constexpr size_t TOTAL_MINMAX = SCRATCH, TOTAL_QUANT = SCRATCH + 8 * QT_NQ * 32 * 16;
};
template <int DSUB>
__device__ __forceinline__ void stage_chunk(const float *__restrict__ cb_tiled, const float *__restrict__ cb_n2, uint32_t ch,
                                            unsigned char *sm)
{
    if constexpr (QtSmem<DSUB>::STAGE) {
        // cp.async: every 16-byte request of the thread in flight at once (register copies waited for one L2 or DRAM
        // round trip per float4)
        const float4 *src = reinterpret_cast<const float4 *>(cb_tiled + (size_t)ch * 2048 * DSUB);
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(sm);
        for (int i = threadIdx.x; i < 2048 * DSUB / 4; i += 256)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16u * i), "l"(src + i) : "memory");
        const float4 *s2 = reinterpret_cast<const float4 *>(cb_n2 + (size_t)ch * 2048);
        const uint32_t d2 = dst + (uint32_t)QtSmem<DSUB>::N2;
        for (int i = threadIdx.x; i < 512; i += 256)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d2 + 16u * i), "l"(s2 + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
    }
}
template <int DSUB>
__device__ __forceinline__ void load_entry(SubVec<DSUB> &cv, float &cn, const float *__restrict__ cb_tiled,
                                           const float *__restrict__ cb_n2, uint32_t ch, uint32_t c, int s,
                                           const unsigned char *sm)
{
    if constexpr (QtSmem<DSUB>::STAGE) {
        const float *e = reinterpret_cast<const float *>(sm) + ((size_t)c * 8 + s) * DSUB;
        if constexpr (DSUB % 4 == 0) {
#pragma unroll
            for (int i = 0; i < DSUB / 4; i++) {
                const float4 v = reinterpret_cast<const float4 *>(e)[i];
                cv.p[2 * i] = pack2(v.x, v.y); cv.p[2 * i + 1] = pack2(v.z, v.w);
            }
        } else if constexpr (DSUB == 2) {
            const float2 v = *reinterpret_cast<const float2 *>(e);
            cv.p[0] = pack2(v.x, v.y);
        } else {
            cv.p[0] = pack2(e[0], 0.f);
        }
        cn = reinterpret_cast<const float *>(sm + QtSmem<DSUB>::N2)[c * 8 + s];
    } else {
        cv.load(cb_tiled + (((size_t)ch * 256 + c) * 8 + s) * DSUB);
        cn = __ldg(cb_n2 + ((size_t)ch * 256 + c) * 8 + s);
    }
}

// ---- pass 1: min_c / max_c of T_q[i][.] for every (query, sub-space)
template <int DSUB, bool DOT>
__global__ void __launch_bounds__(256) qtable_minmax_kernel(const float *__restrict__ Q, const float *__restrict__ cb_tiled,
                                                            const float *__restrict__ cb_n2, uint32_t B, uint32_t dim,
                                                            uint32_t m, uint32_t nch, float *__restrict__ mm)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(16) unsigned char qsm[];
    const uint32_t q0 = blockIdx.x * 32 + (threadIdx.x >> 5) * QT_NQ, ch = blockIdx.y;
    const int lane = threadIdx.x & 31, s = lane & 7, cq = lane >> 3;
    stage_chunk<DSUB>(cb_tiled, cb_n2, ch, qsm);
    if (q0 >= B) return;
    const uint32_t i = ch * 8 + s;
    float mn[QT_NQ], mx[QT_NQ];
    bool nan[QT_NQ];
#pragma unroll
    for (int j = 0; j < QT_NQ; j++) { mn[j] = 0.f; mx[j] = 0.f; nan[j] = false; }
    if (i < m) {
        SubVec<DSUB> qv[QT_NQ];
        float qi2[QT_NQ];
#pragma unroll
        for (int j = 0; j < QT_NQ; j++) {
            qv[j].load(Q + (size_t)min(q0 + j, B - 1) * dim + i * DSUB);
            qi2[j] = qv[j].dot(qv[j]);
            mn[j] = CUDART_INF_F; mx[j] = -CUDART_INF_F;
        }
#pragma unroll 2
        for (int t = 0; t < 64; t++) {
            SubVec<DSUB> cv;
            float cn;
            load_entry<DSUB>(cv, cn, cb_tiled, cb_n2, ch, 4 * t + cq, s, qsm);
#pragma unroll
            for (int j = 0; j < QT_NQ; j++) {
                const float v = filter_entry<DSUB, DOT>(qv[j], qi2[j], cv, cn);
                mn[j] = fminf(mn[j], v); mx[j] = fmaxf(mx[j], v);
                nan[j] |= v != v;                          // fminf / fmaxf drop NaN
            }
        }
    }
#pragma unroll
    for (int j = 0; j < QT_NQ; j++) {
        float a = nan[j] ? CUDART_NAN_F : mn[j], b = nan[j] ? CUDART_NAN_F : mx[j];
#pragma unroll
        for (int o = 8; o <= 16; o <<= 1) {
            const float on = __shfl_xor_sync(0xffffffffu, a, o), ox = __shfl_xor_sync(0xffffffffu, b, o);
            a = (on != on || a != a) ? CUDART_NAN_F : fminf(a, on);
            b = (ox != ox || b != b) ? CUDART_NAN_F : fmaxf(b, ox);
        }
        if (cq == 0 && q0 + j < B) reinterpret_cast<float2 *>(mm)[(size_t)(q0 + j) * nch * 8 + i] = make_float2(a, b);
    }
}

// ---- pass 2: quantise.  Position j of code c's 16-byte output holds sub-space (j + c) & 7 (the rotation scan3.cu's
// stagers rely on), i.e. sub-space s goes to position (s - c) & 7.
template <int DSUB, bool DOT>
__global__ void __launch_bounds__(256) qtable_quant_kernel(const float *__restrict__ Q, const float *__restrict__ cb_tiled,
                                                           const float *__restrict__ cb_n2, uint32_t B, uint32_t dim,
                                                           uint32_t m, uint32_t nch, const float *__restrict__ mm,
                                                           uint4 *__restrict__ qt, float *__restrict__ step_out,
                                                           float *__restrict__ base_out, float *__restrict__ sbound_out,
                                                           uint32_t *__restrict__ bad_out)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(16) unsigned char qsm[];
    const int wid = threadIdx.x >> 5;
    const uint32_t q0 = blockIdx.x * 32 + wid * QT_NQ, ch = blockIdx.y;
    const int lane = threadIdx.x & 31, s = lane & 7, cq = lane >> 3;
    stage_chunk<DSUB>(cb_tiled, cb_n2, ch, qsm);
    if (q0 >= B) return;
    unsigned short *scratch = reinterpret_cast<unsigned short *>(qsm + QtSmem<DSUB>::SCRATCH) + wid * (QT_NQ * 32 * 8);
    const uint32_t m8 = nch * 8;
    const float qmax = (float)(65535u / m);
    const uint32_t i = ch * 8 + s;
    float inv[QT_NQ], mn[QT_NQ];
    // per-query step / base / bound from the min-max table (every warp of the query's nch CTAs recomputes it)
#pragma unroll
    for (int j = 0; j < QT_NQ; j++) {
        const uint32_t q = min(q0 + j, B - 1);
        const float2 *row = reinterpret_cast<const float2 *>(mm) + (size_t)q * m8;
        float rng = 0.f, base = 0.f, sb = 0.f;
        bool bad = false;
        for (uint32_t ii = lane; ii < m; ii += 32) {
            const float2 v = row[ii];
            rng = fmaxf(rng, v.y - v.x);
            base += v.x;
            sb += fmaxf(fabsf(v.x), fabsf(v.y));
            bad |= !(fabsf(v.x) < CUDART_INF_F) || !(fabsf(v.y) < CUDART_INF_F);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            rng = fmaxf(rng, __shfl_xor_sync(0xffffffffu, rng, o));
            base += __shfl_xor_sync(0xffffffffu, base, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        bad = __any_sync(0xffffffffu, bad) || !(rng < CUDART_INF_F) || !(fabsf(base) < CUDART_INF_F) || !(sb < CUDART_INF_F);
        float step = (!bad && rng > 0.f) ? rng / qmax : 0.f;
        float iv = (step > 0.f && qmax / rng < CUDART_INF_F) ? qmax / rng : 0.f;
        if (rng > 0.f && iv == 0.f) bad = true;         // a range too small to invert: take the exact path
        if (bad) { step = 0.f; iv = 0.f; }
        if (ch == 0 && lane == 0 && q0 + j < B) {
            step_out[q] = step;
            bad_out[q] = bad ? 1u : 0u;
            base_out[q] = DOT ? base - (float)(m - 1) : base;
            sbound_out[q] = sb;
        }
        inv[j] = iv;
        mn[j] = i < m ? row[i].x : 0.f;
    }
    SubVec<DSUB> qv[QT_NQ];
    float qi2[QT_NQ];
#pragma unroll
    for (int j = 0; j < QT_NQ; j++) {
        if (i < m) qv[j].load(Q + (size_t)min(q0 + j, B - 1) * dim + i * DSUB);
        else { for (int e = 0; e < SubVec<DSUB>::NP; e++) qv[j].p[e] = 0ull; }
        qi2[j] = qv[j].dot(qv[j]);
    }
    const size_t qstride = (size_t)nch * 256;                           // uint4 per query
    uint4 *out0 = qt + ((size_t)q0 * nch + ch) * 256;
    for (int t8 = 0; t8 < 8; t8++) {                                    // 32 codes at a time
#pragma unroll 2
        for (int tt = 0; tt < 8; tt++) {
            const int t = t8 * 8 + tt;
            const uint32_t c = 4 * t + cq;
            SubVec<DSUB> cv;
            float cn;
            load_entry<DSUB>(cv, cn, cb_tiled, cb_n2, ch, c, s, qsm);
            const uint32_t at = (4 * tt + cq) * 8 + ((s - c) & 7);
#pragma unroll
            for (int j = 0; j < QT_NQ; j++) {
                const float v = filter_entry<DSUB, DOT>(qv[j], qi2[j], cv, cn);
                float x = (v - mn[j]) * inv[j];
                x = (x >= 0.f && i < m) ? fminf(floorf(x), qmax) : 0.f;  // NaN -> 0 (flagged bad); padding sub-space -> 0
                scratch[j * 256 + at] = (unsigned short)x;
            }
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < QT_NQ; j++)
            if (q0 + j < B)
                out0[j * qstride + t8 * 32 + lane] = reinterpret_cast<const uint4 *>(scratch + j * 256)[lane];
        __syncwarp();
    }
}

// |b|^2 of every tiled codebook entry (open time), same pairing as SubVec::dot
template <int DSUB>
__global__ void cb_norms_kernel(const float *__restrict__ cb_tiled, uint64_t n, float *__restrict__ out)
{
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    SubVec<DSUB> v;
    v.load(cb_tiled + e * DSUB);
    out[e] = v.dot(v);
}

// DSUB floats from global memory; 16-byte loads when DSUB is a multiple of 4 and the address allows it
template <int DSUB>
__device__ __forceinline__ void load_cb(float *dst, const float *src)
{
    if constexpr (DSUB % 4 == 0) {
        if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
            for (int i = 0; i < DSUB / 4; i++) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(src) + i);
                dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
            }
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < DSUB; i++) dst[i] = __ldg(src + i);
}

// same with generic (global or shared) loads: the finalize kernel keeps the query in shared memory
template <int DSUB>
__device__ __forceinline__ void load_any(float *dst, const float *src)
{
    if constexpr (DSUB % 4 == 0) {
        if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
            for (int i = 0; i < DSUB / 4; i++) {
                const float4 v = reinterpret_cast<const float4 *>(src)[i];
                dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
            }
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < DSUB; i++) dst[i] = src[i];
}

__device__ __forceinline__ uint32_t find_partition(const uint64_t *__restrict__ part_off, uint32_t nlist, uint64_t pos)
{
    uint32_t lo = 0, hi = nlist - 1;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (part_off[mid + 1] > pos) hi = mid; else lo = mid + 1;
    }
    return lo;
}
__device__ __forceinline__ uint32_t stream_code(const unsigned char *__restrict__ codes, uint64_t base, uint32_t npad,
                                                uint32_t row, uint32_t i)
{
    const uint32_t M = i + (row & 7);                   // position in the row's skewed byte stream (retile.cu)
    return codes[base + ((uint64_t)(M >> 3) * npad + row) * 8 + (M & 7)];
}

// R[pos] = 2 * sum_i codebook_i[code_i] . c_p,i ; rmax = max |R| (as int bits)
template <int DSUB>
__global__ void row_const_kernel(const unsigned char *__restrict__ codes, const uint64_t *__restrict__ code_base,
                                 const uint32_t *__restrict__ part_npad, const uint64_t *__restrict__ part_off,
                                 uint32_t nlist, uint64_t nrows, const float *__restrict__ centroids,
                                 const float *__restrict__ cb_tiled, uint32_t dim, uint32_t m, float *__restrict__ R,
                                 int *__restrict__ rmax_bits)
{
    const uint64_t pos = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= nrows) return;
    const uint32_t p = find_partition(part_off, nlist, pos);
    const uint32_t row = (uint32_t)(pos - part_off[p]);
    const float *cen = centroids + (size_t)p * dim;
    double acc = 0.0;                                   // f64: keeps R within 1 ulp(f32) of the real value
    for (uint32_t i = 0; i < m; i++) {
        const uint32_t c = stream_code(codes, code_base[p], part_npad[p], row, i);
        const float *cb = cb_tiled + (((size_t)(i >> 3) * 256 + c) * 8 + (i & 7)) * DSUB;
#pragma unroll
        for (int t = 0; t < DSUB; t++) acc = fma((double)cb[t], (double)cen[i * DSUB + t], acc);
    }
    const float r = (float)(2.0 * acc);
    R[pos] = r;
    atomicMax(rmax_bits, __float_as_int(fabsf(r)));
}

// exact PQ distance of one (query, stored row) pair, exactly as oracle.c::partition_distances:
// residual -> sub-vector table entry (l2_once tree for dsub 8/16) -> sequential f32 sum -> metric scale.
// Warp-cooperative: lane l evaluates the entries of sub-spaces l, l + 32, ... (independent loads of the code byte,
// the codeword and the query / centroid sub-vectors), then the entries are summed in order i = 0..m-1 (the oracle's
// order) by walking them through a shuffle.  m <= 512.  Every lane returns the distance.
template <int DSUB>
__device__ __forceinline__ float exact_pq_distance_warp(const float *qv, const float *__restrict__ cen,
                                                        const unsigned char *__restrict__ codes, uint64_t cbase,
                                                        uint32_t npad, uint32_t row, const float *__restrict__ cb_tiled,
                                                        uint32_t m, int metric, int lane)
{
    float tv[16];
#pragma unroll
    for (int it = 0; it < 16; it++) tv[it] = 0.f;
    // U sub-spaces per lane at a time, in three phases (code bytes -> operands -> arithmetic) so that the loads of a
    // phase are all in flight together: interleaved, ptxas serialised them into one L2 round trip after the other.
    // U = 3 covers m = 96 in one block at DSUB <= 8; longer sub-vectors keep the register count down with U = 1.
    constexpr int U = DSUB <= 8 ? 3 : 1;
#pragma unroll
    for (int blk = 0; blk * U < 16; blk++) {
        if ((uint32_t)blk * U * 32 < m) {
            uint32_t c[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const uint32_t i = (uint32_t)(blk * U + u) * 32 + lane;
                c[u] = i < m ? stream_code(codes, cbase, npad, row, i) : 0u;
            }
            float cv[U][DSUB], qq[U][DSUB], cc[U][DSUB];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const uint32_t i = min((uint32_t)(blk * U + u) * 32 + lane, m - 1);
                load_cb<DSUB>(cv[u], cb_tiled + (((size_t)(i >> 3) * 256 + c[u]) * 8 + (i & 7)) * DSUB);
                load_any<DSUB>(qq[u], qv + i * DSUB);
                if (metric != LGPU_DOT) load_cb<DSUB>(cc[u], cen + i * DSUB);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (blk * U + u < 16) {
                    const uint32_t i = (uint32_t)(blk * U + u) * 32 + lane;
                    float r[DSUB];
#pragma unroll
                    for (int t = 0; t < DSUB; t++) r[t] = (metric == LGPU_DOT) ? qq[u][t] : __fsub_rn(qq[u][t], cc[u][t]);
                    const float e = (metric == LGPU_DOT) ? subvec_dot_dist<DSUB>(r, cv[u]) : subvec_l2<DSUB>(r, cv[u]);
                    tv[blk * U + u] = i < m ? e : 0.f;
                }
            }
        }
    }
    float acc = 0.f;
#pragma unroll
    for (int it = 0; it < 16; it++) {
        if ((uint32_t)it * 32 < m) {
            const uint32_t lim = min(32u, m - (uint32_t)it * 32);
            if (lim == 32u) {
                // full group: unrolled, so the 32 shuffles issue back to back ahead of the dependent adds (rolled, every
                // add waited for its own shuffle: ~30 cycles x m per row, a third of the re-score kernel at k = 100)
#pragma unroll
                for (int l = 0; l < 32; l++) acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, tv[it], l));
            } else {
                for (uint32_t l = 0; l < lim; l++) acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, tv[it], (int)l));
            }
        }
    }
    if (metric == LGPU_COSINE) acc = __fmul_rn(acc, 0.5f);
    else if (metric == LGPU_DOT) acc = __fsub_rn(acc, (float)(m - 1));
    return acc;
}

// one warp per (query, candidate position) pair
template <int DSUB>
__global__ void __launch_bounds__(256, 2) pq_rescore_kernel(const float *__restrict__ Q, const uint64_t *__restrict__ pos,
                                                         uint32_t B, uint32_t nc, const unsigned char *__restrict__ codes,
                                                         const uint64_t *__restrict__ code_base,
                                                         const uint32_t *__restrict__ part_npad,
                                                         const uint64_t *__restrict__ part_off, uint32_t nlist,
                                                         const float *__restrict__ centroids,
                                                         const float *__restrict__ cb_tiled, uint32_t dim, uint32_t m,
                                                         int metric, const uint32_t *__restrict__ ncols_q,
                                                         float *__restrict__ out)
{
    const uint64_t pair = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pair >= (uint64_t)B * nc) return;
    const uint32_t q = (uint32_t)(pair / nc);
    if (ncols_q && (uint32_t)(pair - (uint64_t)q * nc) >= ncols_q[q]) return;      // beyond the query's proven prefix
    const uint64_t ps = pos[pair];
    if (ps == UINT64_MAX) { if (lane == 0) out[pair] = CUDART_INF_F; return; }
    const uint32_t p = find_partition(part_off, nlist, ps);
    const uint32_t row = (uint32_t)(ps - part_off[p]);
    const float d = exact_pq_distance_warp<DSUB>(Q + (size_t)q * dim, centroids + (size_t)p * dim, codes, code_base[p],
                                                 part_npad[p], row, cb_tiled, m, metric, lane);
    if (lane == 0) out[pair] = d;
}

// ---- candidate mode of the filter scan: per-query band, then the final exact top-k over the survivors ----
__global__ void cand_prepare_kernel(const float *__restrict__ step, const float *__restrict__ sbound,
                                    const float *__restrict__ amax, const int *__restrict__ rmax_bits,
                                    const float *__restrict__ qn2, float cb2, float scale, uint32_t m, bool dot,
                                    uint32_t B, float *__restrict__ slack, uint32_t *__restrict__ thr,
                                    uint32_t *__restrict__ cand_cnt, uint32_t *__restrict__ cand_last)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    const ScanBand bd = scan_band(step[q], sbound[q], amax ? amax[q] : 0.f, rmax_bits ? __int_as_float(*rmax_bits) : 0.f,
                                  qn2[q], cb2, m, dot);
    slack[q] = scale * (bd.W + 2.0f * bd.E);
    thr[q] = CAND_NO_THR;
    cand_cnt[q] = 0u;
    cand_last[q] = 0u;
}

// ---- candidate mode, after the scan.  Three fully parallel kernels instead of one latency chain per query:
//   cand_filter_kernel   one warp per query: the k-th smallest lower bound of the query's candidates (the tightest
//                        threshold this family of bounds allows: every row with L <= tau is in the list and the list
//                        holds k of them) -> the survivors L <= L_(k) + slack go to a batch-wide work list;
//   cand_rescore_kernel  persistent warps over the work list: exact distance (oracle arithmetic), row id, position;
//   launch_select        mode 2 over each query's survivors: the k best by (_distance, _rowid).
constexpr int FLT_THREADS = 128;
template <int PER>                                           // candidates per lane: cand_cap <= 32 * PER
__global__ void __launch_bounds__(FLT_THREADS) cand_filter_kernel(FinalizeArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint32_t q = (blockIdx.x * FLT_THREADS + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= a.B) return;
    const uint32_t total = a.cand_cnt[q];
    const uint32_t n = min(total, a.cand_cap);
    const bool flagged = total > a.cand_cap || a.bad[q];
    const uint32_t *ckey = a.cand_key + (size_t)q * a.cand_cap;
    uint32_t key[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const uint32_t i = (uint32_t)j * 32 + lane;
        key[j] = i < n ? __ldcg(ckey + i) : 0xffffffffu;
    }
    const uint32_t tkey = a.thr[q];
    float tau = tkey == CAND_NO_THR ? CUDART_INF_F : key_f32(tkey);
    if (n >= a.k && !flagged) {
        uint32_t kth = 0;                                   // largest v with count(key < v) < k  ==  k-th smallest key
#pragma unroll 1
        for (int bit = 31; bit >= 0; bit--) {
            const uint32_t probe = kth | (1u << bit);
            uint32_t c = 0;
#pragma unroll
            for (int j = 0; j < PER; j++) c += key[j] < probe ? 1u : 0u;
            c = __reduce_add_sync(0xffffffffu, c);
            if (c < a.k) kth = probe;
        }
        tau = fminf(tau, key_f32(kth));
    }
    const float lim = tau + a.slack[q];
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) mine += ((uint32_t)j * 32 + lane < n && key_f32(key[j]) <= lim) ? 1u : 0u;
    uint32_t pre = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += t; }
    const uint32_t cnt = __shfl_sync(0xffffffffu, pre, 31);
    uint32_t base = 0;
    if (lane == 31 && cnt) base = atomicAdd(a.work_cnt, cnt);
    base = __shfl_sync(0xffffffffu, base, 31);
    uint32_t at = pre - mine;
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const uint32_t i = (uint32_t)j * 32 + lane;
        if (i < n && key_f32(key[j]) <= lim) { a.work[base + at] = make_uint2(q, (i << 16) | at); at++; }
    }
    if (lane == 0) {
        a.surv_cnt[q] = cnt;
        a.flags[q] = flagged ? 1u : 0u;
        if (flagged) a.work_cnt[1] = 1u;                    // opens the gate of the exact fix-up pass
        if (a.stats) {
            atomicAdd(a.stats + 0, (unsigned long long)total); atomicAdd(a.stats + 1, (unsigned long long)cnt);
            atomicAdd(a.stats + 2, (unsigned long long)(flagged ? 1 : 0)); atomicAdd(a.stats + 3, 1ull);
        }
    }
}

constexpr int RSC_THREADS = 256;
template <int DSUB>
__global__ void __launch_bounds__(RSC_THREADS, 2) cand_rescore_kernel(FinalizeArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const int lane = threadIdx.x & 31;
    const uint32_t total = *a.work_cnt;
    const uint32_t nwarps = gridDim.x * (RSC_THREADS / 32);
    for (uint32_t it = blockIdx.x * (RSC_THREADS / 32) + (threadIdx.x >> 5); it < total; it += nwarps) {
        const uint2 wk = a.work[it];
        const uint32_t q = wk.x, ci = wk.y >> 16, slot = wk.y & 0xffffu;
        const CandRec rec = a.cand[(size_t)q * a.cand_cap + ci];
        float d = exact_pq_distance_warp<DSUB>(a.Q + (size_t)q * a.dim, a.centroids + (size_t)rec.p * a.dim, a.codes,
                                               a.code_base[rec.p], a.part_npad[rec.p], rec.row, a.cb_tiled, a.m, a.metric,
                                               lane);
        if (lane == 0) {
            const uint64_t ps = a.part_off[rec.p] + rec.row;
            const size_t o = (size_t)q * a.cand_cap + slot;
            a.ex_dist[o] = d; a.ex_id[o] = a.row_ids[ps]; a.ex_pos[o] = ps;
        }
    }
}

// probe_A[slot] = coarse_dist - |q|^2 ; amax[q] = max_j coarse + |q|^2
// bad[q] |= |q|^2, amax or some base + A not finite (|q|^2 above FLT_MAX with finite coarse distances makes A = -inf:
// every L would be -inf and the candidate mode's limit tau + slack NaN)
__global__ void probe_terms_kernel(const float *__restrict__ probe_dist, const float *__restrict__ Q, uint32_t B,
                                   uint32_t nprobes, uint32_t dim, float *__restrict__ probe_A,
                                   float *__restrict__ amax, float *__restrict__ qn2, const float *__restrict__ base,
                                   uint32_t *__restrict__ bad)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;    // one warp per query
    const int lane = threadIdx.x & 31;
    if (q >= B) return;
    double n2d = 0.0;                                   // f64: |q|^2 within 1 ulp(f32)
    for (uint32_t t = lane; t < dim; t += 32) { double v = Q[(size_t)q * dim + t]; n2d = fma(v, v, n2d); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n2d += __shfl_xor_sync(0xffffffffu, n2d, o);
    const float n2 = (float)n2d;
    float mx = 0.f;
    bool inf = false;
    if (probe_A) {                                       // (dot: no residual, A = 0)
        const float b = base[q];
        for (uint32_t j = lane; j < nprobes; j += 32) {
            const float cd = probe_dist[(size_t)q * nprobes + j];
            const float A = cd - n2;
            probe_A[(size_t)q * nprobes + j] = A;
            mx = fmaxf(mx, fabsf(cd));
            inf |= !(fabsf(b + A) < CUDART_INF_F);      // the same sum as scan3's epilogue
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    inf = __any_sync(0xffffffffu, inf);
    if (lane == 0) {
        qn2[q] = n2;
        const float am = mx + n2;                       // >= |A| and also covers the coarse distance's own rounding
        if (amax) amax[q] = am;
        if (inf || !(n2 < CUDART_INF_F) || !(am < CUDART_INF_F)) bad[q] = 1u;
    }
}

// flags[q] = 1 when the shortlist cannot be proven to contain the exact top-k (see the header and kernels.cuh).
// Error budget of scan_band (kernels.cuh), u = 2^-24, mag = sbound + amax + rmax + 2 (|q|^2 + CB2),
// CB2 = sum_i max_c |codebook_i[c]|^2.  In the normal range every f32 operation errs by <= u of its result:
//   - the exact (oracle-order) distance d* differs from the real-arithmetic distance D of the same f32 inputs by
//     <= (m + 16) u (D + |q - c_p|^2) <= 2 (m + 16) u mag: m - 1 sequential sums, <= log2(dsub) + 2 per entry;
//   - a table entry (filter_entry) errs by <= (dsub / 2 + 2) u |q_i| |b| in its dot chain (dsub / 2 FMAs per lane, up to
//     16 at dsub 32), as much in |q_i|^2 and in |b|^2, and u |T| in the final FMA: <= (dsub + 6) u (|q_i|^2 + |b|^2) +
//     u |T|, summed over i <= 38 u (|q|^2 + CB2) + u sbound at dsub 32.  The entry's error enters L once through the
//     entry itself and once through min_i (base): twice that;
//   - the quantiser's floor can be off by one step when (T - min) / step lands within 2^-11 of an integer, and step is
//     rounded: both are absorbed by the factor 1 + 2^-10 on W (not by E);
//   - A carries <= 70 u (coarse + |q|^2) <= 70 u amax, R one ulp of rmax, the epilogue of scan3 (fmaf, + R) two more
//     roundings of values bounded by sbound + amax + rmax;
//   so for m <= 96: <= (224 + 2 + 70 + 1 + 2) u mag + 76 u (|q|^2 + CB2) < 2^9 u mag = 2^-15 mag.  For m > 96 only the
//   first term grows, and (m + 16) <= 112 ceil(m/96): ceil(m/96) times the budget covers it.
// dot: T = 1 - q_i.b has an absolute 1 per entry, whose rounding is not proportional to |q_i||b|: m more in mag.
// Subnormal range: products, FMAs, quotients and conversions that underflow err by an absolute <= 2^-150 on top
// (additions and subtractions are exact there).  Per row: 3 dsub + 1 per table entry, twice (entry and min), dsub per
// oracle entry, dim for each of the two coarse computations, 65535 through step * S, a few in the epilogue: below
// 2^18 x 2^-150 = 2^-132 for dim <= 16384 (m <= 512, dsub <= 32).  The floor 2^-126 covers it with a margin of 64;
// it vanishes in the rounding of E once 2^-15 mag >= 2^-101, so E is homogeneous of degree 2 in the data there.
__global__ void band_check3_kernel(const float *__restrict__ lb, const uint32_t *__restrict__ cnt,
                                   const float *__restrict__ step, const float *__restrict__ sbound,
                                   const float *__restrict__ amax, const int *__restrict__ rmax_bits,
                                   const uint32_t *__restrict__ bad, const float *__restrict__ qn2, float cb2, float scale,
                                   uint32_t m, bool dot, uint32_t B, uint32_t k, uint32_t kp, uint32_t *__restrict__ flags,
                                   uint32_t *__restrict__ gate, uint32_t *__restrict__ surv)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    uint32_t f = bad[q] ? 1u : 0u;
    const ScanBand bd = scan_band(step[q], sbound[q], amax ? amax[q] : 0.f, rmax_bits ? __int_as_float(*rmax_bits) : 0.f,
                                  qn2[q], cb2, m, dot);
    const float slack = scale * (bd.W + 2.0f * bd.E);
    if (surv) {
        // the rows that can still be among the exact top-k: the ascending prefix with L <= L_(k) + scale (W + 2E)
        const uint32_t n = min(cnt[q], kp);
        uint32_t pre = n;
        if (n > k && !f) {
            const float lim = lb[(size_t)q * kp + k - 1] + slack;
            pre = k;
            while (pre < n && !(lb[(size_t)q * kp + pre] > lim)) pre++;
        }
        surv[q] = pre;
    }
    if (!f && cnt[q] >= kp && kp > 0) {
        const float kth = lb[(size_t)q * kp + (k - 1 < kp ? k - 1 : kp - 1)];
        const float last = lb[(size_t)q * kp + kp - 1];
        f = (k >= kp || !(last > kth + slack)) ? 1u : 0u;
    }
    flags[q] = f;
    if (f && gate) *gate = 1u;                              // opens the gate of the exact fix-up pass
}

__global__ void scan_band_kernel(const float *__restrict__ step, const float *__restrict__ sbound,
                                 const float *__restrict__ amax, const int *__restrict__ rmax_bits,
                                 const float *__restrict__ qn2, float cb2, uint32_t m, bool dot, uint32_t B,
                                 float *__restrict__ W, float *__restrict__ E)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    const ScanBand bd = scan_band(step[q], sbound[q], amax ? amax[q] : 0.f, rmax_bits ? __int_as_float(*rmax_bits) : 0.f,
                                  qn2[q], cb2, m, dot);
    W[q] = bd.W;
    E[q] = bd.E;
}

template <class F> void dispatch_dsub(uint32_t dsub, F &&f)
{
    switch (dsub) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 4: f(std::integral_constant<int, 4>{}); break;
    case 8: f(std::integral_constant<int, 8>{}); break;
    case 16: f(std::integral_constant<int, 16>{}); break;
    case 32: f(std::integral_constant<int, 32>{}); break;
    default: set_error("unsupported PQ sub-vector length"); throw Failure{LGPU_INVALID_INPUT};
    }
}

}  // namespace

void launch_query_tables_q16(const float *Q, const float *cb_tiled, const float *cb_n2, uint32_t B, uint32_t dim,
                             uint32_t m, uint32_t nch, uint32_t dsub, int metric, float *mm, uint4 *qt, float *step,
                             float *base, float *sbound, uint32_t *bad, cudaStream_t st)
{
    if (B == 0) return;
    const dim3 grid((B + 31) / 32, nch);
    dispatch_dsub(dsub, [&](auto D) {
        constexpr int DS = decltype(D)::value;
        constexpr size_t s1 = QtSmem<DS>::TOTAL_MINMAX, s2 = QtSmem<DS>::TOTAL_QUANT;
        auto run = [&](auto k1, auto k2) {
            LGPU_CUDA(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s1));
            LGPU_CUDA(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s2));
            launch_k(k1, grid, dim3(256), s1, st, Q, cb_tiled, cb_n2, B, dim, m, nch, mm); LGPU_COUNT_LAUNCH();
            launch_k(k2, grid, dim3(256), s2, st, Q, cb_tiled, cb_n2, B, dim, m, nch, mm, qt, step, base, sbound, bad); LGPU_COUNT_LAUNCH();
        };
        if (metric == LGPU_DOT) run(qtable_minmax_kernel<DS, true>, qtable_quant_kernel<DS, true>);
        else run(qtable_minmax_kernel<DS, false>, qtable_quant_kernel<DS, false>);
    });
    LGPU_CUDA(cudaGetLastError());
}

void launch_cb_norms(const float *cb_tiled, uint32_t nch, uint32_t dsub, float *out, cudaStream_t st)
{
    const uint64_t n = (uint64_t)nch * 256 * 8;
    dispatch_dsub(dsub, [&](auto D) {
        cb_norms_kernel<decltype(D)::value><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cb_tiled, n, out); LGPU_COUNT_LAUNCH();
    });
    LGPU_CUDA(cudaGetLastError());
}

void launch_row_const(const unsigned char *codes, const uint64_t *code_base, const uint32_t *part_npad,
                      const uint64_t *part_off, uint32_t nlist, uint64_t nrows, const float *centroids,
                      const float *cb_tiled, uint32_t dim, uint32_t m, uint32_t dsub, float *R, int *rmax_bits,
                      cudaStream_t st)
{
    LGPU_CUDA(cudaMemsetAsync(rmax_bits, 0, sizeof(int), st));
    if (nrows == 0) return;
    dispatch_dsub(dsub, [&](auto D) {
        row_const_kernel<decltype(D)::value><<<(unsigned)((nrows + 255) / 256), 256, 0, st>>>(
            codes, code_base, part_npad, part_off, nlist, nrows, centroids, cb_tiled, dim, m, R, rmax_bits); LGPU_COUNT_LAUNCH();
    });
    LGPU_CUDA(cudaGetLastError());
}

void launch_pq_rescore(const float *Q, const uint64_t *pos, uint32_t B, uint32_t nc, const unsigned char *codes,
                       const uint64_t *code_base, const uint32_t *part_npad, const uint64_t *part_off, uint32_t nlist,
                       const float *centroids, const float *cb_tiled, uint32_t dim, uint32_t m, uint32_t dsub, int metric,
                       const uint32_t *ncols_q, float *out, cudaStream_t st)
{
    if (B == 0 || nc == 0) return;
    if (m > 512) { set_error("internal: pq_rescore supports m <= 512"); throw Failure{LGPU_RUNTIME}; }
    const uint64_t total = (uint64_t)B * nc * 32;              // one warp per pair
    dispatch_dsub(dsub, [&](auto D) {
        pq_rescore_kernel<decltype(D)::value><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            Q, pos, B, nc, codes, code_base, part_npad, part_off, nlist, centroids, cb_tiled, dim, m, metric, ncols_q, out); LGPU_COUNT_LAUNCH();
    });
    LGPU_CUDA(cudaGetLastError());
}

void launch_probe_terms(const float *probe_dist, const float *Q, uint32_t B, uint32_t nprobes, uint32_t dim,
                        float *probe_A, float *amax, float *qn2, const float *base, uint32_t *bad, cudaStream_t st)
{
    if (B == 0) return;
    launch_k(probe_terms_kernel, dim3((B * 32 + 255) / 256), dim3(256), 0, st, probe_dist, Q, B, nprobes, dim, probe_A, amax, qn2,
             base, bad); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_cand_prepare(const float *step, const float *sbound, const float *amax, const int *rmax_bits, const float *qn2,
                         float cb2, float scale, uint32_t m, bool dot, uint32_t B, float *slack, uint32_t *thr,
                         uint32_t *cand_cnt, uint32_t *cand_last, uint32_t *cand_key, uint32_t cand_cap, cudaStream_t st)
{
    if (B == 0) return;
    LGPU_CUDA(cudaMemsetAsync(cand_key, 0xff, (size_t)B * cand_cap * 4, st));
    launch_k(cand_prepare_kernel, dim3((B + 127) / 128), dim3(128), 0, st, step, sbound, amax, rmax_bits, qn2, cb2, scale, m, dot, B, slack, thr, cand_cnt, cand_last); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_cand_finalize(const FinalizeArgs &a, cudaStream_t st)
{
    if (a.B == 0) return;
    if (a.m > 512 || a.cand_cap < 32 || a.cand_cap > CAND_CAP_MAX || (a.cand_cap & (a.cand_cap - 1)) || a.k > a.cand_cap) {
        set_error("internal: cand_finalize needs m <= 512 and a power-of-two candidate capacity in [32, 2048] >= k");
        throw Failure{LGPU_RUNTIME};
    }
    LGPU_CUDA(cudaMemsetAsync(a.work_cnt, 0, 8, st));       // survivor counter + fix-up gate
    const unsigned fgrid = (a.B * 32 + FLT_THREADS - 1) / FLT_THREADS;
    if (a.cand_cap <= 512) { launch_k(cand_filter_kernel<16>, dim3(fgrid), dim3(FLT_THREADS), 0, st, a); LGPU_COUNT_LAUNCH(); }
    else if (a.cand_cap <= 1024) { launch_k(cand_filter_kernel<32>, dim3(fgrid), dim3(FLT_THREADS), 0, st, a); LGPU_COUNT_LAUNCH(); }
    else { launch_k(cand_filter_kernel<64>, dim3(fgrid), dim3(FLT_THREADS), 0, st, a); LGPU_COUNT_LAUNCH(); }
    dispatch_dsub(a.dsub, [&](auto D) {
        launch_k(cand_rescore_kernel<decltype(D)::value>, dim3(a.num_sms * 4), dim3(RSC_THREADS), 0, st, a); LGPU_COUNT_LAUNCH();
    });
    SelectArgs sb{};
    sb.mode = 2; sb.dense = a.ex_dist; sb.cand_ids = a.ex_id; sb.cand_pos = a.ex_pos; sb.ncols_q = a.surv_cnt;
    sb.ncols = a.cand_cap; sb.inner = a.cand_cap; sb.row_stride = a.cand_cap; sb.outer_stride = 0;
    sb.B = a.B; sb.k = a.k; sb.out_ids = a.out_ids; sb.out_dist = a.out_dist; sb.out_count = a.out_count;
    sb.out_pos = a.out_pos;
    launch_select(sb, st);
    LGPU_CUDA(cudaGetLastError());
}

void launch_scan_band(const float *step, const float *sbound, const float *amax, const int *rmax_bits, const float *qn2,
                      float cb2, uint32_t m, bool dot, uint32_t B, float *W, float *E, cudaStream_t st)
{
    if (B == 0) return;
    scan_band_kernel<<<(B + 127) / 128, 128, 0, st>>>(step, sbound, amax, rmax_bits, qn2, cb2, m, dot, B, W, E); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_band_check3(const float *lb, const uint32_t *cnt, const float *step, const float *sbound, const float *amax,
                        const int *rmax_bits, const uint32_t *bad, const float *qn2, float cb2, float scale, uint32_t m,
                        bool dot, uint32_t B, uint32_t k, uint32_t kp, uint32_t *flags, uint32_t *gate, uint32_t *surv,
                        cudaStream_t st)
{
    if (B == 0) return;
    if (gate) LGPU_CUDA(cudaMemsetAsync(gate, 0, 4, st));
    band_check3_kernel<<<(B + 127) / 128, 128, 0, st>>>(lb, cnt, step, sbound, amax, rmax_bits, bad, qn2, cb2, scale, m, dot, B, k, kp, flags, gate, surv); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
