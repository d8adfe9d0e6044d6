// dist.cu -- exact f32 distance kernels in lance's rounding order.
//
// K1 (coarse): IvfModel::find_partitions computes dist(q, every centroid) with
// lance-linalg's l2 / dot [lance, recalled; SURVEY.md 8a row a3].  l2_scalar::<f32,16>
// keeps 16 lane accumulators (lane l sums dims l, l+16, ...) and then adds the 16
// lane sums sequentially; to be bit-identical the kernel keeps exactly that structure:
// the 16 K-lanes are 16 threads, every thread register-tiles 4 queries x 8 centroids
// for its lane, and one thread per (query, centroid) pair adds the 16 lane sums in order.
// The same kernel is the exact flat KNNVectorDistance (SURVEY.md 8a row a11) and
// `launch_pair_distance` is the exact re-rank used by refine_factor (row a10).
#include "kernels.cuh"

#include <math_constants.h>

#include <algorithm>

namespace lgpu {

namespace {

constexpr int DM_Q = 16, DM_C = 32, DM_KT = 32, DM_STR = 36, DM_THREADS = 256;

__global__ void __launch_bounds__(DM_THREADS) dist_matrix_kernel(
    const float *__restrict__ Q, const float *__restrict__ C, uint32_t B, uint64_t N, uint32_t d, int mode,
    const float *__restrict__ xnorm, const float *__restrict__ ysqrt, float *__restrict__ D, uint64_t ldD,
    const uint32_t *__restrict__ only, const uint32_t *__restrict__ gate)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    if (gate && *gate == 0) return;              // fix-up pass with nothing flagged
    if (only) {                                  // fix-up pass: skip query tiles with no flagged query
        bool any = false;
        for (uint32_t i = 0; i < DM_Q; i++) {
            uint32_t gq = blockIdx.y * DM_Q + i;
            if (gq < B && only[gq]) any = true;
        }
        if (!any) return;
    }
    __shared__ float qs[DM_Q][DM_STR];
    __shared__ float cs[DM_C][DM_STR];
    __shared__ float red[DM_Q * DM_C][17];

    const int tid = threadIdx.x;
    const int klane = tid & 15, pt = tid >> 4;
    const int tq = pt & 3, tc = pt >> 2;
    const uint32_t q0 = blockIdx.y * DM_Q;
    const uint32_t d16 = d & ~15u;
    const uint64_t ncol_tiles = (N + DM_C - 1) / DM_C;
  for (uint64_t ctile = blockIdx.x; ctile < ncol_tiles; ctile += gridDim.x) {     // column tiles of this CTA
    const uint64_t c0 = ctile * DM_C;
    __syncthreads();

    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

    for (uint32_t k0 = 0; k0 < d16; k0 += DM_KT) {
#pragma unroll
        for (int u = 0; u < 2; u++) {
            int idx = tid + DM_THREADS * u, row = idx >> 5, col = idx & 31;
            uint32_t gq = q0 + row, gk = k0 + col;
            qs[row][col] = (gq < B && gk < d16) ? Q[(size_t)gq * d + gk] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            int idx = tid + DM_THREADS * u, row = idx >> 5, col = idx & 31;
            uint64_t gc = c0 + row; uint32_t gk = k0 + col;
            cs[row][col] = (gc < N && gk < d16) ? C[(size_t)gc * d + gk] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int step = 0; step < 2; step++) {
            if (k0 + 16 * step < d16) {
                const int kk = 16 * step + klane;
                float qv[4], cv[8];
#pragma unroll
                for (int i = 0; i < 4; i++) qv[i] = qs[4 * tq + i][kk];
#pragma unroll
                for (int j = 0; j < 8; j++) cv[j] = cs[8 * tc + j][kk];
                if (mode == 0) {
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int j = 0; j < 8; j++) {
                            float df = __fsub_rn(qv[i], cv[j]);
                            acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(df, df));
                        }
                } else {
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int j = 0; j < 8; j++) acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(qv[i], cv[j]));
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) red[(4 * tq + i) * DM_C + 8 * tc + j][klane] = acc[i][j];
    __syncthreads();
    for (int pair = tid; pair < DM_Q * DM_C; pair += DM_THREADS) {
        const int qrow = pair / DM_C, ccol = pair % DM_C;
        const uint32_t gq = q0 + qrow; const uint64_t gc = c0 + ccol;
        if (gq >= B || gc >= N) continue;
        float t = 0.f;
#pragma unroll
        for (int l = 0; l < 16; l++) t = __fadd_rn(t, red[pair][l]);
        float s = 0.f;                                   // remainder dims, sequential
        const float *x = Q + (size_t)gq * d, *y = C + (size_t)gc * d;
        for (uint32_t i = d16; i < d; i++) {
            if (mode == 0) { float df = __fsub_rn(x[i], y[i]); s = __fadd_rn(s, __fmul_rn(df, df)); }
            else s = __fadd_rn(s, __fmul_rn(x[i], y[i]));
        }
        float v = __fadd_rn(s, t);
        if (mode == 1) v = __fsub_rn(1.0f, v);
        else if (mode == 2) v = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(v, xnorm[gq]), ysqrt[gc]));
        D[(size_t)gq * ldD + gc] = v;
    }
  }
}

// half-warp per row: lane l (< 16) is lance's accumulator lane l
__device__ __forceinline__ float halfwarp_dot(const float *__restrict__ x, const float *__restrict__ y,
                                               uint32_t d, int hl, unsigned hmask, int hbase)
{
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    for (uint32_t k = hl; k < d16; k += 16) a = __fadd_rn(a, __fmul_rn(x[k], y[k]));
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) s = __fadd_rn(s, __fmul_rn(x[i], y[i]));
    return __fadd_rn(s, t);
}
__device__ __forceinline__ float halfwarp_l2(const float *__restrict__ x, const float *__restrict__ y,
                                              uint32_t d, int hl, unsigned hmask, int hbase)
{
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    uint32_t k = hl;
    for (; k + 7 * 16 < d16; k += 8 * 16) {             // eight independent loads of each operand in flight
        float xv[8], yv[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { xv[u] = x[k + 16 * u]; yv[u] = y[k + 16 * u]; }
#pragma unroll
        for (int u = 0; u < 8; u++) { const float df = __fsub_rn(xv[u], yv[u]); a = __fadd_rn(a, __fmul_rn(df, df)); }
    }
    for (; k < d16; k += 16) { float df = __fsub_rn(x[k], y[k]); a = __fadd_rn(a, __fmul_rn(df, df)); }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) { float df = __fsub_rn(x[i], y[i]); s = __fadd_rn(s, __fmul_rn(df, df)); }
    return __fadd_rn(s, t);
}

// the same sum with x in shared memory and U loads of y in flight per lane: one or two L2 round trips per candidate row
// instead of d / 128 (coarse_finish_kernel re-scores ~100 centroids per query at nlist 16384, a latency chain each)
template <int U>
__device__ __forceinline__ float halfwarp_l2_sx(const float *sx, const float *__restrict__ y, uint32_t d, int hl,
                                                unsigned hmask, int hbase)
{
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    for (uint32_t k0 = 0; k0 < d16; k0 += 16 * U) {
        float yv[U];
#pragma unroll
        for (int u = 0; u < U; u++) yv[u] = __ldg(y + min(k0 + 16 * u + hl, d - 1));
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (k0 + 16 * u < d16) { const float df = __fsub_rn(sx[k0 + 16 * u + hl], yv[u]); a = __fadd_rn(a, __fmul_rn(df, df)); }
        }
    }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) { float df = __fsub_rn(sx[i], y[i]); s = __fadd_rn(s, __fmul_rn(df, df)); }
    return __fadd_rn(s, t);
}

__global__ void row_norms_kernel(const float *__restrict__ X, uint64_t n, uint32_t d, float *__restrict__ out)
{
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (row >= n) return;                               // whole half-warp exits together
    const float *x = X + row * d;
    float v = sqrtf(halfwarp_dot(x, x, d, hl, hmask, hbase));
    if (hl == 0) out[row] = v;
}

__global__ void normalize_kernel(const float *__restrict__ X, uint32_t B, uint32_t d, float *__restrict__ out)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (row >= B) return;
    const float *x = X + (size_t)row * d;
    const float nrm = sqrtf(halfwarp_dot(x, x, d, hl, hmask, hbase));
    for (uint32_t k = hl; k < d; k += 16) out[(size_t)row * d + k] = __fdiv_rn(x[k], nrm);
}

__global__ void pair_distance_kernel(const float *__restrict__ Q, const float *__restrict__ V,
                                     const uint64_t *__restrict__ pos, uint32_t B, uint32_t nc, uint32_t d,
                                     int metric, float *__restrict__ out)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint64_t pair = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (pair >= (uint64_t)B * nc) return;
    const uint32_t q = (uint32_t)(pair / nc);
    const uint64_t ps = pos[pair];
    if (ps == UINT64_MAX) { if (hl == 0) out[pair] = CUDART_INF_F; return; }
    const float *x = Q + (size_t)q * d, *y = V + ps * d;
    float v;
    if (metric == LGPU_L2) v = halfwarp_l2(x, y, d, hl, hmask, hbase);
    else if (metric == LGPU_DOT) v = __fsub_rn(1.0f, halfwarp_dot(x, y, d, hl, hmask, hbase));
    else {   // cosine_scalar: 1 - xy / |x| / sqrt(yy)
        float xn = sqrtf(halfwarp_dot(x, x, d, hl, hmask, hbase));
        float yy = halfwarp_dot(y, y, d, hl, hmask, hbase);
        float xy = halfwarp_dot(x, y, d, hl, hmask, hbase);
        v = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(xy, xn), sqrtf(yy)));
    }
    if (hl == 0) out[pair] = v;
}

// exact MaxSim re-score of the multivector shortlist, half a warp per (query, candidate row): for each query vector i
// in order, the NaN-skipping min over the row's vectors j of 1 - xy / |q_i| / |v_j| (xy in lance's lane order: the
// same roundings as dist_matrix_kernel mode 2), added onto a sum that starts at 0.0f -- the exact path's bits
__global__ void mv_rescore_kernel(const float *__restrict__ Q, const uint32_t *__restrict__ q_off, uint32_t qa,
                                  const float *__restrict__ xnorm, const float *__restrict__ V,
                                  const float *__restrict__ ysqrt, const uint64_t *__restrict__ offsets,
                                  const uint64_t *__restrict__ row_ids, uint32_t d, uint32_t B,
                                  const uint32_t *__restrict__ cand, const uint32_t *__restrict__ count, uint32_t cap,
                                  float *__restrict__ out, uint64_t *__restrict__ ids)
{
    pdl_entry();
    const uint64_t pair = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (pair >= (uint64_t)B * cap) return;                  // whole half-warp exits together
    const uint32_t b = (uint32_t)(pair / cap), slot = (uint32_t)(pair % cap);
    if (slot >= min(count[b], cap)) {
        if (hl == 0) { out[pair] = CUDART_NAN_F; ids[pair] = UINT64_MAX; }
        return;
    }
    const uint32_t r = cand[pair];
    const uint64_t j0 = offsets[r], j1 = offsets[r + 1];
    float s = 0.f;
    for (uint32_t i = q_off[qa + b]; i < q_off[qa + b + 1]; i++) {
        const float *x = Q + (size_t)i * d;
        float m = CUDART_NAN_F;
        for (uint64_t j = j0; j < j1; j++) {
            const float xy = halfwarp_dot(x, V + j * d, d, hl, hmask, hbase);
            const float c = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(xy, xnorm[i]), ysqrt[j]));
            if (c < m || m != m) m = c;
        }
        s = __fadd_rn(s, m);
    }
    if (hl == 0) { out[pair] = s; ids[pair] = row_ids ? row_ids[r] : r; }
}

// ---- the coarse step after the tensor-core GEMM, in one kernel (one CTA per query):
// S[q][x] = |x|^2 - 2 bf16(q).bf16(x) differs from |q - x|^2 - |q|^2 by at most E_q (gemm.cu's band).  (1) an upper
// bound tau of the k-th smallest S of the row by counting bisection; (2) every column with S <= tau + 2 E_q -- a
// superset of the exact k nearest -- is (3) re-scored exactly in lance's lane order, half a warp per column, and
// (4) the k best by (distance, column) are written.  More than `cap` candidates (ties, degenerate data): flags[q] = 1
// and the caller's exact kernels redo the query.
constexpr int CF_THREADS = 256;
// VPT = row values per thread, held in registers for the counting passes (N <= 256 VPT); VPT == 0: the row is
// re-read from global memory (L2) in every pass (flat-sized rows)
template <int VPT>
__global__ void __launch_bounds__(CF_THREADS) coarse_finish_kernel(const float *__restrict__ S, uint64_t ld, uint32_t N_,
                                                                   const float *__restrict__ Q, const float *__restrict__ C,
                                                                   const float *__restrict__ qn2,
                                                                   const float *__restrict__ qerr, float xmax, float xerr,
                                                                   uint32_t d,
                                                                   uint32_t k, uint32_t cap,
                                                                   uint64_t *__restrict__ out_ids, float *__restrict__ out_dist,
                                                                   uint32_t *__restrict__ out_cnt, uint32_t *__restrict__ flags,
                                                                   uint32_t *__restrict__ gate,
                                                                   const uint64_t *__restrict__ list_pos,
                                                                   const uint32_t *__restrict__ list_cnt)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    // long rows only are staged through shared memory: at VPT 4 / 16 the few register loads avoid the extra barrier
    constexpr bool STAGED = VPT >= 64;
    constexpr int NV0 = STAGED ? VPT : 0;
    extern __shared__ __align__(16) unsigned char csm[];
    float *s_row = reinterpret_cast<float *>(csm);                  // [VPT * CF_THREADS] the score row (VPT > 0)
    uint32_t *s_col = reinterpret_cast<uint32_t *>(s_row + (size_t)NV0 * CF_THREADS);   // [cap] candidate columns
    uint32_t *s_key = s_col + cap;                                  // [cap] exact distance keys
    float *s_x = reinterpret_cast<float *>(s_key + cap);            // [d] the query
    __shared__ uint32_t s_lo, s_hi, s_valid, s_n, s_cnt[24];
    const uint32_t q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31;
    const float *row = S + (size_t)q * ld;
    // list mode (large nlist): the row is the query's list of admitted scores from the GEMM's filtering epilogue,
    // list_pos maps a list entry to its column; every column with S <= (k-th smallest S of a column sample) + 2 E_q is in
    // the list, so the k-th smallest of the list is the k-th smallest of the whole row and the band below is complete
    const uint32_t listed = list_cnt ? list_cnt[q] : 0u;
    const uint32_t N = list_cnt ? min(listed, (uint32_t)ld) : N_;
    if constexpr (STAGED) {
        // The row goes global -> shared with cp.async (16 B per request, all VPT / 4 requests of a thread in flight at
        // once), then shared -> registers.  Register loads, however they were written, came out of ptxas as
        // load -> use -> load: 64 serial DRAM round trips per thread at nlist 16384.  ld is a multiple of 4 floats and
        // the buffer holds ld floats per row.
        const uint32_t s_base = (uint32_t)__cvta_generic_to_shared(s_row);
        for (uint32_t i = (uint32_t)tid * 4; i < ld && i < (uint32_t)VPT * CF_THREADS; i += CF_THREADS * 4)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s_base + i * 4), "l"(row + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (tid == 0) { s_lo = 0xffffffffu; s_hi = 0u; s_valid = 0u; s_n = 0u; }
    if (tid < 24) s_cnt[tid] = 0u;
    for (uint32_t t = tid; t < d; t += CF_THREADS) s_x[t] = Q[(size_t)q * d + t];
    if constexpr (STAGED) asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    constexpr int NV = VPT > 0 ? VPT : 1;
    float v[NV];
    uint32_t kmin = 0xffffffffu, kmax = 0u, nv = 0;
    if constexpr (VPT > 0) {
        if constexpr (STAGED) {
#pragma unroll
            for (int j = 0; j < VPT; j++) v[j] = s_row[min((uint32_t)j * CF_THREADS + tid, N - 1)];
        } else {
#pragma unroll
            for (int j = 0; j < VPT; j++) v[j] = __ldg(row + min((uint32_t)j * CF_THREADS + tid, N ? N - 1 : 0u));
        }
#pragma unroll
        for (int j = 0; j < VPT; j++) {
            if ((uint32_t)j * CF_THREADS + tid >= N) v[j] = CUDART_NAN_F;       // NaN never counts
            if (v[j] == v[j]) { const uint32_t kk = f32_key(v[j]); kmin = min(kmin, kk); kmax = max(kmax, kk); nv++; }
        }
    } else {
        for (uint32_t i = tid; i < N; i += CF_THREADS) {
            const float x = row[i];
            if (x == x) { const uint32_t kk = f32_key(x); kmin = min(kmin, kk); kmax = max(kmax, kk); nv++; }
        }
    }
    kmin = __reduce_min_sync(0xffffffffu, kmin); kmax = __reduce_max_sync(0xffffffffu, kmax);
    nv = __reduce_add_sync(0xffffffffu, nv);
    if (lane == 0) { atomicMin(&s_lo, kmin); atomicMax(&s_hi, kmax); atomicAdd(&s_valid, nv); }
    __syncthreads();
    const uint32_t kk = min(k, s_valid);
    // a non-finite query (inf, NaN, |q|^2 overflowing) has no finite band: its scores prove nothing, the caller redoes it
    const float E = tc_band(qn2[q], qerr[q], xmax, xerr, d);
    const bool band_ok = isfinite(E);
    float thr = -CUDART_INF_F;
    if (kk > 0 && band_ok) {
        float lo = key_f32(s_lo), hi = key_f32(s_hi);               // invariant: count(S <= hi) >= kk
        if (hi < CUDART_INF_F && lo > -CUDART_INF_F) {
            for (int it = 0; it < 20 && hi - lo > 0.25f * E; it++) {    // the band is 2E wide anyway
                const float mid = 0.5f * lo + 0.5f * hi;
                uint32_t c = 0;
                if constexpr (VPT > 0) {
#pragma unroll
                    for (int j = 0; j < VPT; j++) c += v[j] <= mid ? 1u : 0u;
                } else {
                    for (uint32_t i = tid; i < N; i += CF_THREADS) c += row[i] <= mid ? 1u : 0u;
                }
                c = __reduce_add_sync(0xffffffffu, c);
                if (lane == 0 && c) atomicAdd(&s_cnt[it], c);
                __syncthreads();
                if (s_cnt[it] >= kk) hi = mid; else lo = mid;
            }
        }
        thr = hi + 2.0f * E;
    }
    if constexpr (VPT > 0) {
#pragma unroll
        for (int j = 0; j < VPT; j++) {
            if (v[j] <= thr) {
                const uint32_t at = atomicAdd(&s_n, 1u);
                if (at < cap) {
                    const uint32_t idx = (uint32_t)j * CF_THREADS + tid;
                    s_col[at] = list_pos ? (uint32_t)list_pos[(size_t)q * ld + idx] : idx;
                }
            }
        }
    } else {
        for (uint32_t i = tid; i < N; i += CF_THREADS) {
            if (row[i] <= thr) {
                const uint32_t at = atomicAdd(&s_n, 1u);
                if (at < cap) s_col[at] = list_pos ? (uint32_t)list_pos[(size_t)q * ld + i] : i;
            }
        }
    }
    __syncthreads();
    const uint32_t total = s_n, n = min(total, cap);
    if (tid == 0) {
        const bool redo = total > cap || listed > ld || !band_ok;   // (a list that overflowed is not a superset)
        flags[q] = redo ? 1u : 0u;
        if (redo && gate) *gate = 1u;                               // opens the gate of the caller's exact fix-up
    }
    // exact re-score, half a warp per candidate column (lance's l2: 16 lane accumulators, sequential lane sum)
    const int hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    for (uint32_t c0 = 0; c0 < n; c0 += CF_THREADS / 16) {
        const uint32_t c = c0 + (tid >> 4);
        if (c < n) {                                                 // a whole half-warp takes the branch together
            const float dv = halfwarp_l2_sx<48>(s_x, C + (size_t)s_col[c] * d, d, hl, hmask, hbase);
            if (hl == 0) s_key[c] = (dv != dv) ? 0xffffffffu : f32_key(dv == 0.f ? 0.f : dv);
        }
    }
    __syncthreads();
    uint32_t n2 = 2;
    while (n2 < n) n2 <<= 1;
    for (uint32_t i = n + tid; i < n2 && i < cap; i += CF_THREADS) { s_key[i] = 0xffffffffu; s_col[i] = 0xffffffffu; }
    __syncthreads();
    for (uint32_t size = 2; size <= n2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = tid; i < (n2 >> 1); i += CF_THREADS) {
                const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const uint32_t ka = s_key[lo], kb = s_key[hi], ia = s_col[lo], ib = s_col[hi];
                if ((kb < ka || (kb == ka && ib < ia)) == ((lo & size) == 0)) {
                    s_key[lo] = kb; s_key[hi] = ka; s_col[lo] = ib; s_col[hi] = ia;
                }
            }
            __syncthreads();
        }
    }
    uint32_t have = 0;                                               // NaN distances sort last and are dropped
    for (uint32_t i = tid; i < k; i += CF_THREADS) {
        const bool ok = i < n && s_key[i] != 0xffffffffu;
        out_ids[(size_t)q * k + i] = ok ? (uint64_t)s_col[i] : UINT64_MAX;
        out_dist[(size_t)q * k + i] = ok ? key_f32(s_key[i]) : CUDART_INF_F;
        have += ok ? 1u : 0u;
    }
    have = __reduce_add_sync(0xffffffffu, have);
    if (tid == 0) out_cnt[q] = 0;
    __syncthreads();
    if (lane == 0 && have) atomicAdd(out_cnt + q, have);
}

}  // namespace

void launch_coarse_finish(const float *S, uint64_t ld, uint32_t B, uint32_t N, const float *Q, const float *C,
                          const float *qn2, const float *qerr, float xmax, float xerr, uint32_t d, uint32_t k,
                          uint64_t *out_ids, float *out_dist,
                          uint32_t *out_cnt, uint32_t *flags, uint32_t *gate, cudaStream_t st,
                          const uint64_t *list_pos, const uint32_t *list_cnt)
{
    if (B == 0 || N == 0) return;
    if (gate) LGPU_CUDA(cudaMemsetAsync(gate, 0, 4, st));
    uint32_t cap = 512;                                              // (only the entries in use are sorted)
    while (cap < 4 * k) cap <<= 1;                                   // power of two >= 4 k
    const size_t smem0 = (size_t)cap * 8 + (size_t)d * 4;
    if (smem0 > 128 * 1024) { set_error("internal: coarse_finish candidate list does not fit in shared memory"); throw Failure{LGPU_RUNTIME}; }
#define LGPU_CF(V) do { \
        const size_t smem = smem0 + ((V) >= 64 ? (size_t)(V) * CF_THREADS * 4 : 0); \
        if (smem > 48 * 1024) LGPU_CUDA(cudaFuncSetAttribute(coarse_finish_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        launch_k(coarse_finish_kernel<V>, dim3(B), dim3(CF_THREADS), smem, st, S, ld, N, Q, C, qn2, qerr, xmax, xerr, d, k, cap, out_ids, out_dist, out_cnt, flags, gate, list_pos, list_cnt); \
    } while (0)
    if ((list_pos == nullptr) != (list_cnt == nullptr) || (list_pos && N != ld)) {
        set_error("internal: coarse_finish list mode needs positions, counts and N == list capacity"); throw Failure{LGPU_RUNTIME};
    }
    const bool staged = (ld & 3u) == 0 && ld >= N;                  // cp.async needs 16-byte rows
    if (staged && N <= 4 * CF_THREADS) LGPU_CF(4);
    else if (staged && N <= 16 * CF_THREADS) LGPU_CF(16);
    else if (staged && N <= 64 * CF_THREADS) LGPU_CF(64);
    else LGPU_CF(0);
#undef LGPU_CF
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_dist_matrix(const float *Q, const float *C, uint32_t B, uint64_t N, uint32_t d, int mode,
                        const float *xnorm, const float *ysqrt, float *D, uint64_t ldD, cudaStream_t st,
                        const uint32_t *only, const uint32_t *gate)
{
    if (B == 0 || N == 0) return;
    // the fix-up pass (`only`) is almost always a no-op: keep its CTA count small
    const uint64_t ct = (N + DM_C - 1) / DM_C;
    dim3 grid((unsigned)std::min<uint64_t>(ct, only ? 16 : ((uint64_t)1 << 30)), (B + DM_Q - 1) / DM_Q);
    launch_k(dist_matrix_kernel, grid, dim3(DM_THREADS), 0, st, Q, C, B, N, d, mode, xnorm, ysqrt, D, ldD, only, gate); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_row_norms(const float *X, uint64_t n, uint32_t d, float *out, cudaStream_t st)
{
    if (n == 0) return;
    uint64_t threads = n * 16;
    row_norms_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(X, n, d, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_normalize(const float *X, uint32_t B, uint32_t d, float *out, cudaStream_t st)
{
    if (B == 0) return;
    uint64_t threads = (uint64_t)B * 16;
    launch_k(normalize_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, X, B, d, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_pair_distance(const float *Q, const float *V, const uint64_t *pos, uint32_t B, uint32_t nc,
                          uint32_t d, int metric, float *out, cudaStream_t st)
{
    if (B == 0 || nc == 0) return;
    uint64_t threads = (uint64_t)B * nc * 16;
    launch_k(pair_distance_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, Q, V, pos, B, nc, d, metric, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_rescore(const float *Q, const uint32_t *q_off, uint32_t qa, const float *xnorm, const float *V,
                       const float *ysqrt, const uint64_t *offsets, const uint64_t *row_ids, uint32_t d, uint32_t B,
                       const uint32_t *cand, const uint32_t *count, uint32_t cap, float *out, uint64_t *ids,
                       cudaStream_t st)
{
    if (B == 0 || cap == 0) return;
    const uint64_t threads = (uint64_t)B * cap * 16;
    launch_k(mv_rescore_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, Q, q_off, qa, xnorm, V, ysqrt,
             offsets, row_ids, d, B, cand, count, cap, out, ids); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
