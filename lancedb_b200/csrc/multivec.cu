// multivec.cu -- late-interaction (MaxSim) search over multivector columns, list<fixed_size_list<float, d>>:
//     _distance(q, r) = sum_i min_j cosd(q_i, v_j)      (i over the query's vectors in order, f32 from 0.0f)
// with cosd the flat path's exact cosine (dist_matrix_kernel mode 2, lance's lane order).  A pair whose cosd is NaN
// (zero-norm vector, NaN component) is skipped by the min; a query vector with no finite-or-infinite pair (an empty
// row, or every pair NaN) makes the row's distance NaN, and select drops NaN distances.
//
// The tensor-core path (api.cu multivec_search_device) scores fp16 copies of the normalised vectors with the F16MaxSim
// policy of gemm_dist_kernel, whose epilogue keeps the largest approximate similarity per (query vector, document);
// mv_approx_sum_kernel turns those into approximate distances, a shortlist admits every row within 2 E of the k-th
// approximate distance (mv_band below), dist.cu's mv_rescore_kernel re-scores the admitted rows exactly, and a query
// whose list overflowed (or that holds a zero / non-finite vector) is redone by the exact path.
//
// The exact path runs in three steps per (block of query vectors, chunk of whole rows) (api.cu multivec_search_device):
//   dist_matrix_kernel   P[i][j]  = cosd(q_i, v_j) for the chunk's stored vectors j
//   mv_rowmin_kernel     M[i][r]  = min over row r's run of P[i][.], NaN skipped
//   mv_rowsum_kernel     D[b][r] += M[i][r] for the block's vectors i of query b, in order of i
// and a block that starts inside a query continues that query's running sum, so the order of the additions is the
// oracle's whatever the blocking.
#include "kernels.cuh"

#include <cuda_fp16.h>
#include <math_constants.h>

#include <algorithm>

namespace lgpu {

// The error band of the approximate MaxSim distance of a query of nq vectors (dimension d): |A - D| <= E for every
// row, A the tensor-core path's approximate distance, D the exact one (the oracle's).  Per query vector and stored
// vector, with u = 2^-24 and a, b the f32 normalised vectors (|a|, |b| <= 1 + (d + 8) u):
//   - both fp16 roundings: |fp16(a).fp16(b) - a.b| <= |fp16(a) - a| |fp16(b)| + |a| |fp16(b) - b|
//     <= 2^-11 (2 + 2^-11) (1 + (d + 8) u)^2 + 2 * 2^-25 sqrt(d) (subnormal outputs), < 1.01 * 2^-10 + sqrt(d) u;
//   - wgmma's f32 accumulation of the d exact fp16 products: <= 4 d u sum |products| <= 4.1 d u (the bound the
//     bf16 shortlist's band uses, tested on the H100 in tests/test_gpu_tensorcore.py);
//   - a.b against the lance formula 1 - xy / |x| / sqrt(yy): the dot's lane sums (d + 2) u, the two norms and the
//     normalisation (d + 8) u each, the divisions and the final subtraction 4 u: < (3 d + 30) u, and 1 - s~ in f32 2 u;
// so e = 1.01 * 2^-10 + (8 d + sqrt(d) + 40) u per query vector, and |min_j p_j - min_j q_j| <= max_j |p_j - q_j| carries
// e through the min.  The two sums over i (approximate and exact, partial sums <= 2.02 nq) add 2 * 2.02 nq^2 u.  The
// whole is scaled by 1 + 2^-8 for the f32 arithmetic of E itself.
__host__ __device__ __forceinline__ float mv_band(uint32_t nq, uint32_t d)
{
    const float u = 0x1p-24f;
    const float e = 1.01f * 0x1p-10f + (8.0f * (float)d + sqrtf((float)d) + 40.0f) * u;
    return ((float)nq * e + 4.04f * (float)nq * (float)nq * u) * (1.0f + 0x1p-8f);
}

namespace {

constexpr int MV_THREADS = 256;

// fp16(x / |x|), |x| = sqrt of lance's dot (the normalisation of dist.cu normalize_kernel); half a warp per row
__global__ void mv_normalize_f16_kernel(const float *__restrict__ X, uint64_t n, uint32_t d, __half *__restrict__ out,
                                        uint32_t *__restrict__ bad)
{
    pdl_entry();
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (row >= n) return;
    const float *x = X + row * d;
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    bool fin = true;
    for (uint32_t k = hl; k < d16; k += 16) { a = __fadd_rn(a, __fmul_rn(x[k], x[k])); fin = fin && isfinite(x[k]); }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) { s = __fadd_rn(s, __fmul_rn(x[i], x[i])); fin = fin && isfinite(x[i]); }
    const float nrm = sqrtf(__fadd_rn(s, t));
    const bool ok = __all_sync(hmask, fin) && nrm > 0.f && isfinite(nrm);
    for (uint32_t k = hl; k < d; k += 16) out[row * d + k] = __float2half_rn(ok ? __fdiv_rn(x[k], nrm) : 0.f);
    if (hl == 0) bad[row] = ok ? 0u : 1u;
}

// A[b - qa][r] = sum_i (1 - max similarity of vector i over row r); NaN when a vector saw no column (empty row)
__global__ void __launch_bounds__(MV_THREADS) mv_approx_sum_kernel(const uint32_t *__restrict__ M, uint64_t ldM,
                                                                   const uint32_t *__restrict__ q_off, uint32_t qa,
                                                                   uint32_t qb, uint32_t i_base, uint64_t N,
                                                                   float *__restrict__ A, uint64_t ldA)
{
    pdl_entry();
    const uint64_t total = (uint64_t)(qb - qa) * N;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = qa + (uint32_t)(w / N);
        const uint64_t r = w % N;
        float s = 0.f;
        for (uint32_t i = q_off[b]; i < q_off[b + 1]; i++) {
            const uint32_t key = M[(size_t)(i - i_base) * ldM + r];
            s = key ? s + (1.0f - key_f32(key)) : CUDART_NAN_F;
            if (!key) break;
        }
        A[(size_t)(b - qa) * ldA + r] = s;
    }
}

__global__ void mv_threshold_kernel(const float *__restrict__ dist, const uint32_t *__restrict__ cnt,
                                    const uint32_t *__restrict__ q_off, uint32_t qa, uint32_t B, uint32_t k, uint32_t d,
                                    float *__restrict__ thr)
{
    pdl_entry();
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float E = mv_band(q_off[qa + b + 1] - q_off[qa + b], d);
    thr[b] = cnt[b] >= k ? __fadd_ru(dist[(size_t)b * k + k - 1], __fmul_ru(2.0f, E)) : CUDART_INF_F;   // rounded up
}

__global__ void mv_admit_kernel(const float *__restrict__ A, uint64_t ldA, uint64_t N, const float *__restrict__ thr,
                                uint32_t cap, uint32_t *__restrict__ count, uint32_t *__restrict__ cand)
{
    pdl_entry();
    const uint32_t b = blockIdx.y;
    const float t = thr[b];
    const float *row = A + (size_t)b * ldA;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < N; r += (uint64_t)gridDim.x * blockDim.x)
        if (row[r] <= t) {
            const uint32_t slot = atomicAdd(count + b, 1u);
            if (slot < cap) cand[(size_t)b * cap + slot] = (uint32_t)r;
        }
}

// one block
__global__ void __launch_bounds__(1024) mv_flags_kernel(const uint32_t *__restrict__ count, uint32_t cap,
                                                        const uint32_t *__restrict__ qbad, const uint32_t *__restrict__ q_off,
                                                        uint32_t qa, uint32_t B, uint32_t *__restrict__ flags,
                                                        uint32_t *__restrict__ vflags, uint32_t *__restrict__ gate)
{
    pdl_entry();
    __shared__ uint32_t any;
    if (threadIdx.x == 0) any = 0;
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) {
        uint32_t f = count[b] > cap ? 1u : 0u;
        for (uint32_t i = q_off[qa + b]; i < q_off[qa + b + 1]; i++) f |= qbad[i];
        flags[b] = f;
        if (f) any = 1;
    }
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < B; b += blockDim.x)
        for (uint32_t i = q_off[qa + b]; i < q_off[qa + b + 1]; i++) vflags[i - q_off[qa]] = flags[b];
    if (threadIdx.x == 0) *gate = any;
}

// one thread per (query vector i, row r of the chunk); adjacent threads take adjacent rows, which are adjacent runs of
// P's columns
__global__ void __launch_bounds__(MV_THREADS) mv_rowmin_kernel(const float *__restrict__ P, uint64_t ldP, uint32_t nqv,
                                                               const uint64_t *__restrict__ offsets, uint64_t r0,
                                                               uint32_t nr, float *__restrict__ M, uint64_t ldM,
                                                               const uint32_t *__restrict__ gate)
{
    pdl_entry();
    if (gate && *gate == 0) return;
    const uint64_t base = offsets[r0];
    const uint64_t total = (uint64_t)nqv * nr;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t i = (uint32_t)(w / nr), r = (uint32_t)(w % nr);
        const uint64_t j0 = offsets[r0 + r] - base, j1 = offsets[r0 + r + 1] - base;
        const float *p = P + (size_t)i * ldP;
        float m = CUDART_NAN_F;
        for (uint64_t j = j0; j < j1; j++) {
            const float v = __ldg(p + j);
            if (v < m || m != m) m = v;                     // a NaN v never replaces a number
        }
        M[(size_t)i * ldM + r] = m;
    }
}

// one thread per (query b in [b_lo, b_hi), row r of the chunk): adds M[i - i0][r] for the query's vectors i inside the
// block [i0, i1), in order, onto the running sum (which starts at 0.0f in the block holding the query's first vector)
__global__ void __launch_bounds__(MV_THREADS) mv_rowsum_kernel(const float *__restrict__ M, uint64_t ldM,
                                                               const uint32_t *__restrict__ q_off, uint32_t b_lo,
                                                               uint32_t b_hi, uint32_t qa, uint32_t i0, uint32_t i1,
                                                               uint32_t nr, float *__restrict__ D, uint64_t ldD,
                                                               uint64_t col0, const uint32_t *__restrict__ only,
                                                               const uint32_t *__restrict__ gate)
{
    pdl_entry();
    if (gate && *gate == 0) return;
    const uint64_t total = (uint64_t)(b_hi - b_lo) * nr;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = b_lo + (uint32_t)(w / nr), r = (uint32_t)(w % nr);
        if (only && !only[b - qa]) continue;
        const uint32_t qs = q_off[b], qe = q_off[b + 1];
        const uint32_t lo = max(qs, i0), hi = min(qe, i1);
        float *d = D + (size_t)(b - qa) * ldD + col0 + r;
        float s = qs < i0 ? *d : 0.0f;
        for (uint32_t i = lo; i < hi; i++) s = __fadd_rn(s, M[(size_t)(i - i0) * ldM + r]);
        *d = s;
    }
}

unsigned grid_for(uint64_t items, int num_sms)
{
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((items + MV_THREADS - 1) / MV_THREADS, (uint64_t)num_sms * 16));
}

}  // namespace

void launch_mv_rowmin(const float *P, uint64_t ldP, uint32_t nqv, const uint64_t *offsets, uint64_t r0, uint32_t nr,
                      float *M, uint64_t ldM, int num_sms, cudaStream_t st, const uint32_t *gate)
{
    if (nqv == 0 || nr == 0) return;
    launch_k(mv_rowmin_kernel, dim3(grid_for((uint64_t)nqv * nr, num_sms)), dim3(MV_THREADS), 0, st, P, ldP, nqv, offsets,
             r0, nr, M, ldM, gate); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_rowsum(const float *M, uint64_t ldM, const uint32_t *q_off, uint32_t b_lo, uint32_t b_hi, uint32_t qa,
                      uint32_t i0, uint32_t i1, uint32_t nr, float *D, uint64_t ldD, uint64_t col0, int num_sms,
                      cudaStream_t st, const uint32_t *only, const uint32_t *gate)
{
    if (b_hi <= b_lo || nr == 0) return;
    launch_k(mv_rowsum_kernel, dim3(grid_for((uint64_t)(b_hi - b_lo) * nr, num_sms)), dim3(MV_THREADS), 0, st, M, ldM,
             q_off, b_lo, b_hi, qa, i0, i1, nr, D, ldD, col0, only, gate); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

float mv_band_host(uint32_t nq, uint32_t d) { return mv_band(nq, d); }

void launch_mv_normalize_f16(const float *X, uint64_t n, uint32_t d, void *out, uint32_t *bad, cudaStream_t st)
{
    if (n == 0) return;
    launch_k(mv_normalize_f16_kernel, dim3((unsigned)((n * 16 + 255) / 256)), dim3(256), 0, st, X, n, d,
             reinterpret_cast<__half *>(out), bad); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_approx_sum(const uint32_t *M, uint64_t ldM, const uint32_t *q_off, uint32_t qa, uint32_t qb,
                          uint32_t i_base, uint64_t N, float *A, uint64_t ldA, int num_sms, cudaStream_t st)
{
    if (qb <= qa || N == 0) return;
    launch_k(mv_approx_sum_kernel, dim3(grid_for((uint64_t)(qb - qa) * N, num_sms)), dim3(MV_THREADS), 0, st, M, ldM,
             q_off, qa, qb, i_base, N, A, ldA); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_threshold(const float *dist, const uint32_t *cnt, const uint32_t *q_off, uint32_t qa, uint32_t B,
                         uint32_t k, uint32_t d, float *thr, cudaStream_t st)
{
    if (B == 0) return;
    launch_k(mv_threshold_kernel, dim3((B + 127) / 128), dim3(128), 0, st, dist, cnt, q_off, qa, B, k, d, thr);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_admit(const float *A, uint64_t ldA, uint32_t B, uint64_t N, const float *thr, uint32_t cap,
                     uint32_t *count, uint32_t *cand, cudaStream_t st)
{
    if (B == 0 || N == 0) return;
    launch_k(mv_admit_kernel, dim3((unsigned)std::min<uint64_t>((N + 1023) / 1024, 64), B), dim3(256), 0, st, A, ldA, N,
             thr, cap, count, cand); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_mv_flags(const uint32_t *count, uint32_t cap, const uint32_t *qbad, const uint32_t *q_off, uint32_t qa,
                     uint32_t B, uint32_t *flags, uint32_t *vflags, uint32_t *gate, cudaStream_t st)
{
    if (B == 0) return;
    launch_k(mv_flags_kernel, dim3(1), dim3(1024), 0, st, count, cap, qbad, q_off, qa, B, flags, vflags, gate);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
