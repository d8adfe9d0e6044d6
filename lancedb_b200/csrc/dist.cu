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

#include <cuda_fp16.h>
#include <math_constants.h>

#include <algorithm>

namespace lgpu {

namespace {

constexpr int DM_Q = 16, DM_C = 32, DM_KT = 32, DM_STR = 36, DM_THREADS = 256;

// A stored row element as f32: an fp16 row converts exactly in registers, so every kernel below runs the same f32
// arithmetic, in the same lane order, on either row type (the stored-row type T is float or __half)
__device__ __forceinline__ float ldf(float v) { return v; }
__device__ __forceinline__ float ldf(__half v) { return __half2float(v); }

template <class T>
__global__ void __launch_bounds__(DM_THREADS) dist_matrix_kernel(
    const float *__restrict__ Q, const T *__restrict__ C, uint32_t B, uint64_t N, uint32_t d, int mode,
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
            cs[row][col] = (gc < N && gk < d16) ? ldf(C[(size_t)gc * d + gk]) : 0.f;
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
        const float *x = Q + (size_t)gq * d;
        const T *y = C + (size_t)gc * d;
        for (uint32_t i = d16; i < d; i++) {
            if (mode == 0) { float df = __fsub_rn(x[i], ldf(y[i])); s = __fadd_rn(s, __fmul_rn(df, df)); }
            else s = __fadd_rn(s, __fmul_rn(x[i], ldf(y[i])));
        }
        float v = __fadd_rn(s, t);
        if (mode == 1) v = __fsub_rn(1.0f, v);
        else if (mode == 2) v = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(v, xnorm[gq]), ysqrt[gc]));
        D[(size_t)gq * ldD + gc] = v;
    }
  }
}

// half-warp per row: lane l (< 16) is lance's accumulator lane l
template <class TX, class TY>
__device__ __forceinline__ float halfwarp_dot(const TX *__restrict__ x, const TY *__restrict__ y,
                                               uint32_t d, int hl, unsigned hmask, int hbase)
{
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    for (uint32_t k = hl; k < d16; k += 16) a = __fadd_rn(a, __fmul_rn(ldf(x[k]), ldf(y[k])));
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) s = __fadd_rn(s, __fmul_rn(ldf(x[i]), ldf(y[i])));
    return __fadd_rn(s, t);
}
template <class TY>
__device__ __forceinline__ float halfwarp_l2(const float *__restrict__ x, const TY *__restrict__ y,
                                              uint32_t d, int hl, unsigned hmask, int hbase)
{
    const uint32_t d16 = d & ~15u;
    float a = 0.f;
    uint32_t k = hl;
    for (; k + 7 * 16 < d16; k += 8 * 16) {             // eight independent loads of each operand in flight
        float xv[8], yv[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { xv[u] = x[k + 16 * u]; yv[u] = ldf(y[k + 16 * u]); }
#pragma unroll
        for (int u = 0; u < 8; u++) { const float df = __fsub_rn(xv[u], yv[u]); a = __fadd_rn(a, __fmul_rn(df, df)); }
    }
    for (; k < d16; k += 16) { float df = __fsub_rn(x[k], ldf(y[k])); a = __fadd_rn(a, __fmul_rn(df, df)); }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; l++) t = __fadd_rn(t, __shfl_sync(hmask, a, hbase + l));
    float s = 0.f;
    for (uint32_t i = d16; i < d; i++) { float df = __fsub_rn(x[i], ldf(y[i])); s = __fadd_rn(s, __fmul_rn(df, df)); }
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

template <class T>
__global__ void row_norms_kernel(const T *__restrict__ X, uint64_t n, uint32_t d, float *__restrict__ out)
{
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 31, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    if (row >= n) return;                               // whole half-warp exits together
    const T *x = X + row * d;
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

template <class T>
__global__ void pair_distance_kernel(const float *__restrict__ Q, const T *__restrict__ V,
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
    const float *x = Q + (size_t)q * d;
    const T *y = V + ps * d;
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

// pair_distance_kernel's values when the stored rows are in pinned host memory, read through their mapped device alias
// over PCIe.  Each warp owns a run of consecutive (query, candidate) pairs and walks it in steps: step s is one chunk of
// the rows of two pairs, copied by the whole warp into a shared-memory ring slot with cp.async 16-byte requests (one
// instruction = 512 contiguous bytes of a row, where halfwarp_l2's reads would be 64-byte pieces), RH_STAGES - 1 steps
// in flight while the next one is reduced (RH_STAGES 2, 4 and 8 all read at 88-94 % of the pinned memcpy rate on an
// H100 80GB HBM3, 2 the fastest: DESIGN.md section 7).  Half-warp h then reduces pair 2j + h from shared memory with the
// same lane accumulators, lane sum, remainder and roundings as pair_distance_kernel.  Rows are `stride` floats apart (dim rounded up
// to 4, so every row starts 16-byte aligned); a chunk is a multiple of 16 floats, so each lane's accumulator sees its
// dims in lance's order across chunks and the remainder dims [d16, d) all lie in the last chunk.
constexpr int RH_WARPS = 4, RH_STAGES = 2;
constexpr uint32_t RH_CHUNK_MAX = 1024;             // floats of a row per step: at most 64 KB of ring per CTA

__global__ void __launch_bounds__(RH_WARPS * 32) refine_host_kernel(
    const float *__restrict__ Q, const float *V, uint32_t stride, const uint64_t *__restrict__ pos, uint64_t npairs,
    uint32_t nc, uint32_t d, int metric, uint32_t chunk, uint32_t nchunks, uint32_t per_warp, float *__restrict__ out)
{
    pdl_entry();
    extern __shared__ __align__(16) float rh_ring[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, h = lane >> 4, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    const uint64_t p0 = ((uint64_t)blockIdx.x * RH_WARPS + warp) * per_warp;
    if (p0 >= npairs) return;                                    // the whole warp
    const uint64_t p1 = min(p0 + per_warp, npairs);
    const uint32_t nsteps = (uint32_t)((p1 - p0 + 1) / 2) * nchunks, d16 = d & ~15u;
    float *ring = rh_ring + (size_t)warp * RH_STAGES * 2 * chunk;
    const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring);
    // step s -> slot s % RH_STAGES: chunk s % nchunks of the rows of pairs p0 + 2 (s / nchunks) + {0, 1}.  Every lane
    // commits one group per step, empty or not, so that wait_group counts steps.
    auto issue = [&](uint32_t s) {
        if (s < nsteps) {
            const uint32_t j = s / nchunks, k0 = (s % nchunks) * chunk, len = min(chunk, stride - k0);
            for (int r = 0; r < 2; r++) {
                const uint64_t pr = p0 + 2 * j + r;
                const uint64_t ps = pr < p1 ? pos[pr] : UINT64_MAX;
                if (ps == UINT64_MAX) continue;
                const float *src = V + ps * stride + k0;
                const uint32_t dst = ring_s + ((s % RH_STAGES) * 2 + r) * chunk * 4;
                for (uint32_t o = (uint32_t)lane * 4; o < len; o += 128)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + o * 4), "l"(src + o) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (uint32_t s = 0; s < RH_STAGES - 1; s++) issue(s);
    float a0 = 0.f, a1 = 0.f;                    // lane accumulators: l2 / dot in a0; cosine yy in a0, xy in a1
    for (uint32_t s = 0; s < nsteps; s++) {
        issue(s + RH_STAGES - 1);                // into the slot step s - 1 used, released by the last __syncwarp
        asm volatile("cp.async.wait_group %0;" ::"n"(RH_STAGES - 1) : "memory");
        __syncwarp();                            // every lane's copies of step s are in place
        const uint32_t c = s % nchunks, k0 = c * chunk;
        const uint64_t pr = p0 + 2 * (s / nchunks) + h;
        const uint64_t ps = pr < p1 ? pos[pr] : UINT64_MAX;      // uniform over the half-warp
        const float *y = ring + ((s % RH_STAGES) * 2 + h) * chunk;        // y[k - k0]: dim k of the row
        const float *x = Q + (size_t)(pr / nc) * d;
        if (ps != UINT64_MAX) {
            for (uint32_t k = k0 + hl; k < min(k0 + chunk, d16); k += 16) {
                const float xv = x[k], yv = y[k - k0];
                if (metric == LGPU_L2) { const float df = __fsub_rn(xv, yv); a0 = __fadd_rn(a0, __fmul_rn(df, df)); }
                else if (metric == LGPU_DOT) a0 = __fadd_rn(a0, __fmul_rn(xv, yv));
                else { a0 = __fadd_rn(a0, __fmul_rn(yv, yv)); a1 = __fadd_rn(a1, __fmul_rn(xv, yv)); }
            }
        }
        if (c == nchunks - 1 && ps != UINT64_MAX) {              // the row's last chunk: lane sum, remainder, metric
            float t0 = 0.f, t1 = 0.f;
#pragma unroll
            for (int l = 0; l < 16; l++) {
                t0 = __fadd_rn(t0, __shfl_sync(hmask, a0, hbase + l));
                t1 = __fadd_rn(t1, __shfl_sync(hmask, a1, hbase + l));
            }
            float s0 = 0.f, s1 = 0.f;
            for (uint32_t i = d16; i < d; i++) {
                const float xv = x[i], yv = y[i - k0];
                if (metric == LGPU_L2) { const float df = __fsub_rn(xv, yv); s0 = __fadd_rn(s0, __fmul_rn(df, df)); }
                else if (metric == LGPU_DOT) s0 = __fadd_rn(s0, __fmul_rn(xv, yv));
                else { s0 = __fadd_rn(s0, __fmul_rn(yv, yv)); s1 = __fadd_rn(s1, __fmul_rn(xv, yv)); }
            }
            float v;
            if (metric == LGPU_L2) v = __fadd_rn(s0, t0);
            else if (metric == LGPU_DOT) v = __fsub_rn(1.0f, __fadd_rn(s0, t0));
            else {   // cosine_scalar: 1 - xy / |x| / sqrt(yy)
                const float xn = sqrtf(halfwarp_dot(x, x, d, hl, hmask, hbase));
                v = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(__fadd_rn(s1, t1), xn), sqrtf(__fadd_rn(s0, t0))));
            }
            if (hl == 0) out[pr] = v;
        } else if (c == nchunks - 1 && pr < p1 && hl == 0) {
            out[pr] = CUDART_INF_F;
        }
        if (c == nchunks - 1) { a0 = 0.f; a1 = 0.f; }
        __syncwarp();                            // slot s % RH_STAGES is read: step s + RH_STAGES may overwrite it
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// one step of the exact MaxSim's min over a row: the running NaN-skipping minimum m after the pair of query vector i and
// stored vector j, cosd = 1 - xy / |q_i| / |v_j| (dist_matrix_kernel mode 2's roundings; a NaN c never replaces a number)
__device__ __forceinline__ float mv_min_step(float m, float xy, float xn, float ys)
{
    const float c = __fsub_rn(1.0f, __fdiv_rn(__fdiv_rn(xy, xn), ys));
    return (c < m || m != m) ? c : m;
}

// exact MaxSim re-score of the multivector shortlist, half a warp per (query, candidate row): for each query vector i
// in order, the NaN-skipping min over the row's vectors j of 1 - xy / |q_i| / |v_j| (xy in lance's lane order: the
// same roundings as dist_matrix_kernel mode 2), added onto a sum that starts at 0.0f -- the exact path's bits.  V: the
// stored vectors as kept (T float, or __half converted in registers)
template <class T>
__global__ void mv_rescore_kernel(const float *__restrict__ Q, const uint32_t *__restrict__ q_off, uint32_t qa,
                                  const float *__restrict__ xnorm, const T *__restrict__ V,
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
        for (uint64_t j = j0; j < j1; j++) m = mv_min_step(m, halfwarp_dot(x, V + j * d, d, hl, hmask, hbase), xnorm[i], ysqrt[j]);
        s = __fadd_rn(s, m);
    }
    if (hl == 0) { out[pair] = s; ids[pair] = row_ids ? row_ids[r] : r; }
}

// mv_rescore_kernel's values when the stored vectors are in pinned host memory, read through their mapped device alias
// over PCIe.  One warp per (query, candidate row) pair at a time.  The row is one contiguous run of n_r x d floats;
// the warp copies it in chunks of whole vectors into a shared-memory ring with cp.async 16-byte requests (one
// instruction = 512 contiguous bytes, refine_host_kernel's technique), the next chunk in flight while this one is
// scored.  The query's vectors are taken in blocks of MH_QV: half-warp h keeps the running minima of vectors
// i0 + 32 h + 16 u + l (u = 0, 1) in lane l, updated in order of j by the same mv_min_step as mv_rescore_kernel, and
// the block's minima are added onto the sum in order of i once the row was streamed.  A query of more than MH_QV
// vectors streams the row once per block.  `staged` false (d not a multiple of 4, or a vector longer than a ring slot):
// the half-warps read the mapped alias directly.  fp16 vectors (T = __half) are staged as they are, twice as many per
// slot, and converted in registers by halfwarp_dot: the bits of their exact f32 upcast.
constexpr int MH_WARPS = 4;
constexpr uint32_t MH_QV = 64, MH_SLOT_BYTES = 4096;  // query vectors per block; bytes per ring slot (2 slots per warp)

template <class T>
__global__ void __launch_bounds__(MH_WARPS * 32) mv_rescore_host_kernel(
    const float *__restrict__ Q, const uint32_t *__restrict__ q_off, uint32_t qa, const float *__restrict__ xnorm,
    const T *V, const float *__restrict__ ysqrt, const uint64_t *__restrict__ offsets,
    const uint64_t *__restrict__ row_ids, uint32_t d, uint32_t B, const uint32_t *__restrict__ cand,
    const uint32_t *__restrict__ count, uint32_t cap, bool staged, float *__restrict__ out, uint64_t *__restrict__ ids)
{
    constexpr uint32_t SLOT = MH_SLOT_BYTES / sizeof(T), E16 = 16 / sizeof(T);   // elements per slot, per request
    pdl_entry();
    __shared__ __align__(16) T mh_ring[MH_WARPS][2][SLOT];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, h = lane >> 4, hl = lane & 15, hbase = lane & 16;
    const unsigned hmask = 0xffffu << hbase;
    const uint32_t vps = staged ? SLOT / d : 1;                    // vectors per chunk
    const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(&mh_ring[warp][0][0]);
    const uint64_t npairs = (uint64_t)B * cap, nwarps = (uint64_t)gridDim.x * MH_WARPS;
    for (uint64_t pair = (uint64_t)blockIdx.x * MH_WARPS + warp; pair < npairs; pair += nwarps) {
        const uint32_t b = (uint32_t)(pair / cap), slot = (uint32_t)(pair % cap);
        if (slot >= min(count[b], cap)) {
            if (lane == 0) { out[pair] = CUDART_NAN_F; ids[pair] = UINT64_MAX; }
            continue;
        }
        const uint32_t r = cand[pair];
        const uint64_t j0 = offsets[r], n = offsets[r + 1] - j0;
        const uint32_t nch = staged ? (uint32_t)((n + vps - 1) / vps) : 0;
        const T *row = V + j0 * d;
        // chunk c of the row into ring slot c & 1; every lane commits one group per chunk, empty or not
        auto issue = [&](uint32_t c) {
            if (c < nch) {
                const uint32_t len = (uint32_t)(min((uint64_t)vps, n - (uint64_t)c * vps) * d);
                const T *src = row + (size_t)c * vps * d;
                const uint32_t dst = ring_s + (c & 1) * MH_SLOT_BYTES;
                for (uint32_t o = (uint32_t)lane * E16; o < len; o += 32 * E16)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + o * (uint32_t)sizeof(T)),
                                 "l"(src + o) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        const uint32_t qs = q_off[qa + b], qe = q_off[qa + b + 1];
        float s = 0.f;
        for (uint32_t i0 = qs; i0 < qe; i0 += MH_QV) {
            float m[2] = {CUDART_NAN_F, CUDART_NAN_F};
            // the minima of this half-warp's vectors i0 + 32 h + 16 u + t over stored vectors [j, j + nv) at y
            auto score = [&](const T *y, uint64_t j, uint32_t nv) {
                for (uint32_t v = 0; v < nv; v++) {
                    const float ys = ysqrt[j0 + j + v];
#pragma unroll
                    for (int u = 0; u < 2; u++)
                        for (uint32_t t = 0; t < 16; t++) {
                            const uint32_t i = i0 + 32 * h + 16 * u + t;
                            if (i >= qe) break;                           // uniform over the half-warp
                            const float xy = halfwarp_dot(Q + (size_t)i * d, y + (size_t)v * d, d, hl, hmask, hbase);
                            if ((uint32_t)hl == t) m[u] = mv_min_step(m[u], xy, xnorm[i], ys);
                        }
                }
            };
            if (staged) {
                issue(0);
                for (uint32_t c = 0; c < nch; c++) {
                    issue(c + 1);                         // into the slot chunk c - 1 used, released by the last __syncwarp
                    asm volatile("cp.async.wait_group 1;" ::: "memory");
                    __syncwarp();                         // every lane's copies of chunk c are in place
                    score(&mh_ring[warp][c & 1][0], (uint64_t)c * vps, (uint32_t)min((uint64_t)vps, n - (uint64_t)c * vps));
                    __syncwarp();                         // slot c & 1 is read: chunk c + 2 may overwrite it
                }
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            } else {
                score(row, 0, (uint32_t)n);
            }
            __syncwarp();
#pragma unroll
            for (int g = 0; g < 4; g++)                   // vectors i0 + 16 g + t: half g >> 1, register g & 1
                for (uint32_t t = 0; t < 16; t++) {
                    const float v = __shfl_sync(0xffffffffu, m[g & 1], (g >> 1) * 16 + t);
                    if (i0 + 16 * g + t < qe) s = __fadd_rn(s, v);
                }
        }
        if (lane == 0) { out[pair] = s; ids[pair] = row_ids ? row_ids[r] : r; }
    }
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

template <class T>
void launch_dist_matrix(const float *Q, const T *C, uint32_t B, uint64_t N, uint32_t d, int mode,
                        const float *xnorm, const float *ysqrt, float *D, uint64_t ldD, cudaStream_t st,
                        const uint32_t *only, const uint32_t *gate)
{
    if (B == 0 || N == 0) return;
    // the fix-up pass (`only`) is almost always a no-op: keep its CTA count small
    const uint64_t ct = (N + DM_C - 1) / DM_C;
    dim3 grid((unsigned)std::min<uint64_t>(ct, only ? 16 : ((uint64_t)1 << 30)), (B + DM_Q - 1) / DM_Q);
    launch_k(dist_matrix_kernel<T>, grid, dim3(DM_THREADS), 0, st, Q, C, B, N, d, mode, xnorm, ysqrt, D, ldD, only, gate); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

template <class T>
void launch_row_norms(const T *X, uint64_t n, uint32_t d, float *out, cudaStream_t st)
{
    if (n == 0) return;
    uint64_t threads = n * 16;
    row_norms_kernel<T><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(X, n, d, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_normalize(const float *X, uint32_t B, uint32_t d, float *out, cudaStream_t st)
{
    if (B == 0) return;
    uint64_t threads = (uint64_t)B * 16;
    launch_k(normalize_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, X, B, d, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

template <class T>
void launch_pair_distance(const float *Q, const T *V, const uint64_t *pos, uint32_t B, uint32_t nc,
                          uint32_t d, int metric, float *out, cudaStream_t st)
{
    if (B == 0 || nc == 0) return;
    uint64_t threads = (uint64_t)B * nc * 16;
    launch_k(pair_distance_kernel<T>, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, Q, V, pos, B, nc, d, metric, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_refine_host(const float *Q, const float *V, uint32_t stride, const uint64_t *pos, uint32_t B, uint32_t nc,
                        uint32_t d, int metric, float *out, int num_sms, cudaStream_t st)
{
    const uint64_t npairs = (uint64_t)B * nc;
    if (npairs == 0) return;
    const uint32_t chunk = std::min<uint32_t>((d + 15) & ~15u, RH_CHUNK_MAX), nchunks = (d + chunk - 1) / chunk;
    // an even run of pairs per warp, sized so that the grid is about 16 warps per SM (a few waves at most)
    const uint64_t want = (uint64_t)std::max(num_sms, 1) * 16;
    const uint32_t per_warp = (uint32_t)std::max<uint64_t>(2, ((npairs + want - 1) / want + 1) & ~1ull);
    const uint64_t warps = (npairs + per_warp - 1) / per_warp;
    const size_t smem = (size_t)RH_WARPS * RH_STAGES * 2 * chunk * 4;
    if (smem > 48 * 1024)
        LGPU_CUDA(cudaFuncSetAttribute(refine_host_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    launch_k(refine_host_kernel, dim3((unsigned)((warps + RH_WARPS - 1) / RH_WARPS)), dim3(RH_WARPS * 32), smem, st, Q,
             V, stride, pos, npairs, nc, d, metric, chunk, nchunks, per_warp, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

// staged: every vector a whole number of 16-byte requests (d a multiple of 4 floats or 8 halves) that fits a slot
template <class T>
void launch_mv_rescore_host(const float *Q, const uint32_t *q_off, uint32_t qa, const float *xnorm, const T *V,
                            const float *ysqrt, const uint64_t *offsets, const uint64_t *row_ids, uint32_t d, uint32_t B,
                            const uint32_t *cand, const uint32_t *count, uint32_t cap, float *out, uint64_t *ids,
                            int num_sms, cudaStream_t st)
{
    if (B == 0 || cap == 0) return;
    const bool staged = ((size_t)d * sizeof(T)) % 16 == 0 && (size_t)d * sizeof(T) <= MH_SLOT_BYTES &&
                        ((uintptr_t)V & 15) == 0;
    const uint64_t npairs = (uint64_t)B * cap;
    const unsigned grid = (unsigned)std::min<uint64_t>((npairs + MH_WARPS - 1) / MH_WARPS, (uint64_t)std::max(num_sms, 1) * 16);
    launch_k(mv_rescore_host_kernel<T>, dim3(grid), dim3(MH_WARPS * 32), 0, st, Q, q_off, qa, xnorm, V, ysqrt, offsets,
             row_ids, d, B, cand, count, cap, staged, out, ids); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

#define LGPU_ROW_TYPE(T)                                                                                                 \
    template void launch_dist_matrix<T>(const float *, const T *, uint32_t, uint64_t, uint32_t, int, const float *,     \
                                        const float *, float *, uint64_t, cudaStream_t, const uint32_t *,               \
                                        const uint32_t *);                                                              \
    template void launch_row_norms<T>(const T *, uint64_t, uint32_t, float *, cudaStream_t);                            \
    template void launch_pair_distance<T>(const float *, const T *, const uint64_t *, uint32_t, uint32_t, uint32_t, int, \
                                          float *, cudaStream_t);
LGPU_ROW_TYPE(float)
LGPU_ROW_TYPE(__half)
#undef LGPU_ROW_TYPE

template <class T>
void launch_mv_rescore(const float *Q, const uint32_t *q_off, uint32_t qa, const float *xnorm, const T *V,
                       const float *ysqrt, const uint64_t *offsets, const uint64_t *row_ids, uint32_t d, uint32_t B,
                       const uint32_t *cand, const uint32_t *count, uint32_t cap, float *out, uint64_t *ids,
                       cudaStream_t st)
{
    if (B == 0 || cap == 0) return;
    const uint64_t threads = (uint64_t)B * cap * 16;
    launch_k(mv_rescore_kernel<T>, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, Q, q_off, qa, xnorm, V,
             ysqrt, offsets, row_ids, d, B, cand, count, cap, out, ids); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

#define LGPU_MV_ROW_TYPE(T)                                                                                              \
    template void launch_mv_rescore<T>(const float *, const uint32_t *, uint32_t, const float *, const T *,             \
                                       const float *, const uint64_t *, const uint64_t *, uint32_t, uint32_t,           \
                                       const uint32_t *, const uint32_t *, uint32_t, float *, uint64_t *, cudaStream_t); \
    template void launch_mv_rescore_host<T>(const float *, const uint32_t *, uint32_t, const float *, const T *,        \
                                            const float *, const uint64_t *, const uint64_t *, uint32_t, uint32_t,      \
                                            const uint32_t *, const uint32_t *, uint32_t, float *, uint64_t *, int,     \
                                            cudaStream_t);
LGPU_MV_ROW_TYPE(float)
LGPU_MV_ROW_TYPE(__half)
#undef LGPU_MV_ROW_TYPE

}  // namespace lgpu
