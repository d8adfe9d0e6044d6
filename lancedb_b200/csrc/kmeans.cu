// kmeans.cu -- index TRAINING on the GPU (SURVEY.md 8f-2): Lloyd iterations for the IVF centroids and for the 256-entry
// PQ codebooks of all m sub-spaces.  The reference builds IVF_PQ through lance (parameters at
// rust/lancedb/src/table/create_index.rs:283-303, rust/lancedb/src/index/vector.rs:246-319; "GPU support in building
// vector index", python/python/lancedb/table.py:2883-2937); training quality is not part of search parity -- the CUDA
// path and the oracle consume whatever arrays come out -- so these kernels follow plain Lloyd (random-sample init by the
// caller, empty clusters keep their previous centre; lance's hierarchical variant above 256 lists
// [python/python/tests/test_index.py:378] is not reproduced) and only have to be good k-means.
//   assignment (IVF)  : the search's own coarse step (api.cu): tensor-core GEMM scores + coarse_finish_kernel with k = 1, i.e.
//                       the exact nearest centre in lance's arithmetic -- a training row is assigned where a query equal
//                       to it would probe first;
//   update (IVF)      : rows bucketed by centre (counting sort), one CTA per centre sums its rows in f64, each bucket
//                       sorted first so the sum does not depend on the order the atomics happened to run in;
//   assignment (PQ)   : pq_encode_kernel (build.cu) against a zero centroid: arg-min of the L2 table entry per sub-space;
//   update (PQ)       : f64 atomics into [m][256][dsub] sums (24 576 small clusters).
#include "kernels.cuh"

namespace lgpu {

namespace {

__global__ void km_count_kernel(const uint64_t *__restrict__ assign, uint64_t n, uint32_t k, uint32_t *__restrict__ counts)
{
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n && assign[r] < k) atomicAdd(counts + (uint32_t)assign[r], 1u);
}

// single CTA: exclusive prefix of counts -> offsets[k+1], cursor[c] = offsets[c]
__global__ void km_scan_kernel(const uint32_t *__restrict__ counts, uint32_t k, uint32_t *__restrict__ offsets,
                               uint32_t *__restrict__ cursor)
{
    __shared__ uint32_t s_part[1024];
    const int tid = threadIdx.x;
    const uint32_t per = (k + 1023) / 1024;
    const uint32_t b = tid * per, e = min(k, b + per);
    uint32_t sum = 0;
    for (uint32_t c = b; c < e; c++) sum += counts[c];
    s_part[tid] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const uint32_t t = tid >= o ? s_part[tid - o] : 0;
        __syncthreads();
        s_part[tid] += t;
        __syncthreads();
    }
    uint32_t run = s_part[tid] - sum;
    for (uint32_t c = b; c < e; c++) { offsets[c] = run; cursor[c] = run; run += counts[c]; }
    if (tid == 1023) offsets[k] = s_part[1023];
}

__global__ void km_fill_kernel(const uint64_t *__restrict__ assign, uint64_t n, uint32_t k, uint32_t *__restrict__ cursor,
                               uint32_t *__restrict__ rows)
{
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n && assign[r] < k) rows[atomicAdd(cursor + (uint32_t)assign[r], 1u)] = (uint32_t)r;
}

constexpr int KM_THREADS = 256, KM_SORT_MAX = 4096, KM_DPT = 16;      // dims per thread: dim <= 4096
__global__ void __launch_bounds__(KM_THREADS) km_update_kernel(const float *__restrict__ x, uint32_t dim,
                                                               const uint32_t *__restrict__ rows,
                                                               const uint32_t *__restrict__ offsets,
                                                               float *__restrict__ centroids)
{
    __shared__ uint32_t s_rows[KM_SORT_MAX];
    const uint32_t c = blockIdx.x;
    const uint32_t b = offsets[c], cnt = offsets[c + 1] - b;
    if (cnt == 0) return;                                           // empty cluster: keep the previous centre
    const int tid = threadIdx.x;
    const bool sorted = cnt <= KM_SORT_MAX;
    if (sorted) {                                                   // a fixed summation order: ascending row
        uint32_t n2 = 2;
        while (n2 < cnt) n2 <<= 1;
        for (uint32_t i = tid; i < n2; i += KM_THREADS) s_rows[i] = i < cnt ? rows[b + i] : 0xffffffffu;
        __syncthreads();
        for (uint32_t size = 2; size <= n2; size <<= 1) {
            for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                for (uint32_t i = tid; i < (n2 >> 1); i += KM_THREADS) {
                    const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                    const uint32_t a0 = s_rows[lo], a1 = s_rows[hi];
                    if ((a1 < a0) == ((lo & size) == 0)) { s_rows[lo] = a1; s_rows[hi] = a0; }
                }
                __syncthreads();
            }
        }
    }
    double acc[KM_DPT];
#pragma unroll
    for (int j = 0; j < KM_DPT; j++) acc[j] = 0.0;
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t r = sorted ? s_rows[i] : rows[b + i];
        const float *xr = x + (size_t)r * dim;
#pragma unroll
        for (int j = 0; j < KM_DPT; j++) {
            const uint32_t t = (uint32_t)j * KM_THREADS + tid;
            if (t < dim) acc[j] += (double)xr[t];
        }
    }
#pragma unroll
    for (int j = 0; j < KM_DPT; j++) {
        const uint32_t t = (uint32_t)j * KM_THREADS + tid;
        if (t < dim) centroids[(size_t)c * dim + t] = (float)(acc[j] / (double)cnt);
    }
}

__global__ void km_inertia_kernel(const float *__restrict__ dist, uint64_t n, double *__restrict__ out)
{
    __shared__ double s[256];
    double v = 0.0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float d = dist[i];
        if (d == d && d < 3.0e38f) v += (double)d;
    }
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) atomicAdd(out, s[0]);
}

// ---- PQ codebooks ----
__global__ void pq_accum_kernel(const float *__restrict__ x, const unsigned char *__restrict__ codes, uint64_t n, uint32_t dim,
                                uint32_t m, uint32_t dsub, double *__restrict__ sums, uint32_t *__restrict__ counts)
{
    const uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * m) return;
    const uint64_t r = idx / m;
    const uint32_t i = (uint32_t)(idx - r * m);
    const uint32_t c = codes[idx];
    const float *xs = x + r * dim + (size_t)i * dsub;
    double *dst = sums + ((size_t)i * 256 + c) * dsub;
    for (uint32_t t = 0; t < dsub; t++) atomicAdd(dst + t, (double)xs[t]);
    atomicAdd(counts + (size_t)i * 256 + c, 1u);
}

__global__ void pq_finish_kernel(const double *__restrict__ sums, const uint32_t *__restrict__ counts, uint32_t entries,
                                 uint32_t dsub, float *__restrict__ codebook)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= entries) return;
    const uint32_t cnt = counts[e];
    if (cnt == 0) return;                                           // unused codeword: keep it
    for (uint32_t t = 0; t < dsub; t++) codebook[(size_t)e * dsub + t] = (float)(sums[(size_t)e * dsub + t] / (double)cnt);
}

}  // namespace

void launch_kmeans_update(const uint64_t *assign, const float *x, uint64_t n, uint32_t dim, uint32_t k, uint32_t *counts,
                          uint32_t *offsets, uint32_t *cursor, uint32_t *rows, float *centroids, cudaStream_t st)
{
    if (n == 0 || k == 0) return;
    if (dim > (uint32_t)KM_THREADS * KM_DPT || n >= (1ull << 32)) {
        set_error("k-means training supports dim <= 4096 and fewer than 2^32 training rows");
        throw Failure{LGPU_INVALID_INPUT};
    }
    LGPU_CUDA(cudaMemsetAsync(counts, 0, (size_t)k * 4, st));
    const unsigned g = (unsigned)((n + 255) / 256);
    km_count_kernel<<<g, 256, 0, st>>>(assign, n, k, counts); LGPU_COUNT_LAUNCH();
    km_scan_kernel<<<1, 1024, 0, st>>>(counts, k, offsets, cursor); LGPU_COUNT_LAUNCH();
    km_fill_kernel<<<g, 256, 0, st>>>(assign, n, k, cursor, rows); LGPU_COUNT_LAUNCH();
    km_update_kernel<<<k, KM_THREADS, 0, st>>>(x, dim, rows, offsets, centroids); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_kmeans_inertia(const float *dist, uint64_t n, double *out, cudaStream_t st)
{
    LGPU_CUDA(cudaMemsetAsync(out, 0, 8, st));
    if (n == 0) return;
    km_inertia_kernel<<<(unsigned)std::min<uint64_t>((n + 255) / 256, 1024), 256, 0, st>>>(dist, n, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_pq_update(const float *x, const unsigned char *codes, uint64_t n, uint32_t dim, uint32_t m, double *sums,
                      uint32_t *counts, float *codebook, cudaStream_t st)
{
    if (n == 0) return;
    const uint32_t dsub = dim / m, entries = m * 256;
    LGPU_CUDA(cudaMemsetAsync(sums, 0, (size_t)entries * dsub * 8, st));
    LGPU_CUDA(cudaMemsetAsync(counts, 0, (size_t)entries * 4, st));
    const uint64_t total = n * m;
    pq_accum_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, codes, n, dim, m, dsub, sums, counts); LGPU_COUNT_LAUNCH();
    pq_finish_kernel<<<(entries + 255) / 256, 256, 0, st>>>(sums, counts, entries, dsub, codebook); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
