// rowmask.cu -- the live-row bitmap of a handle with deleted rows (lgpu_*_delete, DESIGN.md section 3): one bit per
// row id in [0, id_bound), bit r & 31 of word r >> 5 (the layout of an allow bitmap), set while the id belongs to a
// row of the handle that was not deleted.  A search on such a handle filters by this bitmap, or by its AND with the
// call's own allow bitmap.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int RM_THREADS = 256;

__global__ void rowmask_max_kernel(const uint64_t *ids, uint64_t n, unsigned long long *out)
{
    unsigned long long m = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)RM_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * RM_THREADS)
        m = max(m, (unsigned long long)ids[i]);
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void rowmask_set_kernel(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t first, uint64_t n)
{
    for (uint64_t i = blockIdx.x * (uint64_t)RM_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * RM_THREADS) {
        const uint64_t id = ids ? ids[i] : first + i;
        if (id < nbits) atomicOr(bits + (id >> 5), 1u << (id & 31));
    }
}

// rows whose id is marked and not live: deleted rows an append would make live again
__global__ void rowmask_revived_kernel(const uint32_t *mark, const uint32_t *live, uint64_t nbits, const uint64_t *ids,
                                       uint64_t n, unsigned long long *count)
{
    uint32_t hits = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)RM_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * RM_THREADS) {
        const uint64_t id = ids ? ids[i] : i;
        if (id < nbits && ((mark[id >> 5] & ~live[id >> 5]) >> (id & 31) & 1u)) hits++;
    }
    for (int o = 16; o; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(count, (unsigned long long)hits);
}

// the old value of atomicAnd tells which call cleared a bit: each id is counted once, duplicates and repeats included
__global__ void rowmask_clear_kernel(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t n,
                                     unsigned long long *count)
{
    uint32_t cleared = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)RM_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * RM_THREADS) {
        const uint64_t id = ids[i];
        if (id >= nbits) continue;                          // absent from the handle
        const uint32_t bit = 1u << (id & 31);
        if (atomicAnd(bits + (id >> 5), ~bit) & bit) cleared++;
    }
    for (int o = 16; o; o >>= 1) cleared += __shfl_xor_sync(0xffffffffu, cleared, o);
    if ((threadIdx.x & 31) == 0 && cleared) atomicAdd(count, (unsigned long long)cleared);
}

__global__ void rowmask_and_kernel(const uint32_t *a, const uint32_t *b, uint64_t words, uint32_t *out)
{
    for (uint64_t i = blockIdx.x * (uint64_t)RM_THREADS + threadIdx.x; i < words; i += (uint64_t)gridDim.x * RM_THREADS)
        out[i] = a[i] & b[i];
}

unsigned rm_grid(uint64_t n) { return (unsigned)std::min<uint64_t>((n + RM_THREADS - 1) / RM_THREADS, 4096); }

}  // namespace

void launch_rowmask_max(const uint64_t *ids, uint64_t n, unsigned long long *out, cudaStream_t st)
{
    if (n == 0) return;
    rowmask_max_kernel<<<rm_grid(n), RM_THREADS, 0, st>>>(ids, n, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rowmask_set(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t first, uint64_t n, cudaStream_t st)
{
    if (n == 0) return;
    rowmask_set_kernel<<<rm_grid(n), RM_THREADS, 0, st>>>(bits, nbits, ids, first, n); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rowmask_revived(const uint32_t *mark, const uint32_t *live, uint64_t nbits, const uint64_t *ids, uint64_t n,
                            unsigned long long *count, cudaStream_t st)
{
    if (n == 0) return;
    rowmask_revived_kernel<<<rm_grid(n), RM_THREADS, 0, st>>>(mark, live, nbits, ids, n, count); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rowmask_clear(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t n, unsigned long long *count,
                          cudaStream_t st)
{
    if (n == 0) return;
    rowmask_clear_kernel<<<rm_grid(n), RM_THREADS, 0, st>>>(bits, nbits, ids, n, count); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rowmask_and(const uint32_t *a, const uint32_t *b, uint64_t words, uint32_t *out, cudaStream_t st)
{
    if (words == 0) return;
    rowmask_and_kernel<<<rm_grid(words), RM_THREADS, 0, st>>>(a, b, words, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
