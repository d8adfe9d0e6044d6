// hamming.cu -- the SIMT side of binary (packed uint8) vector search: operand packing, the dense Hamming kernel
// (small batches, prefilters / distance ranges, the fix-up of overflowed queries) and the small helpers of the
// tensor-core path's orchestration (api.cu binary_search_device).  The tensor-core kernel itself is the b1
// instantiation of gemm_dist_kernel (gemm.cu).
//
// Rows are stored zero-padded to a multiple of 32 bytes (one k256 b1 wgmma slice): zero bits add nothing to
// popc(q AND x) nor to popc(q XOR x), so every distance is the one over the caller's nbytes.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int HD_THREADS = 256;   // one row per thread
constexpr int HD_Q = 8;           // queries per work item: each row word loaded once serves 8 queries

// one warp per row
__global__ void ham_pack_kernel(const uint8_t *__restrict__ src, uint64_t src_stride, uint32_t nbytes, uint64_t n,
                                uint8_t *__restrict__ dst, uint32_t nbytes_pad, uint32_t *__restrict__ pop)
{
    pdl_entry();
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (row >= n) return;
    const uint8_t *s = src + row * src_stride;
    uint8_t *d = dst + row * nbytes_pad;
    uint32_t p = 0;
    for (uint32_t c = lane; c < nbytes_pad; c += 32) {
        const uint32_t b = c < nbytes ? s[c] : 0u;
        d[c] = (uint8_t)b;
        p += __popc(b);
    }
    p = __reduce_add_sync(0xffffffffu, p);
    if (lane == 0) pop[row] = p;
}

// Work item w = (group of HD_Q query slots, tile of HD_THREADS rows), walked tile-major inside a group so the blocks
// in flight share the group's query words in L1/L2.  Persistent grid: with a device query count of 0 (a fix-up pass
// with nothing flagged) every block returns at once.
__global__ void __launch_bounds__(HD_THREADS) ham_dense_kernel(const uint8_t *__restrict__ Q, const uint8_t *__restrict__ X,
                                                               uint32_t B, uint64_t N, uint32_t nbytes_pad,
                                                               float *__restrict__ D, uint64_t ldD,
                                                               const uint32_t *__restrict__ qlist,
                                                               const uint32_t *__restrict__ qcount)
{
    pdl_entry();
    const uint32_t nq = qcount ? *qcount : B;
    const uint64_t ntile = (N + HD_THREADS - 1) / HD_THREADS;
    const uint64_t total = (uint64_t)((nq + HD_Q - 1) / HD_Q) * ntile;
    const uint32_t nw = nbytes_pad / 16;
    for (uint64_t w = blockIdx.x; w < total; w += gridDim.x) {
        const uint32_t g0 = (uint32_t)(w / ntile) * HD_Q;
        const uint64_t x = (w % ntile) * HD_THREADS + threadIdx.x;
        if (x >= N) continue;
        uint32_t qi[HD_Q];
        int acc[HD_Q];
#pragma unroll
        for (int g = 0; g < HD_Q; g++) {
            const uint32_t s = g0 + g;
            qi[g] = s < nq ? (qlist ? qlist[s] : s) : 0xffffffffu;
            acc[g] = 0;
        }
        const uint4 *xr = reinterpret_cast<const uint4 *>(X + x * nbytes_pad);
        for (uint32_t c = 0; c < nw; c++) {
            const uint4 v = __ldg(xr + c);
#pragma unroll
            for (int g = 0; g < HD_Q; g++) {
                if (qi[g] == 0xffffffffu) continue;
                const uint4 q = __ldg(reinterpret_cast<const uint4 *>(Q + (size_t)qi[g] * nbytes_pad) + c);
                acc[g] += __popc(v.x ^ q.x) + __popc(v.y ^ q.y) + __popc(v.z ^ q.z) + __popc(v.w ^ q.w);
            }
        }
#pragma unroll
        for (int g = 0; g < HD_Q; g++)
            if (qi[g] != 0xffffffffu) D[(size_t)qi[g] * ldD + x] = (float)acc[g];
    }
}

// chunk c = queries [c chunk, (c + 1) chunk): list[c chunk + i] (i < count[c]) = the chunk-local indices of its flagged
// queries.  One block.
__global__ void __launch_bounds__(1024) ham_flag_list_kernel(const uint32_t *__restrict__ flags, uint32_t B, uint32_t chunk,
                                                             uint32_t *__restrict__ list, uint32_t *__restrict__ count)
{
    pdl_entry();
    const uint32_t nchunks = (B + chunk - 1) / chunk;
    for (uint32_t c = threadIdx.x; c < nchunks; c += blockDim.x) count[c] = 0;
    __syncthreads();
    for (uint32_t q = threadIdx.x; q < B; q += blockDim.x)
        if (flags[q]) {
            const uint32_t c = q / chunk;
            list[c * chunk + atomicAdd(count + c, 1u)] = q - c * chunk;
        }
}

__global__ void ham_threshold_kernel(const float *__restrict__ dist, const uint32_t *__restrict__ cnt, uint32_t B,
                                     uint32_t k, float *__restrict__ thr)
{
    pdl_entry();
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < B) thr[q] = cnt[q] >= k ? dist[(size_t)q * k + k - 1] : __int_as_float(0x7f800000);
}

}  // namespace

void launch_ham_pack(const uint8_t *src, uint64_t src_stride, uint32_t nbytes, uint64_t n, uint8_t *dst,
                     uint32_t nbytes_pad, uint32_t *pop, cudaStream_t st)
{
    if (n == 0) return;
    const uint64_t threads = n * 32;
    launch_k(ham_pack_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, src, src_stride, nbytes, n, dst,
             nbytes_pad, pop); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_ham_dense(const uint8_t *Q, const uint8_t *X, uint32_t B, uint64_t N, uint32_t nbytes_pad, float *D,
                      uint64_t ldD, int num_sms, cudaStream_t st, const uint32_t *qlist, const uint32_t *qcount)
{
    if (B == 0 || N == 0) return;
    const uint64_t items = (uint64_t)((B + HD_Q - 1) / HD_Q) * ((N + HD_THREADS - 1) / HD_THREADS);
    const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(items, (uint64_t)num_sms * 8));
    launch_k(ham_dense_kernel, dim3(grid), dim3(HD_THREADS), 0, st, Q, X, B, N, nbytes_pad, D, ldD, qlist, qcount);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_ham_flag_list(const uint32_t *flags, uint32_t B, uint32_t chunk, uint32_t *list, uint32_t *count,
                          cudaStream_t st)
{
    if (B == 0) return;
    launch_k(ham_flag_list_kernel, dim3(1), dim3(1024), 0, st, flags, B, chunk, list, count); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_ham_threshold(const float *dist, const uint32_t *cnt, uint32_t B, uint32_t k, float *thr, cudaStream_t st)
{
    if (B == 0) return;
    launch_k(ham_threshold_kernel, dim3((B + 127) / 128), dim3(128), 0, st, dist, cnt, B, k, thr); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
