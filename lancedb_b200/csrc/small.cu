// small.cu -- the low-latency form of K2+K3 for tiny batches (B * nprobes <= ~1000 probe slots: a single query, or
// the handful a micro-batch collects).  The batched kernels (group.cu -> scan3.cu / scan2.cu -> finalize) amortise
// their ~25 launches over a thousand queries; one query pays them all.
// Here every (query, probed partition) pair is one CTA, which is the reference's own decomposition
// [lance, recalled: ANNIvfSubIndexExec runs per partition; SURVEY.md 8a rows a4-a7]:
//     r   = q - centroid[p]                      (L2 / cosine; the query itself for dot)
//     LUT = the m x 256 f32 distance table, in shared memory (96 KB at m = 96)
//     d_j = sum_i LUT[i][code_i(j)], sequentially in i, metric post-scale
// in the oracle's arithmetic (`subvec_l2` tree entries, sequential row sums), so the distances are bit-identical to
// scan2.cu's.  They go to fixed-stride segments of dist_out; the usual K4 (select.cu, mode 0) follows.  Launches per
// search: coarse distances, select, this kernel, select.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int SM_THREADS = 256;

template <int DSUB, bool DOT>
__global__ void __launch_bounds__(SM_THREADS) small_scan_kernel(SmallScanArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(16) unsigned char ssm[];
    float *lut = reinterpret_cast<float *>(ssm);                 // [m][256]
    float *res = lut + (size_t)a.m * 256;                        // [dim]
    const uint32_t slot = blockIdx.x;
    const uint32_t q = slot / a.nprobes;
    const int tid = threadIdx.x;
    if (tid == 0) a.seg_off[slot] = (uint64_t)slot * a.seg_stride;
    const uint64_t pp = a.probes[slot];
    if (pp >= a.nlist) return;                                   // unused probe slot
    const uint32_t p = (uint32_t)pp;
    const uint32_t n_p = a.part_n[p];
    if (n_p == 0) return;
    const float *qv = a.queries + (size_t)q * a.dim, *cen = a.centroids + (size_t)p * a.dim;
    for (uint32_t t = tid; t < a.dim; t += SM_THREADS) res[t] = DOT ? qv[t] : __fsub_rn(qv[t], cen[t]);
    __syncthreads();
    // the distance table: thread -> code, loop over sub-spaces (codebook tiled [nch][256][8][dsub])
    for (uint32_t i = 0; i < a.m; i++) {
        float r[DSUB], cv[DSUB];
        const float *cb = a.cb_tiled + (((size_t)(i >> 3) * 256 + tid) * 8 + (i & 7)) * DSUB;
#pragma unroll
        for (int t = 0; t < DSUB; t++) { r[t] = res[i * DSUB + t]; cv[t] = cb[t]; }
        lut[i * 256 + tid] = DOT ? subvec_dot_dist<DSUB>(r, cv) : subvec_l2<DSUB>(r, cv);
    }
    __syncthreads();
    // the scan: one row per thread and step, the row's skewed 8-byte code words block by block (retile.cu)
    const uint2 *cs = reinterpret_cast<const uint2 *>(a.codes + a.code_base[p]);
    const uint32_t npad = a.part_npad[p];
    float *out = a.dist_out + (uint64_t)slot * a.seg_stride;
    const float mcorr = (float)(a.m - 1);
    for (uint32_t row = tid; row < n_p; row += SM_THREADS) {
        const int sig = (int)(row & 7);
        float acc = 0.f;
        for (uint32_t blk = 0; blk <= a.nch; blk++) {
            const uint2 w = __ldg(cs + (size_t)blk * npad + row);
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const int i = (int)(blk * 8) + e - sig;          // sub-space of stream position 8 blk + e
                if (i >= 0 && i < (int)a.m) {
                    const uint32_t word = e < 4 ? w.x : w.y;
                    acc = __fadd_rn(acc, lut[i * 256 + ((word >> (8 * (e & 3))) & 0xffu)]);
                }
            }
        }
        if (a.metric == LGPU_COSINE) acc = __fmul_rn(acc, 0.5f);
        else if (a.metric == LGPU_DOT) acc = __fsub_rn(acc, mcorr);
        out[row] = acc;
    }
}

}  // namespace

size_t small_scan_smem(uint32_t m, uint32_t dim) { return ((size_t)m * 256 + dim) * sizeof(float); }

void launch_small_scan(const SmallScanArgs &a, uint32_t dsub, uint32_t slots, cudaStream_t st)
{
    if (slots == 0) return;
    const size_t smem = small_scan_smem(a.m, a.dim);
#define LGPU_SMALL(D)                                                                                          \
    do {                                                                                                       \
        auto k0 = small_scan_kernel<D, false>; auto k1 = small_scan_kernel<D, true>;                            \
        auto kern = a.metric == LGPU_DOT ? k1 : k0;                                                             \
        LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));          \
        launch_k(kern, dim3(slots), dim3(SM_THREADS), smem, st, a); LGPU_COUNT_LAUNCH();                                          \
    } while (0)
    switch (dsub) {
    case 1: LGPU_SMALL(1); break;
    case 2: LGPU_SMALL(2); break;
    case 4: LGPU_SMALL(4); break;
    case 8: LGPU_SMALL(8); break;
    case 16: LGPU_SMALL(16); break;
    case 32: LGPU_SMALL(32); break;
    default: set_error("unsupported PQ sub-vector length"); throw Failure{LGPU_INVALID_INPUT};
    }
#undef LGPU_SMALL
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
