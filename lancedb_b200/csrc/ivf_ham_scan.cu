// ivf_ham_scan.cu -- binary IVF_FLAT: the probed partitions of packed binary rows scanned exactly on the binary tensor
// cores.
//
// A stored row x is nbytes packed bytes zero-padded to nbytes_pad (a multiple of 32 bytes = one k256 b1 MMA step), with
// popc(x) computed at open; a query q is packed the same way (launch_ham_pack).  Zero bits add nothing to either
// popcount, so for every row of a probed partition
//     d = popc(q) + popc(x) - 2 popc(q AND x) = popc(q XOR x)
// is the exact Hamming distance over the caller's nbytes, written as f32 (exact: d <= 2^24).  The scan reads the tile
// queue of the other IVF scans (group.cu): a tile is <= HAM_ROWS_TILE rows of one partition and the <= 8 probe slots that
// probe it.  Each warp owns 32-row groups (two m16 tiles) of the tile, 8 warps stepping by 256 rows; per 256-bit K step it
// issues 2 mma.m16n8k256 b1 AND.POPC (one per m-tile; rows = M, the tile's query slots = N = 8).  Lane (g, t) loads 8
// bytes at offset 8 t of the step's 32 bytes of rows g, g + 8, g + 16, g + 24 and of query slot g: fragment half h gets
// word 2 t + h, the same bijection of K for A and B, so the popcounts are those of the true bit order (the layout of
// rq_scan.cu with one plane).  Two MMAs per 32 row bytes are far below the tensor cores' rate, so operands come straight
// from global memory with no shared-memory staging: the kernel streams the probed rows once per tile.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int HAM_NT = 256;                 // 8 warps x 32 rows per pass; HAM_ROWS_TILE / 256 passes per tile

__device__ __forceinline__ void ham_mma(uint32_t (&d)[4], uint2 a_lo, uint2 a_hi, uint2 b)
{
    asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a_lo.x), "r"(a_hi.x), "r"(a_lo.y), "r"(a_hi.y), "r"(b.x), "r"(b.y));
}

// One warp's 32 rows [r0, r0 + 32) of a tile against the tile's <= 8 query slots.  a_lo = row 16 m + g,
// a_hi = row 16 m + g + 8: fragment registers a0 / a1 are (row g / g + 8, K half 0), a2 / a3 (K half 1), b0 / b1 (K half
// 0 / 1).  Rows past the tile are re-read (clamped), never written.
__device__ __forceinline__ void ham_rows(const HamScanArgs &a, const TileDesc &T, uint32_t r0, uint32_t row_end, int lane)
{
    const int g = lane >> 2, t = lane & 3;
    const uint32_t nbp = a.nbytes_pad;
    const uint2 *arow[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t r = min(r0 + (uint32_t)(g + 8 * i), row_end - 1u);
        arow[i] = reinterpret_cast<const uint2 *>(a.rows + ((uint64_t)T.part_off32 + r) * nbp + 8 * t);
    }
    const uint32_t qg = (uint32_t)g < T.ng ? T.q[g] : T.q[0];
    const uint2 *bq = reinterpret_cast<const uint2 *>(a.queries + (uint64_t)qg * nbp + 8 * t);
    // the epilogue's operands do not depend on the MMAs: their loads go out before the K loop
    int xp[2][2], qp[2];
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int h = 0; h < 2; h++)
            xp[m][h] = (int)__ldg(a.row_pop + T.part_off32 + min(r0 + 16u * m + (uint32_t)g + 8u * h, row_end - 1u));
#pragma unroll
    for (int j2 = 0; j2 < 2; j2++) {
        const uint32_t col = 2u * t + (uint32_t)j2;
        qp[j2] = (int)__ldg(a.qpop + (col < T.ng ? T.q[col] : T.q[0]));
    }
    uint32_t acc[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
    const uint32_t nstep = nbp / 32;
#pragma unroll 4
    for (uint32_t s = 0; s < nstep; s++) {
        const uint32_t off = s * 4;                      // uint2 per 256-bit step: 4
        uint2 va[4];
#pragma unroll
        for (int i = 0; i < 4; i++) va[i] = __ldg(arow[i] + off);
        const uint2 vb = __ldg(bq + off);
        ham_mma(acc[0], va[0], va[1], vb);
        ham_mma(acc[1], va[2], va[3], vb);
    }
    // accumulator x of m-tile m: row 16 m + g + 8 (x >> 1), slot column 2 t + (x & 1)
#pragma unroll
    for (int j2 = 0; j2 < 2; j2++) {
        const uint32_t col = 2u * t + (uint32_t)j2;
        if (col >= T.ng) continue;
        const uint32_t out = T.out[col];
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t r = r0 + 16u * m + (uint32_t)g + 8u * h;
                if (r >= row_end) continue;
                const int d = qp[j2] + xp[m][h] - 2 * (int)acc[m][2 * h + j2];
                if (a.out_u32) reinterpret_cast<uint32_t *>(a.dist_out)[(size_t)out + r] = (uint32_t)d;
                else a.dist_out[(size_t)out + r] = (float)d;
            }
    }
}

// persistent CTAs over the tile queue; the next tile is claimed when a tile starts, so the atomic's round trip runs
// under the tile's work
__global__ void __launch_bounds__(HAM_NT, 2) ivf_ham_scan_kernel(HamScanArgs a)
{
    pdl_entry();
    __shared__ TileDesc s_tile;
    __shared__ uint32_t s_t;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t total = *a.total_tiles;
    if (tid == 0) s_t = atomicAdd(a.tile_counter, 1u);
    __syncthreads();
    for (uint32_t t = s_t; t < total;) {
        if (tid < (int)(sizeof(TileDesc) / 4))
            reinterpret_cast<uint32_t *>(&s_tile)[tid] = __ldg(reinterpret_cast<const uint32_t *>(a.tile_desc + t) + tid);
        __syncthreads();                                   // s_tile written; every thread has read s_t
        uint32_t next = 0;
        if (tid == 0) next = atomicAdd(a.tile_counter, 1u);
        const uint32_t row_end = s_tile.row0 + s_tile.nrows;
        for (uint32_t r0 = s_tile.row0 + 32u * (uint32_t)warp; r0 < row_end; r0 += 32u * (HAM_NT / 32))
            ham_rows(a, s_tile, r0, row_end, lane);
        if (tid == 0) s_t = next;
        __syncthreads();                                   // s_tile is rewritten, s_t is read
        t = s_t;
    }
}

__global__ void ham_all_probes_kernel(uint64_t *__restrict__ probes, uint64_t slots, uint32_t nlist)
{
    pdl_entry();
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < slots) probes[e] = e % nlist;
}

}  // namespace

void launch_ham_all_probes(uint64_t *probes, uint32_t B, uint32_t nlist, cudaStream_t st)
{
    const uint64_t slots = (uint64_t)B * nlist;
    if (slots == 0) return;
    launch_k(ham_all_probes_kernel, dim3((unsigned)((slots + 255) / 256)), dim3(256), 0, st, probes, slots, nlist);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_ivf_ham_scan(const HamScanArgs &a, int grid, cudaStream_t st)
{
    if (!a.tile_desc || a.nbytes_pad % 32) {
        set_error("internal: the binary IVF scan needs tile descriptors and rows padded to a multiple of 32 bytes");
        throw Failure{LGPU_RUNTIME};
    }
    launch_k(ivf_ham_scan_kernel, dim3(grid), dim3(HAM_NT), 0, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
