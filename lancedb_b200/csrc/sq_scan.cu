// sq_scan.cu -- IVF_SQ: 8-bit scalar-quantised partitions scanned exactly on the integer tensor cores.
//
// A stored row is dim codes k_i = sat_u8(((double)x_i - lo) * 255 / (hi - lo)) (lance's scale_to_u8 [lance, recalled]),
// laid out row-major with dim zero-padded to dim_pad (a multiple of SQ_K_CHUNK).  A query is encoded the same way on the
// device (sq_encode_kernel), and
//     _distance = (float) sum_i (k_i - q_i)^2 = (float) (|k|^2 + |q|^2 - 2 k.q)
// is computed in u32: the true sum is below 2^32 for dim <= 65536, so the arithmetic modulo 2^32 is exact even where the
// s32 accumulator of the MMA wraps (the MMA is issued without .satfinite, so it wraps instead of clamping).  The one
// rounding is the final u32 -> f32 (round to nearest), so the result is the CPU oracle's bit for bit.
//
// The scan reads the same tile queue as the PQ kernels (group.cu): a tile is <= SQ_ROWS_TILE rows of one partition and
// the <= 8 queries that probe it.  Each warp owns 32 rows of the tile and runs two m16n8k32 u8 MMAs (rows = M, the
// tile's queries = N = 8) per 32 bytes of K.  Each lane loads 16 contiguous code bytes of 4 rows and of its query per
// 64-byte K chunk; because a dot product does not depend on the order of its terms, those bytes are handed to the MMA
// under a permutation of K that is the same for both operands (see sq_tile).  The loads are straight from global
// memory: with 8 queries per tile the scan does 16 integer ops per code byte, far below what the tensor cores sustain,
// so HBM bandwidth bounds it and no shared-memory staging is needed.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int SQ_NT = 256;                 // 8 warps x 32 rows = SQ_ROWS_TILE

// sat_u8(((double)v - lo) * 255 / (hi - lo)): left to right in f64, truncated toward zero, NaN -> 0, lo == hi -> 0
__device__ __forceinline__ uint32_t sq_code(float v, double lo, double hi)
{
    if (!(hi != lo)) return 0u;
    const double t = __ddiv_rn(__dmul_rn(__dsub_rn((double)v, lo), 255.0), __dsub_rn(hi, lo));
    if (!(t > 0.0)) return 0u;                         // negative, -0, NaN
    if (t >= 255.0) return 255u;
    return (uint32_t)t;                                // truncation toward zero
}

// one block per query: codes [dim_pad] (zero padding) and |q|^2 of the codes
__global__ void sq_encode_kernel(const float *__restrict__ Q, uint32_t dim, uint32_t dim_pad, double lo, double hi,
                                 uint8_t *__restrict__ qc, uint32_t *__restrict__ qq)
{
    pdl_entry();
    __shared__ uint32_t s_sum[32];
    const uint32_t b = blockIdx.x;
    const float *q = Q + (size_t)b * dim;
    uint8_t *out = qc + (size_t)b * dim_pad;
    uint32_t s = 0;
    for (uint32_t i = threadIdx.x; i < dim_pad; i += blockDim.x) {
        const uint32_t c = i < dim ? sq_code(q[i], lo, hi) : 0u;
        out[i] = (uint8_t)c;
        s += c * c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (uint32_t w = 0; w < blockDim.x / 32; w++) t += s_sum[w];
        qq[b] = t;
    }
}

// a warp per row: xx[r] = sum of the squared codes of row r ([n][dim_pad], zero padding)
__global__ void sq_row_norms_kernel(const uint8_t *__restrict__ codes, uint64_t n, uint32_t dim_pad,
                                    uint32_t *__restrict__ xx)
{
    const uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    const uint32_t *row = reinterpret_cast<const uint32_t *>(codes + r * dim_pad);
    uint32_t s = 0;
    for (uint32_t w = lane; w < dim_pad / 4; w += 32) {
        const uint32_t v = __ldg(row + w);
#pragma unroll
        for (int j = 0; j < 4; j++) { const uint32_t c = (v >> (8 * j)) & 0xffu; s += c * c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) xx[r] = s;
}

__device__ __forceinline__ void mma_u8(uint32_t (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                       uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// One warp's 32 rows of a tile against the tile's <= 8 queries.  Lane (g = lane / 4, t = lane % 4) loads, per 64-byte K
// chunk, the 16 bytes at offset 16 t of rows g, g + 8, g + 16, g + 24 and of query g.  In MMA step s of the chunk, the
// fragment slot (t, half h) -- logical K 16 h + 4 t .. + 3 for both the A rows and the B column -- gets word 2 s + h of
// those 16 bytes, i.e. physical K 16 t + 8 s + 4 h .. + 3: the same bijection of the chunk's 64 bytes for A and B.
__device__ __forceinline__ void sq_tile(const SqScanArgs &a, const TileDesc &T, int warp, int lane)
{
    const uint32_t row_end = T.row0 + T.nrows;                 // rows of the partition this tile covers
    const uint32_t r0 = T.row0 + 32u * (uint32_t)warp;
    if (r0 >= row_end) return;
    const int g = lane >> 2, t = lane & 3;
    const uint8_t *arow[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t r = min(r0 + (uint32_t)(g + 8 * i), row_end - 1u);      // rows past the tile: re-read, not written
        arow[i] = a.codes + ((uint64_t)(T.part_off32 - a.range.row_shift) + r) * a.dim_pad + 16 * t;
    }
    const uint32_t qg = (uint32_t)g < T.ng ? T.q[g] : T.q[0];
    const uint8_t *brow = a.qcodes + (uint64_t)qg * a.dim_pad + 16 * t;
    uint32_t acc[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
    const uint32_t nchunk = a.dim_pad / SQ_K_CHUNK;
#pragma unroll 2
    for (uint32_t c = 0; c < nchunk; c++) {
        const size_t off = (size_t)c * SQ_K_CHUNK;
        uint4 va[4];
#pragma unroll
        for (int i = 0; i < 4; i++) va[i] = __ldg(reinterpret_cast<const uint4 *>(arow[i] + off));
        const uint4 vb = __ldg(reinterpret_cast<const uint4 *>(brow + off));
        // step 0: words x, y; step 1: words z, w
        mma_u8(acc[0], va[0].x, va[1].x, va[0].y, va[1].y, vb.x, vb.y);
        mma_u8(acc[1], va[2].x, va[3].x, va[2].y, va[3].y, vb.x, vb.y);
        mma_u8(acc[0], va[0].z, va[1].z, va[0].w, va[1].w, vb.z, vb.w);
        mma_u8(acc[1], va[2].z, va[3].z, va[2].w, va[3].w, vb.z, vb.w);
    }
    // accumulator j of m-tile m: row 16 m + g + 8 (j >> 1), query column 2 t + (j & 1)
#pragma unroll
    for (int j2 = 0; j2 < 2; j2++) {
        const uint32_t col = 2u * t + (uint32_t)j2;
        if (col >= T.ng) continue;
        const uint32_t qi = T.q[col], qn = __ldg(a.qq + qi), out = T.out[col];
#pragma unroll
        for (int m = 0; m < 2; m++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t r = r0 + 16u * m + (uint32_t)g + 8u * h;
                if (r >= row_end) continue;
                const uint32_t d = __ldg(a.xx + T.part_off32 + r) + qn - 2u * acc[m][2 * h + j2];   // exact mod 2^32
                if (a.out_u32) reinterpret_cast<uint32_t *>(a.dist_out)[(size_t)out + r] = d;
                else a.dist_out[(size_t)out + r] = __uint2float_rn(d);
            }
        }
    }
}

// persistent CTAs over the tile queue
__global__ void __launch_bounds__(SQ_NT, 2) sq_scan_kernel(SqScanArgs a)
{
    pdl_entry();
    __shared__ TileDesc s_tile;
    __shared__ uint32_t s_t;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t total = tile_range_total(a.range, a.total_tiles);
    for (;;) {
        if (tid == 0) s_t = atomicAdd(a.tile_counter, 1u);
        __syncthreads();
        const uint32_t t = s_t;
        if (t >= total) break;
        const TileDesc *d = a.tile_desc + tile_range_at(a.range, t);
        if (tid < (int)(sizeof(TileDesc) / 4))
            reinterpret_cast<uint32_t *>(&s_tile)[tid] = __ldg(reinterpret_cast<const uint32_t *>(d) + tid);
        __syncthreads();
        sq_tile(a, s_tile, warp, lane);
        __syncthreads();                                   // s_t and s_tile are rewritten by the next claim
    }
}

}  // namespace

void launch_sq_encode(const float *Q, uint32_t B, uint32_t dim, uint32_t dim_pad, double lo, double hi, uint8_t *qc,
                      uint32_t *qq, cudaStream_t st)
{
    if (B == 0) return;
    launch_k(sq_encode_kernel, dim3(B), dim3(256), 0, st, Q, dim, dim_pad, lo, hi, qc, qq); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_sq_row_norms(const uint8_t *codes, uint64_t n, uint32_t dim_pad, uint32_t *xx, cudaStream_t st)
{
    if (n == 0) return;
    const uint64_t blocks = (n * 32 + 255) / 256;
    sq_row_norms_kernel<<<(unsigned)blocks, 256, 0, st>>>(codes, n, dim_pad, xx); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_sq_scan(const SqScanArgs &a, int grid, cudaStream_t st)
{
    if (!a.tile_desc || a.dim_pad % SQ_K_CHUNK) {
        set_error("internal: the SQ scan needs tile descriptors and rows padded to a multiple of 64 bytes");
        throw Failure{LGPU_RUNTIME};
    }
    launch_k(sq_scan_kernel, dim3(grid), dim3(SQ_NT), 0, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
