// pq4_scan.cu -- 4-bit IVF_PQ: packed nibble codes scanned exactly over quantised per-probe tables.
//
// A stored row is m 4-bit codes, two per byte: byte j holds sub-vector 2j's code in bits 0-3 and sub-vector 2j+1's in
// bits 4-7 (lance's packing [lance, recalled]).  Per probe slot (query q, partition p; r = q - c_p for l2 / cosine, q for
// dot) the float table T[i][c] (i < m, c < 16) is the 8-bit path's table on the 16 codewords (subvec_l2 /
// subvec_dot_dist, common.cuh), and lance's quantize_distance_table [lance, recalled] turns it into u8:
//     qmin = min_{i,c} T[i][c]
//     qmax = max_{i < m-1} (max_c T[i][c] + max_c T[i+1][c])            (both folds skip NaN)
//     Q[i][c] = sat_u8(round(((T[i][c] - qmin) * 255) / (qmax - qmin)))  (half away from zero, NaN -> 0)
// A row's distance is then a function of the exact integer S = sum_i Q[i][code_i]:
//     d = ((float) S * (qmax - qmin)) / 255 + qmin * (float) m,  then cosine 0.5 d, dot d - (m - 1)
// every f32 operation rounded on its own, so the result is the CPU oracle's (tests/pq4_oracle.c) bit for bit whatever
// order the sum is formed in.  The three recalled details live in pq4_quant, pq4_tables_kernel's qmax fold and
// pq4_distance, one place each.
//
// pq4_tables_kernel: one warp per probe slot, PQ4_TAB_WARPS slots per CTA.  A lane computes T for one codeword of
// every other sub-space, reading the codebook in the layout [m][dsub][16] the open writes (a half-warp's 16 codewords
// of one element are contiguous); the folds are warp shuffles; the u8 tables go to [slots][m][16] and (qmin, qmax) to
// Pq4Slot.
//
// pq4_scan_kernel is persistent over the regroup's tile queue (group.cu): a tile is <= PQ4_ROWS_TILE rows of one
// partition and the <= 8 probe slots that probe it.  A code byte indexes a pair table PT[j][b] (b < 256) of 8 u16
// lanes, lane s = Q_s[2j][b & 15] + Q_s[2j+1][b >> 4]: per row and code byte one 16-byte shared load and four packed
// u16x2 adds serve all 8 slots.  A lane sum is at most 255 m <= 65280 (m <= LGPU_PQ4_MAX_M), so it never carries into
// its neighbour.  The pair tables are built in chunks of PQ4_CHUNK pairs (4 KB each) into two alternating buffers, one
// barrier per chunk, so every m up to the limit runs in the same kernel.  Codes are stored per partition as
// [m/2][npad] bytes: thread t reads one u32 (4 consecutive rows) per pair and row group, a warp 128 contiguous bytes.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int PQ4_TAB_WARPS = 4;           // tables: probe slots (warps) per CTA
constexpr int PQ4_NT = 256;                // scan threads
constexpr int PQ4_RG = 2;                  // row groups of 4 rows per thread: PQ4_ROWS_TILE = 256 x 2 x 4
constexpr int PQ4_CHUNK = 8;               // pairs per pair-table chunk
static_assert(PQ4_ROWS_TILE == (uint32_t)(PQ4_NT * PQ4_RG * 4), "tile height");

// step 3 of the contract [lance, recalled]: ((t - qmin) * 255) / (qmax - qmin), rounded half away from zero (roundf),
// then Rust's saturating `as u8` (NaN -> 0)
__device__ __forceinline__ uint32_t pq4_quant(float t, float qmin, float qmax)
{
    const float x = __fdiv_rn(__fmul_rn(__fsub_rn(t, qmin), 255.0f), __fsub_rn(qmax, qmin));
    const float r = roundf(x);
    if (!(r > 0.f)) return 0u;                       // negative, zero, NaN
    if (r >= 255.f) return 255u;
    return (uint32_t)r;
}

// step 5 [lance, recalled] and the 8-bit path's finish_pq: the distance of a row whose quantised sum is S
__device__ __forceinline__ float pq4_distance(uint32_t S, float qmin, float qmax, uint32_t m, uint32_t metric)
{
    const float d = __fadd_rn(__fdiv_rn(__fmul_rn((float)S, __fsub_rn(qmax, qmin)), 255.0f), __fmul_rn(qmin, (float)m));
    if (metric == LGPU_COSINE) return __fmul_rn(d, 0.5f);
    if (metric == LGPU_DOT) return __fsub_rn(d, (float)(m - 1));
    return d;
}

// one warp per probe slot e = q * nprobes + j.  Shared memory per warp: T [m][16] f32, then the sub-space maxima [m].
// Slots without a partition are skipped: they get no tiles.
template <int DSUB>
__global__ void __launch_bounds__(32 * PQ4_TAB_WARPS) pq4_tables_kernel(
    const float *__restrict__ Q, const float *__restrict__ centroids, const float *__restrict__ codebook,
    const uint64_t *__restrict__ probes, uint32_t slots, uint32_t nprobes, uint32_t nlist, uint32_t m, uint32_t metric,
    uint8_t *__restrict__ tables, Pq4Slot *__restrict__ slot_out)
{
    pdl_entry();
    extern __shared__ float s_tab[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t e = blockIdx.x * PQ4_TAB_WARPS + w;
    if (e >= slots) return;
    const uint64_t pp = probes[e];
    if (pp >= nlist) return;
    const uint32_t dim = m * DSUB;
    const bool dot = metric == LGPU_DOT;
    const float *qv = Q + (size_t)(e / nprobes) * dim, *c = centroids + (size_t)pp * dim;
    float *T = s_tab + (size_t)w * m * 17, *rmax = T + (size_t)m * 16;
    const uint32_t j = lane & 15;
    float qmin = INFINITY;
    // lanes 0-15: codeword j of the even sub-spaces, lanes 16-31 of the odd ones (m is even: equal trip counts)
    for (uint32_t i = lane >> 4; i < m; i += 2) {
        float r[DSUB];
#pragma unroll
        for (int t = 0; t < DSUB; t++) {
            const uint32_t x = i * DSUB + t;
            r[t] = dot ? qv[x] : __fsub_rn(qv[x], c[x]);
        }
        float cw[DSUB];                              // codeword j: the 16 lanes of a half read 64 contiguous bytes
#pragma unroll
        for (int t = 0; t < DSUB; t++) cw[t] = __ldg(codebook + ((size_t)i * DSUB + t) * 16 + j);
        const float v = dot ? subvec_dot_dist<DSUB>(r, cw) : subvec_l2<DSUB>(r, cw);
        T[i * 16 + j] = v;
        qmin = fminf(qmin, v);                       // fminf / fmaxf return the other operand for NaN (f32::min/max)
        float mx = v;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (j == 0) rmax[i] = fmaxf(-INFINITY, mx);   // an all-NaN sub-space folds to -inf
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) qmin = fminf(qmin, __shfl_xor_sync(0xffffffffu, qmin, o));
    __syncwarp();
    // qmax: adjacent sub-space pairs, overlapping windows [lance, recalled]
    float qmax = -INFINITY;
    for (uint32_t i = lane; i + 1 < m; i += 32) qmax = fmaxf(qmax, __fadd_rn(rmax[i], rmax[i + 1]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, o));
    uint32_t *out = reinterpret_cast<uint32_t *>(tables + (size_t)e * m * 16);
    for (uint32_t x = lane; x < m * 4; x += 32) {
        const float *t4 = T + 4 * x;
        out[x] = pq4_quant(t4[0], qmin, qmax) | pq4_quant(t4[1], qmin, qmax) << 8 | pq4_quant(t4[2], qmin, qmax) << 16 |
                 pq4_quant(t4[3], qmin, qmax) << 24;
    }
    if (lane == 0) slot_out[e] = Pq4Slot{qmin, qmax};
}

// the 8 slot bytes of a staged table entry as u16 lanes: {s0 s1, s2 s3, s4 s5, s6 s7}
__device__ __forceinline__ uint4 pq4_widen(uint2 v)
{
    return make_uint4(__byte_perm(v.x, 0u, 0x7170u), __byte_perm(v.x, 0u, 0x7372u), __byte_perm(v.y, 0u, 0x7170u),
                      __byte_perm(v.y, 0u, 0x7372u));
}

// one tile: stage the slots' u8 tables, then per chunk of pairs build the pair tables and accumulate every row's 8 sums
__device__ __forceinline__ void pq4_tile(const Pq4ScanArgs &a, const TileDesc &T, uint4 *s_pt, uint2 *s_q, int tid)
{
    const uint32_t m = a.m, mh = m >> 1, ng = T.ng;
    // s_q[i * 16 + c] = byte s: Q_s[i][c] of the tile's slot s (0 for s >= ng)
    for (uint32_t x = (uint32_t)tid; x < m * 16; x += PQ4_NT) {
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int s = 0; s < SCAN_G; s++) {
            const uint32_t b = (uint32_t)s < ng ? (uint32_t)__ldg(a.tables + (size_t)T.slot[s] * m * 16 + x) : 0u;
            if (s < 4) lo |= b << (8 * s); else hi |= b << (8 * (s - 4));
        }
        s_q[x] = make_uint2(lo, hi);
    }
    __syncthreads();
    const uint32_t *words = a.codes + (size_t)T.code_base8 * 2 + T.row0 / 4;     // pair 0, the tile's first row group
    const uint32_t wstride = T.npad / 4;
    bool valid[PQ4_RG];
#pragma unroll
    for (int r = 0; r < PQ4_RG; r++) valid[r] = 4u * (uint32_t)(tid + PQ4_NT * r) < T.nrows;
    uint32_t acc[PQ4_RG][4][4];
#pragma unroll
    for (int r = 0; r < PQ4_RG; r++)
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int x = 0; x < 4; x++) acc[r][k][x] = 0u;
    for (uint32_t c0 = 0, bi = 0; c0 < mh; c0 += PQ4_CHUNK, bi ^= 1u) {
        const uint32_t nc = min((uint32_t)PQ4_CHUNK, mh - c0);
        uint32_t wv[PQ4_RG][PQ4_CHUNK];              // the chunk's code words, in flight during the build
#pragma unroll
        for (int jj = 0; jj < PQ4_CHUNK; jj++)
#pragma unroll
            for (int r = 0; r < PQ4_RG; r++)
                wv[r][jj] = valid[r] && (uint32_t)jj < nc
                                ? __ldg(words + (size_t)(c0 + jj) * wstride + tid + PQ4_NT * r) : 0u;
        uint4 *pt = s_pt + (size_t)bi * PQ4_CHUNK * 256;
        for (uint32_t jj = 0; jj < nc; jj++) {       // entry b = tid of every pair of the chunk
            const uint32_t i0 = 2 * (c0 + jj);
            const uint4 lo = pq4_widen(s_q[i0 * 16 + (tid & 15)]), hi = pq4_widen(s_q[(i0 + 1) * 16 + (tid >> 4)]);
            pt[jj * 256 + tid] = make_uint4(lo.x + hi.x, lo.y + hi.y, lo.z + hi.z, lo.w + hi.w);
        }
        __syncthreads();                             // the other buffer is rebuilt only after the next barrier
#pragma unroll
        for (int jj = 0; jj < PQ4_CHUNK; jj++) {
            if ((uint32_t)jj >= nc) break;
#pragma unroll
            for (int r = 0; r < PQ4_RG; r++) {
                if (!valid[r]) continue;
                const uint32_t wd = wv[r][jj];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint4 v = pt[jj * 256 + __byte_perm(wd, 0u, 0x4440u + k)];
                    acc[r][k][0] += v.x; acc[r][k][1] += v.y; acc[r][k][2] += v.z; acc[r][k][3] += v.w;
                }
            }
        }
    }
    // epilogue: rows 4 g .. 4 g + 3 of each valid group, one float4 per slot (segments are padded to 4 floats and
    // row0 is a multiple of 32, so the store is aligned and stays inside the slot's segment)
#pragma unroll
    for (int r = 0; r < PQ4_RG; r++) {
        if (!valid[r]) continue;
        const uint32_t row = T.row0 + 4u * (uint32_t)(tid + PQ4_NT * r);
#pragma unroll
        for (int s = 0; s < SCAN_G; s++) {
            if ((uint32_t)s >= ng) break;
            uint32_t S[4];
#pragma unroll
            for (int k = 0; k < 4; k++) S[k] = (acc[r][k][s >> 1] >> (16 * (s & 1))) & 0xffffu;
            float4 *dst = reinterpret_cast<float4 *>(a.dist_out + (size_t)T.out[s] + row);
            if (a.out_u32) {
                *dst = make_float4(__uint_as_float(S[0]), __uint_as_float(S[1]), __uint_as_float(S[2]),
                                   __uint_as_float(S[3]));
            } else {
                const Pq4Slot sl = a.slots[T.slot[s]];
                *dst = make_float4(pq4_distance(S[0], sl.qmin, sl.qmax, m, a.metric),
                                   pq4_distance(S[1], sl.qmin, sl.qmax, m, a.metric),
                                   pq4_distance(S[2], sl.qmin, sl.qmax, m, a.metric),
                                   pq4_distance(S[3], sl.qmin, sl.qmax, m, a.metric));
            }
        }
    }
}

// persistent CTAs over the tile queue; the next tile is claimed when a tile starts
__global__ void __launch_bounds__(PQ4_NT, 2) pq4_scan_kernel(Pq4ScanArgs a)
{
    pdl_entry();
    extern __shared__ uint4 s_dyn[];
    uint4 *s_pt = s_dyn;                                                   // [2][PQ4_CHUNK][256] pair tables
    uint2 *s_q = reinterpret_cast<uint2 *>(s_dyn + 2 * PQ4_CHUNK * 256);  // [m][16] x 8 slot bytes
    __shared__ TileDesc s_tile;
    __shared__ uint32_t s_t;
    const int tid = threadIdx.x;
    const uint32_t total = *a.total_tiles;
    if (tid == 0) s_t = atomicAdd(a.tile_counter, 1u);
    __syncthreads();
    for (uint32_t t = s_t; t < total;) {
        if (tid < (int)(sizeof(TileDesc) / 4))
            reinterpret_cast<uint32_t *>(&s_tile)[tid] = __ldg(reinterpret_cast<const uint32_t *>(a.tile_desc + t) + tid);
        __syncthreads();                                   // s_tile written; every thread has read s_t
        uint32_t next = 0;
        if (tid == 0) next = atomicAdd(a.tile_counter, 1u);
        pq4_tile(a, s_tile, s_pt, s_q, tid);
        if (tid == 0) s_t = next;
        __syncthreads();                                   // s_tile, s_q and the pair tables are rewritten, s_t is read
        t = s_t;
    }
}

// open: codes (row-major [n][m/2] or per partition [m/2][n_p]) -> per partition [m/2][npad] at code_base[p]
__global__ void pq4_relayout_kernel(const uint8_t *__restrict__ codes, int layout, const uint64_t *__restrict__ part_off,
                                    uint32_t nlist, uint64_t nrows, uint32_t mh, const uint64_t *__restrict__ code_base,
                                    const uint32_t *__restrict__ part_npad, uint8_t *__restrict__ out)
{
    const uint64_t grow = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (grow >= nrows) return;
    uint32_t lo = 0, hi = nlist - 1;                   // partition of grow: part_off[p] <= grow < part_off[p+1]
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (part_off[mid + 1] > grow) hi = mid; else lo = mid + 1;
    }
    const uint64_t pbase = part_off[lo];
    const uint32_t row = (uint32_t)(grow - pbase), n_p = (uint32_t)(part_off[lo + 1] - pbase), npad = part_npad[lo];
    uint8_t *dst = out + code_base[lo] + row;
    for (uint32_t j = 0; j < mh; j++)
        dst[(size_t)j * npad] = layout == LGPU_CODES_ROW_MAJOR ? codes[grow * mh + j]
                                                               : codes[pbase * mh + (uint64_t)j * n_p + row];
}

}  // namespace

size_t pq4_scan_smem(uint32_t m) { return (size_t)2 * PQ4_CHUNK * 256 * 16 + (size_t)m * 16 * 8; }

void launch_pq4_tables(const float *Q, const float *centroids, const float *codebook, const uint64_t *probes,
                       uint32_t slots, uint32_t nprobes, uint32_t nlist, uint32_t m, uint32_t dsub, int metric,
                       uint8_t *tables, Pq4Slot *slot_out, cudaStream_t st)
{
    if (slots == 0) return;
    const size_t smem = (size_t)PQ4_TAB_WARPS * m * 17 * 4;
    const dim3 grid(ceil_div(slots, PQ4_TAB_WARPS)), block(32 * PQ4_TAB_WARPS);
#define LGPU_PQ4_TAB(D)                                                                                                \
    case D: {                                                                                                          \
        auto kern = pq4_tables_kernel<D>;                                                                              \
        LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                 \
        launch_k(kern, grid, block, smem, st, Q, centroids, codebook, probes, slots, nprobes, nlist, m, (uint32_t)metric, \
                 tables, slot_out); LGPU_COUNT_LAUNCH();                                                               \
        break;                                                                                                         \
    }
    switch (dsub) {
        LGPU_PQ4_TAB(1) LGPU_PQ4_TAB(2) LGPU_PQ4_TAB(4) LGPU_PQ4_TAB(8) LGPU_PQ4_TAB(16) LGPU_PQ4_TAB(32)
    default:
        set_error("internal: unsupported 4-bit PQ sub-vector length");
        throw Failure{LGPU_RUNTIME};
    }
#undef LGPU_PQ4_TAB
    LGPU_CUDA(cudaGetLastError());
}

void launch_pq4_scan(const Pq4ScanArgs &a, int grid, cudaStream_t st)
{
    if (!a.tile_desc || a.m < 2 || a.m % 2 || a.m > LGPU_PQ4_MAX_M) {
        set_error("internal: the 4-bit PQ scan needs tile descriptors and an even m <= LGPU_PQ4_MAX_M");
        throw Failure{LGPU_RUNTIME};
    }
    const size_t smem = pq4_scan_smem(a.m);
    LGPU_CUDA(cudaFuncSetAttribute(pq4_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    launch_k(pq4_scan_kernel, dim3(grid), dim3(PQ4_NT), smem, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_pq4_relayout(const uint8_t *codes, int layout, const uint64_t *part_off, uint32_t nlist, uint64_t nrows,
                         uint32_t m, const uint64_t *code_base, const uint32_t *part_npad, uint8_t *out, cudaStream_t st)
{
    if (nrows == 0) return;
    pq4_relayout_kernel<<<(unsigned)((nrows + 255) / 256), 256, 0, st>>>(codes, layout, part_off, nlist, nrows, m / 2,
                                                                       code_base, part_npad, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
