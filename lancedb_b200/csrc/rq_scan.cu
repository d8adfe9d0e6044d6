// rq_scan.cu -- IVF_RQ: 1-bit RaBitQ partitions scanned exactly on the binary tensor cores.
//
// A stored row x of partition p is o = P (x - c_p) (P an orthogonal rotation, f64 at build time), kept as one sign bit
// per dimension b_i = [o_i > 0] (LSB first, rows zero-padded to dim_pad = a multiple of 256 bits) and two f32 factors
// add = |o|^2 and scale = -2 |o|^2 / sum |o_i|.  A query probe slot (query q, partition p) is the rotated residual
// q'_i = fl(rq_i - rc_{p,i}) (rq = P q, rc_p = P c_p, both in lance's lane order), quantised to 4 bits on its own grid
//     lo = min q', delta = fl(fl(max q' - lo) / 15), u_i = min(15, trunc(fl(fl(fl(q'_i - lo) / delta) + 0.5)))
// and kept as four bit-planes.  The RaBitQ estimate of |x - q|^2 is then, with ip = sum_i b_i u_i exact in integers,
//     y   = fl(fl(delta * (float)(2 ip - S)) + fl(lo * (float)(2 popc(b) - dim)))          S = sum_i u_i
//     est = fl(fl(add + qq) + fl(scale * y))                                               qq = lance_l2(rq, rc_p)
// (cosine: fl(0.5 est)), every operation rounded on its own so the result is the CPU oracle's (tests/rq_oracle.c) bit
// for bit.  A slot whose delta is not finite contributes NaN rows, which the select drops.
//
// ip is integer work for the b1 MMA: ip = sum_j 2^j popc(b AND plane_j).  The scan reads the same tile queue as the
// IVF_SQ scan (group.cu): a tile is <= RQ_ROWS_TILE rows of one partition and the <= 8 probe slots that probe it.  Each
// warp owns 32 rows (two m16 tiles); per 256-bit K step it issues 2 x 4 mma.m16n8k256 b1 AND.POPC (one per m-tile and
// plane; rows = M, the tile's slots = N = 8).  Lane (g, t) loads 8 bytes at offset 8 t of the step's 32 bytes of rows
// g, g + 8, g + 16, g + 24 and of each plane of slot g: fragment half h gets word 2 t + h, the same bijection of K for
// A and B, so the popcounts are those of the true bit order.  A row is 96 code bytes at dim 768 and the MMAs do 32
// integer ops per byte, far below the tensor cores' rate, so operands come straight from global memory with no
// shared-memory staging; what bounds the kernel is the latency of each small tile (DESIGN.md section 6).
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr int RQ_NT = 256;                 // 8 warps x 32 rows = RQ_ROWS_TILE
constexpr int RQ_ROT_T = 16;               // rotation: 16 x 16 threads, 32 vectors x 32 dimensions per CTA
constexpr int RQ_PLANES_NT = 128;          // planes: threads per probe slot (short CTAs, many resident per SM)

// out[v][i] = lance_dot(P row i, x[v]) for v < n, i < dim.  A CTA covers 32 dimensions x 32 vectors and stages
// 16-column chunks of both in shared memory; a thread owns 2 x 2 outputs (i, i + 16) x (v, v + 16), so each staged
// value it reads serves two products.  Every output keeps lance's 16 lane sums, so the order of the additions is
// lance_dot's (remainder first, then the lanes in order)
__global__ void __launch_bounds__(256) rq_rotate_kernel(const float *__restrict__ P, const float *__restrict__ x,
                                                        uint32_t n, uint32_t dim, float *__restrict__ out)
{
    pdl_entry();
    constexpr int T = 2 * RQ_ROT_T;
    __shared__ float sP[T][RQ_ROT_T + 1], sX[T][RQ_ROT_T + 1];
    const int tx = threadIdx.x % RQ_ROT_T, ty = threadIdx.x / RQ_ROT_T;
    const uint32_t i0 = blockIdx.x * T, v0 = blockIdx.y * T;
    const uint32_t nch = dim >> 4, rem0 = nch << 4;
    float s[2][2], sums[2][2][16];
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
        for (int b = 0; b < 2; b++) {
            const float *prow = P + (size_t)min(i0 + tx + 16 * a, dim - 1) * dim;
            const float *xrow = x + (size_t)min(v0 + ty + 16 * b, n - 1) * dim;
            float t = 0.f;
            for (uint32_t j = rem0; j < dim; j++) t = __fadd_rn(t, __fmul_rn(prow[j], xrow[j]));
            s[a][b] = t;
#pragma unroll
            for (int l = 0; l < 16; l++) sums[a][b][l] = 0.f;
        }
    // staging: thread (ty, tx) loads element tx of the chunk of rows ty and ty + 16 of the tile (P rows, x rows)
    for (uint32_t c = 0; c < nch; c++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            sP[ty + 16 * h][tx] = P[(size_t)min(i0 + ty + 16 * h, dim - 1) * dim + c * 16 + tx];
            sX[ty + 16 * h][tx] = x[(size_t)min(v0 + ty + 16 * h, n - 1) * dim + c * 16 + tx];
        }
        __syncthreads();
#pragma unroll
        for (int l = 0; l < 16; l++) {
            const float p0 = sP[tx][l], p1 = sP[tx + 16][l], x0 = sX[ty][l], x1 = sX[ty + 16][l];
            sums[0][0][l] = __fadd_rn(sums[0][0][l], __fmul_rn(p0, x0));
            sums[0][1][l] = __fadd_rn(sums[0][1][l], __fmul_rn(p0, x1));
            sums[1][0][l] = __fadd_rn(sums[1][0][l], __fmul_rn(p1, x0));
            sums[1][1][l] = __fadd_rn(sums[1][1][l], __fmul_rn(p1, x1));
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
        for (int b = 0; b < 2; b++) {
            const uint32_t i = i0 + tx + 16 * a, v = v0 + ty + 16 * b;
            float t = 0.f;
#pragma unroll
            for (int l = 0; l < 16; l++) t = __fadd_rn(t, sums[a][b][l]);
            if (i < dim && v < n) out[(size_t)v * dim + i] = __fadd_rn(s[a][b], t);
        }
}

// min / max that skip NaN (tracked on its own) and order -0 below +0, so the extremes do not depend on the reduction order
__device__ __forceinline__ float rq_min(float a, float b) { return (b < a || (b == a && signbit(b))) ? b : a; }
__device__ __forceinline__ float rq_max(float a, float b) { return (b > a || (b == a && !signbit(b))) ? b : a; }

// one CTA per probe slot e = q * nprobes + j: q' = fl(rq[q] - rc[p]) in shared memory, lo / hi, delta, the 4-bit
// codes u as four bit-planes [4][wpr] (zero past dim), S = sum u, qq = lance_l2(rq[q], rc[p]).  Unused slots (no
// partition) are skipped: they get no tiles.
__global__ void __launch_bounds__(RQ_PLANES_NT) rq_planes_kernel(const float *__restrict__ rq, const float *__restrict__ rc,
                                                        const uint64_t *__restrict__ probes, uint32_t nprobes,
                                                        uint32_t nlist, uint32_t dim, uint32_t wpr,
                                                        uint32_t *__restrict__ planes, RqSlot *__restrict__ slots)
{
    pdl_entry();
    extern __shared__ float s_q[];                       // [dim]
    __shared__ float s_lo[8], s_hi[8], s_l2[16];
    __shared__ uint32_t s_nan[8], s_sum[8];
    const uint32_t e = blockIdx.x, q = e / nprobes;
    const uint64_t pp = probes[e];
    if (pp >= nlist) return;
    const float *a = rq + (size_t)q * dim, *c = rc + (size_t)pp * dim;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    float lo = INFINITY, hi = -INFINITY;
    uint32_t nan = 0;
    for (uint32_t i = tid; i < dim; i += blockDim.x) {
        const float d = __fsub_rn(a[i], c[i]);
        s_q[i] = d;
        nan |= d != d;
        lo = rq_min(lo, d); hi = rq_max(hi, d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = rq_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = rq_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        nan |= __shfl_xor_sync(0xffffffffu, nan, o);
    }
    if (lane == 0) { s_lo[w] = lo; s_hi[w] = hi; s_nan[w] = nan; }
    __syncthreads();
    lo = s_lo[0]; hi = s_hi[0]; nan = s_nan[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); k++) { lo = rq_min(lo, s_lo[k]); hi = rq_max(hi, s_hi[k]); nan |= s_nan[k]; }
    if (nan) lo = hi = __int_as_float(0x7fc00000);       // a NaN component: no finite grid, the slot has no rows
    const float delta = __fdiv_rn(__fsub_rn(hi, lo), 15.0f);
    const bool grid = delta > 0.f && isfinite(delta);    // otherwise every u is 0 (and a non-finite slot has no rows)
    // planes: a warp per 32-dimension word, a lane per dimension; bit k of a plane word is lane k's ballot
    uint32_t S = 0;
    uint32_t *pl = planes + (size_t)e * 4 * wpr;
    for (uint32_t wd = w; wd < wpr; wd += blockDim.x >> 5) {
        const uint32_t i = wd * 32 + lane;
        uint32_t u = 0;
        if (grid && i < dim) {
            const float f = __fadd_rn(__fdiv_rn(__fsub_rn(s_q[i], lo), delta), 0.5f);
            u = min(15u, (uint32_t)f);
        }
        S += u;
        const uint32_t p0 = __ballot_sync(0xffffffffu, u & 1u), p1 = __ballot_sync(0xffffffffu, u & 2u);
        const uint32_t p2 = __ballot_sync(0xffffffffu, u & 4u), p3 = __ballot_sync(0xffffffffu, u & 8u);
        if (lane < 4) pl[lane * wpr + wd] = lane == 0 ? p0 : (lane == 1 ? p1 : (lane == 2 ? p2 : p3));
    }
    // qq = lance_l2(rq, rc) = lance's lane sums of fl(q'_i)^2: lane l of 16 threads, then the remainder and the lanes
    // in lance's order by thread 0
    if (tid < 16) {
        float acc = 0.f;
#pragma unroll 8
        for (uint32_t ch = 0; ch < (dim >> 4); ch++) { const float d = s_q[ch * 16 + tid]; acc = __fadd_rn(acc, __fmul_rn(d, d)); }
        s_l2[tid] = acc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
    if (lane == 0) s_sum[w] = S;
    __syncthreads();
    if (tid == 0) {
        float s = 0.f;
        for (uint32_t i = (dim >> 4) << 4; i < dim; i++) s = __fadd_rn(s, __fmul_rn(s_q[i], s_q[i]));
        float t = 0.f;
        for (int l = 0; l < 16; l++) t = __fadd_rn(t, s_l2[l]);
        uint32_t tot = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); k++) tot += s_sum[k];
        RqSlot r;
        r.lo = lo; r.delta = delta; r.S = tot; r.qq = __fadd_rn(s, t);
        slots[e] = r;
    }
}

// per row: clear the code bits past dim (the contract says they are 0; a stray bit would change ip and popc) and
// count the set bits; a warp per row
__global__ void rq_row_prep_kernel(uint32_t *__restrict__ codes, uint64_t n, uint32_t dim, uint32_t wpr,
                                   uint32_t *__restrict__ popc)
{
    const uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    uint32_t *row = codes + r * wpr;
    uint32_t s = 0;
    for (uint32_t w = lane; w < wpr; w += 32) {
        uint32_t v = row[w];
        const uint32_t b0 = w * 32;
        const uint32_t keep = b0 >= dim ? 0u : (dim - b0 >= 32 ? 0xffffffffu : (1u << (dim - b0)) - 1u);
        if ((v & keep) != v) { v &= keep; row[w] = v; }
        s += __popc(v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) popc[r] = s;
}

__device__ __forceinline__ void mma_b1(uint32_t (&d)[4], uint2 a_lo, uint2 a_hi, uint2 b)
{
    asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a_lo.x), "r"(a_hi.x), "r"(a_lo.y), "r"(a_hi.y), "r"(b.x), "r"(b.y));
}

// One warp's 32 rows of a tile against the tile's <= 8 probe slots.  a_lo = row 16 m + g, a_hi = row 16 m + g + 8:
// fragment registers a0 / a1 are (row g / g + 8, K half 0), a2 / a3 (row g / g + 8, K half 1), b0 / b1 (K half 0 / 1).
__device__ __forceinline__ void rq_tile(const RqScanArgs &a, const TileDesc &T, int warp, int lane)
{
    const uint32_t row_end = T.row0 + T.nrows;
    const uint32_t r0 = T.row0 + 32u * (uint32_t)warp;
    if (r0 >= row_end) return;
    const int g = lane >> 2, t = lane & 3;
    const uint32_t wpr = a.wpr;
    const uint2 *arow[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t r = min(r0 + (uint32_t)(g + 8 * i), row_end - 1u);      // rows past the tile: re-read, not written
        arow[i] = reinterpret_cast<const uint2 *>(a.codes + ((uint64_t)T.part_off32 + r) * wpr + 2 * t);
    }
    const uint32_t eg = (uint32_t)g < T.ng ? T.slot[g] : T.slot[0];
    const uint2 *bp = reinterpret_cast<const uint2 *>(a.planes + (uint64_t)eg * 4 * wpr + 2 * t);
    const uint32_t pstride = wpr / 2;                    // uint2 per plane
    // the epilogue's operands do not depend on the MMAs: their loads go out before the K loop
    float f_add[2][2], f_scale[2][2];
    int f_pc[2][2];
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t row = T.part_off32 + min(r0 + 16u * m + (uint32_t)g + 8u * h, row_end - 1u);
            f_add[m][h] = __ldg(a.add + row); f_scale[m][h] = __ldg(a.scale + row); f_pc[m][h] = (int)__ldg(a.popc + row);
        }
    RqSlot sl[2];
#pragma unroll
    for (int j2 = 0; j2 < 2; j2++) {
        const uint32_t col = 2u * t + (uint32_t)j2;
        sl[j2] = a.slots[col < T.ng ? T.slot[col] : T.slot[0]];
    }
    uint32_t acc[2][4][4];
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int x = 0; x < 4; x++) acc[m][j][x] = 0u;
    const uint32_t nstep = wpr / 8;
#pragma unroll 3
    for (uint32_t s = 0; s < nstep; s++) {
        const uint32_t off = s * 4;                      // uint2 per 256-bit step: 4
        uint2 va[4], vb[4];
#pragma unroll
        for (int i = 0; i < 4; i++) va[i] = __ldg(arow[i] + off);
#pragma unroll
        for (int j = 0; j < 4; j++) vb[j] = __ldg(bp + j * pstride + off);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            mma_b1(acc[0][j], va[0], va[1], vb[j]);
            mma_b1(acc[1][j], va[2], va[3], vb[j]);
        }
    }
    // accumulator x of m-tile m: row 16 m + g + 8 (x >> 1), slot column 2 t + (x & 1)
#pragma unroll
    for (int j2 = 0; j2 < 2; j2++) {
        const uint32_t col = 2u * t + (uint32_t)j2;
        if (col >= T.ng) continue;
        const uint32_t out = T.out[col];
        const bool ok = isfinite(sl[j2].delta);
#pragma unroll
        for (int m = 0; m < 2; m++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t r = r0 + 16u * m + (uint32_t)g + 8u * h;
                if (r >= row_end) continue;
                const int x = 2 * h + j2;
                const uint32_t ip = acc[m][0][x] + 2u * acc[m][1][x] + 4u * acc[m][2][x] + 8u * acc[m][3][x];
                if (a.out_ip) { reinterpret_cast<uint32_t *>(a.dist_out)[(size_t)out + r] = ip; continue; }
                const float y = __fadd_rn(__fmul_rn(sl[j2].delta, (float)(2 * (int)ip - (int)sl[j2].S)),
                                          __fmul_rn(sl[j2].lo, (float)(2 * f_pc[m][h] - (int)a.dim)));
                float est = __fadd_rn(__fadd_rn(f_add[m][h], sl[j2].qq), __fmul_rn(f_scale[m][h], y));
                if (a.cosine) est = __fmul_rn(0.5f, est);
                a.dist_out[(size_t)out + r] = ok ? est : __int_as_float(0x7fc00000);
            }
        }
    }
}

// persistent CTAs over the tile queue; the next tile is claimed when a tile starts, so the atomic's round trip runs
// under the tile's work
__global__ void __launch_bounds__(RQ_NT, 2) rq_scan_kernel(RqScanArgs a)
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
        rq_tile(a, s_tile, warp, lane);
        if (tid == 0) s_t = next;
        __syncthreads();                                   // s_tile is rewritten, s_t is read
        t = s_t;
    }
}

}  // namespace

void launch_rq_rotate(const float *P, const float *x, uint32_t n, uint32_t dim, float *out, cudaStream_t st)
{
    if (n == 0) return;
    const dim3 grid(ceil_div(dim, 2 * RQ_ROT_T), ceil_div(n, 2 * RQ_ROT_T));
    launch_k(rq_rotate_kernel, grid, dim3(RQ_ROT_T * RQ_ROT_T), 0, st, P, x, n, dim, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rq_planes(const float *rq, const float *rc, const uint64_t *probes, uint32_t slots, uint32_t nprobes,
                      uint32_t nlist, uint32_t dim, uint32_t wpr, uint32_t *planes, RqSlot *slot_out, cudaStream_t st)
{
    if (slots == 0) return;
    launch_k(rq_planes_kernel, dim3(slots), dim3(RQ_PLANES_NT), (size_t)dim * 4, st, rq, rc, probes, nprobes, nlist, dim, wpr,
             planes, slot_out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rq_row_prep(uint32_t *codes, uint64_t n, uint32_t dim, uint32_t wpr, uint32_t *popc, cudaStream_t st)
{
    if (n == 0) return;
    const uint64_t blocks = (n * 32 + 255) / 256;
    rq_row_prep_kernel<<<(unsigned)blocks, 256, 0, st>>>(codes, n, dim, wpr, popc); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_rq_scan(const RqScanArgs &a, int grid, cudaStream_t st)
{
    if (!a.tile_desc || a.wpr % 8) {
        set_error("internal: the RQ scan needs tile descriptors and rows padded to a multiple of 256 bits");
        throw Failure{LGPU_RUNTIME};
    }
    launch_k(rq_scan_kernel, dim3(grid), dim3(RQ_NT), 0, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
