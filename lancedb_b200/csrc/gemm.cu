// gemm.cu -- wgmma / TMA bf16 GEMM used as a *shortlist generator*.
//
// Where the path is a true dense Q x C contraction -- the IVF coarse step
// (IvfModel::find_partitions, SURVEY.md 8a row a3) at large nlist and the flat
// KNNVectorDistance (row a11, BASELINE config 4) -- the reference spends
// B*N*d fused multiply-adds of f32 SIMD.  Here the bulk of that work runs on the Hopper
// tensor cores in bf16 with f32 accumulation in registers:
//     S[q][x] = |x|^2 - 2 * sum_k bf16(q_k) * bf16(x_k)          (= |q-x|^2 - |q|^2, approx.)
// and is only used to pick candidates: the caller keeps every column whose S is within a
// rigorous error band of the k-th best and re-scores those exactly in f32 in lance's
// rounding order (dist.cu), so the final ids / distances are still bit-identical to the
// oracle while >99.9% of the arithmetic is tensor-core work.
//
// Kernel anatomy (one persistent CTA per SM, 384 threads, 128 x 128 output tiles):
//   warps 8-11  producer warpgroup (its registers go to the consumers, setmaxnreg); one lane
//               issues cp.async.bulk.tensor.2d of a 128x64 Q tile and a 128x64 X tile (bf16,
//               K-major, SWIZZLE_128B) into a 6-stage shared-memory ring, mbarrier complete_tx
//               signalling;
//   warps 0-7   two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: each issues
//               wgmma.mma_async m64n128k16 x4 per stage into a 64-register f32 accumulator,
//               keeps one stage's MMAs in flight while it waits for the next, releases a stage
//               once its MMAs have retired, then runs the epilogue (|x|^2 - 2*acc) straight
//               from the registers while the producer already fills the ring for the next tile.
// Tiles are walked N-tile-major so the query tiles of a batch reuse an X tile from L2.
#include "kernels.cuh"

#include <cuda.h>
#include <cuda_bf16.h>

namespace lgpu {

namespace {

constexpr int GM = 128, GN = 128, GK = 64, GSTAGES = 6, G_CONSUMERS = 256, G_THREADS = G_CONSUMERS + 128;
constexpr uint32_t A_STAGE_BYTES = GM * GK * 2;     // 16 KB
constexpr uint32_t B_STAGE_BYTES = GN * GK * 2;     // 16 KB
constexpr uint32_t G_SMEM_TILES = GSTAGES * (A_STAGE_BYTES + B_STAGE_BYTES);   // 192 KB
constexpr uint32_t G_SMEM_BYTES = G_SMEM_TILES + 256 + 1024;                   // + barriers + alignment slack

// ---- raw PTX wrappers ---------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (wgmma): start>>4 | LBO(=1, unused for swizzled K-major)<<16 |
// SBO(=1024 B between 8-row groups)>>4 <<32 | layout SWIZZLE_128B(1) <<62
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr)
{
    uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both bf16 K-major in shared memory; `accumulate` = 0 overwrites D.
// Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4 j + 2 h + e] is row 16 w + l / 4 + 8 h,
// column 8 j + 2 (l % 4) + e.
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// the same with fp16 operands (the multivector MaxSim score, F16MaxSim)
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// D[64 x 128] (+)= popc(A[64 x 256] AND B[128 x 256]^T), both b1 K-major in shared memory (32 bytes of K per row, the
// same bytes as one k16 bf16 slice, so the descriptors and the fragment layout are those of wgmma_m64n128k16)
__device__ __forceinline__ void wgmma_m64n128k256_b1(int (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k256.s32.b1.b1.and.popc "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n\t"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// keeps the compiler from moving accumulator reads above the wgmma.wait_group that makes them valid
__device__ __forceinline__ void fence_acc(float (&d)[64])
{
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void fence_acc(int (&d)[64])
{
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// MMA / score policies of gemm_dist_kernel.  Bf16Dist: bf16 operands, per-row term |x|^2 (f32),
// S = |x|^2 - 2 acc (the shortlist score above).  B1Hamming: packed bits (rows zero-padded to 32 bytes), per-row
// term popc(x) (s32), S = popc(q) + popc(x) - 2 popc(q AND x) = popc(q XOR x) exactly: every term is an integer
// below 2^24, so S is the final Hamming distance and needs no re-score.
struct Bf16Dist {
    static constexpr bool BIN = false, MAXSIM = false;
    static constexpr int K_BOX = GK;          // tensor-map elements per stage row (128 bytes)
    using Acc = float; using Row = float; using Row2 = float2; using Filter = GemmFilter;
    __device__ static __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128k16(d, a, b, acc); }
    __device__ static __forceinline__ int qterm(const GemmFilter &, uint32_t) { return 0; }
    __device__ static __forceinline__ float score(float xn, float acc, int) { return xn - 2.0f * acc; }
};
struct B1Hamming {
    static constexpr bool BIN = true, MAXSIM = false;
    static constexpr int K_BOX = 2 * GK;      // the map is over bytes
    using Acc = int; using Row = int; using Row2 = int2; using Filter = HamFilter;
    __device__ static __forceinline__ void mma(int (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128k256_b1(d, a, b, acc); }
    __device__ static __forceinline__ int qterm(const HamFilter &f, uint32_t q) { return __ldg(f.qpop + q); }
    __device__ static __forceinline__ float score(int xn, int acc, int pq) { return (float)(pq + xn - 2 * acc); }
};
// F16MaxSim: fp16 copies of the NORMALISED query and stored vectors of a multivector column, acc = the approximate
// cosine similarity.  Its epilogue writes nothing dense: per (query vector, document) it keeps the largest similarity
// over the document's run of columns (MaxSimOut, kernels.cuh), one atomicMax per run of a thread's columns.
struct F16MaxSim {
    static constexpr bool BIN = false, MAXSIM = true;
    static constexpr int K_BOX = GK;
    using Acc = float; using Row = float; using Row2 = float2; using Filter = MaxSimOut;
    __device__ static __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128k16_f16(d, a, b, acc); }
    __device__ static __forceinline__ int qterm(const MaxSimOut &, uint32_t) { return 0; }
    __device__ static __forceinline__ float score(float, float acc, int) { return acc; }
};

// LIST: the filtering epilogue for DENSE hit rates (coarse step at many lists), see the epilogue; a separate
// instantiation so that the dense / sparse-filter kernel of the flat path and of the small coarse problems carries
// none of its code.  Pol: Bf16Dist or B1Hamming (above).
template <bool LIST, class Pol>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_dist_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                 const typename Pol::Row *__restrict__ xnorm2, float *__restrict__ out, uint64_t ld_out, uint32_t B,
                 uint64_t N, uint32_t num_kb, typename Pol::Filter flt)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ unsigned char smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;         // SWIZZLE_128B needs 1024 B alignment
    const uint32_t smem_a = base, smem_b = base + GSTAGES * A_STAGE_BYTES;
    const uint32_t bars = base + G_SMEM_TILES;
    const uint32_t full_bar = bars, empty_bar = bars + 8 * GSTAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t num_m = (B + GM - 1) / GM;
    const uint64_t num_n = (N + GN - 1) / GN;
    const uint64_t num_tiles = num_m * num_n;

    if (warp == G_CONSUMERS / 32 && lane == 0) {
        // full: the producer's expect_tx arrival; empty: one arrival per consumer warpgroup
        for (int i = 0; i < GSTAGES; i++) { mbar_init(full_bar + 8 * i, 1); mbar_init(empty_bar + 8 * i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= G_CONSUMERS / 32) {
        // ===== TMA producer =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == G_CONSUMERS / 32 && lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (uint64_t t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const uint32_t m_tile = (uint32_t)(t % num_m);
                const uint64_t n_tile = t / num_m;
                for (uint32_t kb = 0; kb < num_kb; kb++) {
                    mbar_wait(empty_bar + 8 * stage, phase ^ 1);
                    mbar_expect_tx(full_bar + 8 * stage, A_STAGE_BYTES + B_STAGE_BYTES);
                    tma_load_2d(smem_a + stage * A_STAGE_BYTES, &tmap_q, full_bar + 8 * stage, (int)(kb * Pol::K_BOX), (int)(m_tile * GM));
                    tma_load_2d(smem_b + stage * B_STAGE_BYTES, &tmap_x, full_bar + 8 * stage, (int)(kb * Pol::K_BOX), (int)(n_tile * GN));
                    if (++stage == GSTAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of each tile =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const uint32_t wg = threadIdx.x >> 7;
    const bool leader = (threadIdx.x & 127) == 0;
    uint32_t stage = 0, phase = 0;
    typename Pol::Acc acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0;
    for (uint64_t t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const uint32_t m_tile = (uint32_t)(t % num_m);
        const uint64_t n_tile = t / num_m;
        // this thread's rows r0, r0 + 8 and columns c0 + 8 j + {0, 1}
        const uint32_t r0 = m_tile * GM + wg * 64 + (uint32_t)(warp & 3) * 16 + (uint32_t)(lane >> 2);
        const uint64_t c0 = n_tile * GN + 2 * (uint32_t)(lane & 3);
        // |x|^2 of the thread's 32 columns, requested before the MMAs so that the loads land under them; past N: 0
        typename Pol::Row xn[32];
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const uint64_t x = c0 + 8 * j;
            if (x + 1 < N) {
                const typename Pol::Row2 v = __ldg(reinterpret_cast<const typename Pol::Row2 *>(xnorm2 + x));
                xn[2 * j] = v.x; xn[2 * j + 1] = v.y;
            } else {
                xn[2 * j] = x < N ? __ldg(xnorm2 + x) : 0;
                xn[2 * j + 1] = 0;
            }
        }
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < num_kb; kb++) {
            mbar_wait(full_bar + 8 * stage, phase);                      // TMA bytes landed
            const uint64_t da = make_kmajor_sw128_desc(smem_a + stage * A_STAGE_BYTES + wg * (64 * GK * 2));
            const uint64_t db = make_kmajor_sw128_desc(smem_b + stage * B_STAGE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < GK / 16; k++)                            // +32 B (>>4 = 2) per K=16 (b1: K=256) slice
                Pol::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();                                             // the previous stage's MMAs have retired
            if (kb > 0 && leader) mbar_arrive(empty_bar + 8 * prev);
            prev = stage;
            if (++stage == GSTAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (leader) mbar_arrive(empty_bar + 8 * prev);

        if constexpr (Pol::MAXSIM) {
            // MaxSim epilogue: the thread's 32 columns of row q ascend (c0 + 8 j + e), so the columns of one document
            // form one run; the run's largest similarity goes to M[q][doc - row_base] by an ordered-key atomicMax
            // (M zeroed by the caller: key 0 = no column seen)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t q = r0 + 8 * h;
                if (q >= B) continue;
                uint32_t cur = 0xffffffffu;
                float best = 0.f;
#pragma unroll
                for (int j = 0; j < 16; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const uint64_t x = c0 + 8 * j + e;
                        if (x < N) {
                            const uint32_t doc = __ldg(flt.col_row + x);
                            const float v = acc[4 * j + 2 * h + e];
                            if (doc != cur) {
                                if (cur != 0xffffffffu) atomicMax(flt.M + (size_t)q * flt.ldM + (cur - flt.row_base), f32_key(best));
                                cur = doc; best = v;
                            } else {
                                best = fmaxf(best, v);
                            }
                        }
                    }
                if (cur != 0xffffffffu) atomicMax(flt.M + (size_t)q * flt.ldM + (cur - flt.row_base), f32_key(best));
            }
            continue;
        }
        if constexpr (LIST) {
            // Filtering epilogue for DENSE hit rates (the coarse step's lists: ~1.5 % of the columns pass).  One returning
            // atomic per hit, as in the sparse form below, would serialise on the query's counter; instead the 4 lanes
            // that share a row count their hits, ONE atomicAdd per (row, warpgroup tile) reserves the slots, and each
            // lane stores its (column, score) pairs at its prefix inside the reservation.
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t q = r0 + 8 * h;
                const bool live = q < B;
                const float thr = live ? flt.thr[q] : 0.f;
                const int pq = live ? Pol::qterm(flt, q) : 0;
                uint32_t hit = 0;                                        // bit 2 j + e: column c0 + 8 j + e passes
#pragma unroll
                for (int j = 0; j < 16; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++)
                        if (live && c0 + 8 * j + e < N && Pol::score(xn[2 * j + e], acc[4 * j + 2 * h + e], pq) <= thr)
                            hit |= 1u << (2 * j + e);
                const uint32_t n = __popc(hit);
                uint32_t incl = n, v;                                    // inclusive prefix over the row's 4 lanes
                v = __shfl_up_sync(0xffffffffu, incl, 1, 4); if (lane & 3) incl += v;
                v = __shfl_up_sync(0xffffffffu, incl, 2, 4); if ((lane & 3) >= 2) incl += v;
                const uint32_t tot = __shfl_sync(0xffffffffu, incl, 3, 4);
                uint32_t slot = 0;
                if ((lane & 3) == 0 && tot) slot = atomicAdd(flt.count + q, tot);
                slot = __shfl_sync(0xffffffffu, slot, 0, 4) + incl - n;
                if (hit) {
#pragma unroll
                    for (int j = 0; j < 16; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++)
                            if ((hit >> (2 * j + e)) & 1u) {
                                if (slot < flt.cap) {
                                    flt.cand_pos[(size_t)q * flt.cap + slot] = c0 + 8 * j + e;
                                    flt.cand_s[(size_t)q * flt.cap + slot] = Pol::score(xn[2 * j + e], acc[4 * j + 2 * h + e], pq);
                                    if constexpr (Pol::BIN)
                                        flt.cand_ids[(size_t)q * flt.cap + slot] = flt.col_ids ? flt.col_ids[c0 + 8 * j + e] : c0 + 8 * j + e;
                                }
                                slot++;
                            }
                }
            }
            continue;
        }
        if (!Pol::BIN && flt.thr) {
            // filtering epilogue: nothing dense is written; scores not above the per-query threshold are appended to the
            // query's candidate list (rare: ~1e-4 of the columns)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t q = r0 + 8 * h;
                if (q >= B) continue;
                const float thr = flt.thr[q];
#pragma unroll
                for (int j = 0; j < 16; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const uint64_t x = c0 + 8 * j + e;
                        if (x < N && Pol::score(xn[2 * j + e], acc[4 * j + 2 * h + e], 0) <= thr) {
                            const uint32_t slot = atomicAdd(flt.count + q, 1u);
                            if (slot < flt.cap) {
                                flt.cand_pos[(size_t)q * flt.cap + slot] = x;
                                if (flt.cand_ids) flt.cand_ids[(size_t)q * flt.cap + slot] = flt.col_ids ? flt.col_ids[x] : x;
                            }
                        }
                    }
            }
            continue;
        }
        // dense scores: the 4 lanes of a row write 32 contiguous bytes per column group
        const bool vec = (ld_out & 1) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t q = r0 + 8 * h;
            if (q >= B) continue;
            float *orow = out + (size_t)q * ld_out;
            const int pq = Pol::qterm(flt, q);
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const uint64_t x = c0 + 8 * j;
                const float s0 = Pol::score(xn[2 * j], acc[4 * j + 2 * h], pq);
                const float s1 = Pol::score(xn[2 * j + 1], acc[4 * j + 2 * h + 1], pq);
                if (vec && x + 1 < N) {
                    *reinterpret_cast<float2 *>(orow + x) = make_float2(s0, s1);
                } else {
                    if (x < N) orow[x] = s0;
                    if (x + 1 < N) orow[x + 1] = s1;
                }
            }
        }
    }
}

// X f32 [n][d] -> bf16 [n][d] (round to nearest even), |x|^2 and the rounding error |bf16(x) - x| in f32; one warp
// per row
__global__ void to_bf16_norm_kernel(const float *__restrict__ X, uint64_t n, uint32_t d, __nv_bfloat16 *__restrict__ Xb,
                                    float *__restrict__ norm2, float *__restrict__ err)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float *x = X + row * d;
    __nv_bfloat16 *xb = Xb + row * d;
    float s = 0.f, se = 0.f;
    // U loads of the lane in flight at once (a rolled loop waited for one DRAM round trip per element: 13 us for
    // 1024 x 768 on an H100); the sums still run over k = lane, lane + 32, ... in order
    constexpr uint32_t U = 8;
    for (uint32_t k0 = lane; k0 < d; k0 += 32 * U) {
        float v[U];
#pragma unroll
        for (uint32_t u = 0; u < U; u++) v[u] = k0 + 32 * u < d ? x[k0 + 32 * u] : 0.f;
#pragma unroll
        for (uint32_t u = 0; u < U; u++) {
            if (k0 + 32 * u < d) {
                const __nv_bfloat16 b = __float2bfloat16_rn(v[u]);
                xb[k0 + 32 * u] = b;
                s = fmaf(v[u], v[u], s);
                const float e = __bfloat162float(b) - v[u];         // exact: b and v are within a factor of 2
                se = fmaf(e, e, se);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        se += __shfl_xor_sync(0xffffffffu, se, o);
    }
    if (lane == 0 && norm2) norm2[row] = s;
    if (lane == 0 && err) err[row] = sqrtf(se);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        LGPU_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
        if (!p || qres != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled is not available from the CUDA driver");
            throw Failure{LGPU_RUNTIME};
        }
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// bf16 (f16: fp16) row-major [rows][d] matrix (bytes: u8 [rows][d]), box = box_rows x 128 bytes, 128-byte swizzle,
// OOB = zeros
CUtensorMap make_map(const void *ptr, uint64_t rows, uint32_t d, uint32_t box_rows, bool bytes = false, bool f16 = false)
{
    CUtensorMap m;
    cuuint64_t dims[2] = {d, rows};
    cuuint64_t strides[1] = {(cuuint64_t)d * (bytes ? 1 : 2)};
    cuuint32_t box[2] = {(cuuint32_t)(bytes ? 2 * GK : GK), box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode_fn()(&m, bytes ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : (f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16), 2,
                                 const_cast<void *>(ptr), dims, strides, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
        throw Failure{LGPU_RUNTIME};
    }
    return m;
}

__global__ void band_check_kernel(const float *__restrict__ approx, const uint32_t *__restrict__ cnt,
                                  const float *__restrict__ qnorm2, const float *__restrict__ qerr, float xmax, float xerr,
                                  uint32_t d, uint32_t B, uint32_t k, uint32_t kp, uint32_t *__restrict__ flags)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    uint32_t f = 0;
    if (cnt[q] >= kp && kp > 0) {              // list is full: columns beyond it may exist
        const float E = tc_band(qnorm2[q], qerr[q], xmax, xerr, d);
        const float kth = approx[(size_t)q * kp + (k - 1 < kp ? k - 1 : kp - 1)];
        const float last = approx[(size_t)q * kp + kp - 1];
        f = (k >= kp || !(last > kth + 2.0f * E)) ? 1u : 0u;
    }
    flags[q] = f;
}

// thr[q] = (k-th smallest approximate score of the sample) + 2 E_q, or +inf when the sample holds < k rows;
// every true top-k row of the full set has a score <= thr[q] (E_q: tc_band)
__global__ void sample_threshold_kernel(const float *__restrict__ approx, const uint32_t *__restrict__ cnt,
                                        const float *__restrict__ qnorm2, const float *__restrict__ qerr, float xmax,
                                        float xerr, uint32_t d, uint32_t B, uint32_t k, float *__restrict__ thr)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    float t = __int_as_float(0x7f800000);
    if (cnt[q] >= k) {
        const float E = tc_band(qnorm2[q], qerr[q], xmax, xerr, d);
        t = approx[(size_t)q * k + k - 1] + 2.0f * E;
    }
    thr[q] = t;
}
// The same threshold straight from the dense sample scores D[B][ld] (ns columns), one warp per query: the k-th smallest
// by counting bisection over the lane's register copy of the row (no ids, no sorted output, unlike a top-k select),
// stopped when the bracket is a quarter of the band it feeds; any hi with
// count(S <= hi) >= k is a valid bound.  NaN scores never count.  ns <= 32 * VPL.
template <int VPL>
__global__ void __launch_bounds__(128) sample_kth_threshold_kernel(const float *__restrict__ D, uint64_t ld, uint32_t ns,
                                                                  const float *__restrict__ qnorm2,
                                                                  const float *__restrict__ qerr, float xmax, float xerr,
                                                                  uint32_t d, uint32_t B, uint32_t k, float *__restrict__ thr)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= B) return;
    const float *row = D + (size_t)q * ld;
    // global -> shared with cp.async (all of a lane's requests in flight), then shared -> registers: plain register
    // loads come out of ptxas as load -> use -> load, one DRAM round trip after the other (see coarse_finish_kernel)
    __shared__ __align__(16) float s_rows[4][VPL * 32];
    float *srow = s_rows[threadIdx.x >> 5];
    {
        const uint32_t sb = (uint32_t)__cvta_generic_to_shared(srow);
        for (uint32_t i = (uint32_t)lane * 4; i < ld && i < (uint32_t)VPL * 32; i += 128)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sb + i * 4), "l"(row + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
    }
    float v[VPL];
#pragma unroll
    for (int j = 0; j < VPL; j++) v[j] = srow[min((uint32_t)j * 32 + lane, ns - 1)];
    float lo = __int_as_float(0x7f800000), hi = -lo;
    uint32_t nv = 0;
#pragma unroll
    for (int j = 0; j < VPL; j++) {
        if ((uint32_t)j * 32 + lane >= ns) v[j] = __int_as_float(0x7fc00000);
        if (v[j] == v[j]) { lo = fminf(lo, v[j]); hi = fmaxf(hi, v[j]); nv++; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    nv = __reduce_add_sync(0xffffffffu, nv);
    float t = __int_as_float(0x7f800000);
    if (nv >= k && hi < __int_as_float(0x7f800000) && lo > -__int_as_float(0x7f800000)) {
        const float E = tc_band(qnorm2[q], qerr[q], xmax, xerr, d);
        for (int it = 0; it < 24 && hi - lo > 0.25f * E; it++) {        // invariant: count(S <= hi) >= k
            const float mid = 0.5f * lo + 0.5f * hi;
            uint32_t c = 0;
#pragma unroll
            for (int j = 0; j < VPL; j++) c += v[j] <= mid ? 1u : 0u;
            c = __reduce_add_sync(0xffffffffu, c);
            if (c >= k) hi = mid; else lo = mid;
        }
        t = hi + 2.0f * E;
    }
    if (lane == 0) thr[q] = t;
}

__global__ void overflow_flags_kernel(const uint32_t *__restrict__ count, uint32_t cap, uint32_t B, uint32_t *__restrict__ flags)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < B) flags[q] = count[q] > cap ? 1u : 0u;
}

}  // namespace

void launch_sample_threshold(const float *approx, const uint32_t *cnt, const float *qnorm2, const float *qerr, float xmax,
                             float xerr, uint32_t d, uint32_t B, uint32_t k, float *thr, cudaStream_t st)
{
    if (B == 0) return;
    sample_threshold_kernel<<<(B + 127) / 128, 128, 0, st>>>(approx, cnt, qnorm2, qerr, xmax, xerr, d, B, k, thr); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

bool launch_sample_kth_threshold(const float *D, uint64_t ld, uint32_t ns, const float *qnorm2, const float *qerr, float xmax,
                                 float xerr, uint32_t d, uint32_t B, uint32_t k, float *thr, cudaStream_t st)
{
    if (B == 0) return true;
    if (ns == 0 || ns > 2048 || (ld & 3) || ld < ns) return false;       // caller falls back to select + threshold
    const unsigned grid = (B + 3) / 4;
    if (ns <= 1024) launch_k(sample_kth_threshold_kernel<32>, dim3(grid), dim3(128), 0, st, D, ld, ns, qnorm2, qerr, xmax, xerr, d, B, k, thr);
    else launch_k(sample_kth_threshold_kernel<64>, dim3(grid), dim3(128), 0, st, D, ld, ns, qnorm2, qerr, xmax, xerr, d, B, k, thr);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
    return true;
}

void launch_overflow_flags(const uint32_t *count, uint32_t cap, uint32_t B, uint32_t *flags, cudaStream_t st)
{
    if (B == 0) return;
    overflow_flags_kernel<<<(B + 127) / 128, 128, 0, st>>>(count, cap, B, flags); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_band_check(const float *approx, const uint32_t *cnt, const float *qnorm2, const float *qerr, float xmax,
                       float xerr, uint32_t d, uint32_t B, uint32_t k, uint32_t kp, uint32_t *flags, cudaStream_t st)
{
    if (B == 0) return;
    band_check_kernel<<<(B + 127) / 128, 128, 0, st>>>(approx, cnt, qnorm2, qerr, xmax, xerr, d, B, k, kp, flags); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

bool gemm_shape_supported(uint32_t d) { return d >= 8 && d % 8 == 0; }

void launch_to_bf16(const float *X, uint64_t n, uint32_t d, void *Xb, float *norm2, cudaStream_t st, float *err)
{
    if (n == 0) return;
    uint64_t threads = n * 32;
    launch_k(to_bf16_norm_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, X, n, d, reinterpret_cast<__nv_bfloat16 *>(Xb), norm2, err); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

// The filtering epilogue applied to an already written dense score matrix D[B][ld] (same scores, same
// `<= thr` test, same candidate lists up to order): used when the threshold sample was the whole matrix, so
// a second tensor-core pass would only recompute what D already holds.
__global__ void filter_dense_kernel(const float *__restrict__ D, uint64_t ld, uint64_t N, GemmFilter flt)
{
    const uint32_t q = blockIdx.y;
    const float thr = flt.thr[q];
    const float *row = D + (size_t)q * ld;
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < N; x += (uint64_t)gridDim.x * blockDim.x) {
        if (row[x] <= thr) {
            const uint32_t slot = atomicAdd(flt.count + q, 1u);
            if (slot < flt.cap) {
                flt.cand_pos[(size_t)q * flt.cap + slot] = x;
                flt.cand_ids[(size_t)q * flt.cap + slot] = flt.col_ids ? flt.col_ids[x] : x;
            }
        }
    }
}

void launch_filter_dense(const float *D, uint64_t ld, uint32_t B, uint64_t N, const GemmFilter &flt, cudaStream_t st)
{
    if (B == 0 || N == 0) return;
    dim3 grid((unsigned)std::min<uint64_t>((N + 1023) / 1024, 64), B);
    filter_dense_kernel<<<grid, 256, 0, st>>>(D, ld, N, flt); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_gemm_dist(const void *Qb, const void *Xb, const float *xnorm2, uint32_t B, uint64_t N, uint32_t d,
                      float *out, uint64_t ld_out, int num_sms, cudaStream_t st, const GemmFilter *filter)
{
    if (B == 0 || N == 0) return;
    LGPU_REQUIRE(gemm_shape_supported(d), "tensor-core path needs a dimension that is a multiple of 8");
    CUtensorMap mq = make_map(Qb, B, d, GM);
    CUtensorMap mx = make_map(Xb, N, d, GN);
    const uint64_t tiles = (uint64_t)((B + GM - 1) / GM) * ((N + GN - 1) / GN);
    const unsigned grid = (unsigned)std::min<uint64_t>(tiles, (uint64_t)num_sms);
    GemmFilter flt{};
    if (filter) flt = *filter;
    const bool list = flt.thr && flt.cand_s;                  // dense hit rates: one reservation per row and tile
    auto kern = list ? gemm_dist_kernel<true, Bf16Dist> : gemm_dist_kernel<false, Bf16Dist>;
    LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM_BYTES));
    launch_k(kern, dim3(grid), dim3(G_THREADS), G_SMEM_BYTES, st, mq, mx, xnorm2, out, ld_out, B, N, (uint32_t)((d + GK - 1) / GK), flt); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_ham_gemm(const void *Qp, const void *Xp, const uint32_t *xpop, const uint32_t *qpop, uint32_t B, uint64_t N,
                     uint32_t nbytes_pad, float *out, uint64_t ld_out, int num_sms, cudaStream_t st, const GemmFilter *filter)
{
    if (B == 0 || N == 0) return;
    LGPU_REQUIRE(nbytes_pad % 32 == 0, "binary rows must be padded to a multiple of 32 bytes");
    CUtensorMap mq = make_map(Qp, B, nbytes_pad, GM, true);
    CUtensorMap mx = make_map(Xp, N, nbytes_pad, GN, true);
    const uint64_t tiles = (uint64_t)((B + GM - 1) / GM) * ((N + GN - 1) / GN);
    const unsigned grid = (unsigned)std::min<uint64_t>(tiles, (uint64_t)num_sms);
    HamFilter flt{};
    if (filter) static_cast<GemmFilter &>(flt) = *filter;
    flt.qpop = reinterpret_cast<const int *>(qpop);
    auto kern = flt.thr ? gemm_dist_kernel<true, B1Hamming> : gemm_dist_kernel<false, B1Hamming>;
    LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM_BYTES));
    launch_k(kern, dim3(grid), dim3(G_THREADS), G_SMEM_BYTES, st, mq, mx, reinterpret_cast<const int *>(xpop), out, ld_out,
             B, N, (uint32_t)((nbytes_pad + 2 * GK - 1) / (2 * GK)), flt); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_maxsim_gemm(const void *Qh, const void *Xh, uint32_t B, uint64_t N, uint32_t d, const MaxSimOut &out,
                        int num_sms, cudaStream_t st)
{
    if (B == 0 || N == 0) return;
    LGPU_REQUIRE(gemm_shape_supported(d), "tensor-core path needs a dimension that is a multiple of 8");
    CUtensorMap mq = make_map(Qh, B, d, GM, false, true);
    CUtensorMap mx = make_map(Xh, N, d, GN, false, true);
    const uint64_t tiles = (uint64_t)((B + GM - 1) / GM) * ((N + GN - 1) / GN);
    const unsigned grid = (unsigned)std::min<uint64_t>(tiles, (uint64_t)num_sms);
    auto kern = gemm_dist_kernel<false, F16MaxSim>;
    LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM_BYTES));
    launch_k(kern, dim3(grid), dim3(G_THREADS), G_SMEM_BYTES, st, mq, mx, out.xdummy, nullptr, (uint64_t)0, B, N,
             (uint32_t)((d + GK - 1) / GK), out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
