// scan2.cu -- K2+K3, the EXACT form: fused residual / PQ distance-table build / PQ code scan.
//
// Replaces, for a whole batch at once, what lance runs per (query, probed partition) inside ANNIvfSubIndexExec
// [lance, recalled; SURVEY.md 8a rows a4-a7]:
//     r   = q - centroid[p]                                  (residual, L2/cosine)
//     LUT = build_distance_table_l2(codebook, r)             (m x 256 f32)
//     d_j = sum_i LUT[i][code[i][j]]  sequentially in i      (compute_pq_distance)
// Results are bit-identical to oracle.c: every f32 op is an explicit round-to-nearest op in the reference's
// order (the LUT entry uses the f32x8 reduce tree, the row sum is sequential over sub-vectors).
// The default search runs the filter kernel (scan3.cu) first and only the queries it cannot prove
// come here (plus distance-range queries, debug entry points and LGPU_EXACT_SCAN=1); this kernel is also the
// arithmetic pq_rescore_kernel (tables.cu) restates per candidate row.
//
// Work decomposition (GPU-first, not the reference's per-query loop):
//   tile = (partition p, up to 8 of the queries that probe p, up to 1536 of its rows).  A persistent grid (one
//   512-thread CTA per SM) pulls tiles from an atomic counter; tiles are ordered by partition so a partition's
//   codes are read from HBM once and then hit in L2 for the other query groups.
//   The distance table is never materialised whole: it is built 8 sub-spaces at a time into a ring of three
//   64 KB shared-memory buffers laid out [h][c][s][4 queries] (h = query half, c = code, s = sub-space within the
//   chunk), so one LDS.128 returns the entries of 4 queries.  The codebook chunk is read (L2-resident) once per
//   tile and amortised over the 8 queries.
//   Warp specialisation: the table build is FP32-pipe work (23 flops per entry), the scan is
//   shared-memory-gather work; 8 builder warps build chunk ch+1/ch+2 while 8 scanner warps scan chunk ch, handing
//   buffers over with named barriers (bar.arrive / bar.sync).
//   Bank conflicts: a straightforward "lane = row" scan makes 8 lanes of a quarter-warp gather at random codes =>
//   ~2.6-way conflicts.  Here lane l runs `l % 8` sub-space slots behind lane 0 (the code stream in HBM is
//   pre-skewed by row % 8 bytes, see retile.cu), so at any instant the 8 lanes of a quarter-warp read 8
//   *different* sub-spaces = 8 different 16-byte bank groups: conflict-free by construction, while each row still
//   accumulates its sub-vectors strictly in order 0..m-1 in its own register.
// Pipeline details:
//   * no per-tile drain: the stage counter runs on across tiles -- the all-zero "stage nch" of tile n doubles as
//     the "stage -1" of tile n+1 -- and tile descriptors (group.cu::tile_desc_kernel) are claimed two tiles ahead
//     by builder warp 0 into a 4-slot shared ring, so neither role ever waits for a fetch.
//   * the scanners are split by query half (warps 0-3: queries 0-3, warps 4-7: queries 4-7 of the tile): 12 rows
//     x 4 queries of accumulators per thread (48 registers), two scanner warps per scheduler.
//   * the table build is straight-line code: 16 (or 8) tasks per warp and chunk, the metric and the half count
//     are template parameters; each builder warp streams the codebook entries of its tasks through a private
//     cp.async ring, six tasks ahead, across chunk boundaries (CbStage below).
//   * tiles with <= 4 queries use a 4-codes-per-warp mapping (HALVES = 1): half the build work.
// Algorithmic bytes per tile row and query: m code bytes (SURVEY.md 8d).
#include "kernels.cuh"
#include "scan_common.cuh"

namespace lgpu {

namespace {

constexpr int S2_PW = 8, S2_CW = 8;                 // builder / scanner warps
constexpr int S2_PT = S2_PW * 32, S2_NT = (S2_PW + S2_CW) * 32;
constexpr int S2_CT = 128;                          // scanner threads per query half
constexpr int S2_RMAX = 12;                         // rows per scanner thread: 128 * 12 = SCAN_ROWS_TILE_MID
// registers per builder / scanner thread: the builders schedule better with more registers until the scanners
// start to spill; an even split is the default (override with -DS2_PREG_V / -DS2_CREG_V).
#ifndef S2_PREG_V
#define S2_PREG_V 128
#endif
#ifndef S2_CREG_V
#define S2_CREG_V 128
#endif
constexpr int S2_PREG = S2_PREG_V, S2_CREG = S2_CREG_V;   // 256 * PREG + 256 * CREG <= 65536 registers
constexpr int S2_SLOTS = 4;                         // tile-descriptor ring
constexpr int S2_SLOT_BYTES = 128;
constexpr int S2_STAGE_BYTES = 3072;                // per builder warp: 6 x 512 B (2-code tasks) or 3 x 1 KB
static_assert(SCAN_ROWS_TILE_MID == S2_CT * S2_RMAX, "rows_tile");
static_assert(S2_PT * S2_PREG + S2_CW * 32 * S2_CREG <= 65536, "register budget");

__device__ __forceinline__ int ring_next(int b) { return b == 2 ? 0 : b + 1; }

// ---------------------------------------------------------------- shared-memory carve-up
template <int DSUB>
struct Smem {
    static constexpr int RB = SCAN_G * 8 * DSUB;                     // floats per residual chunk [g][s][e]
    static constexpr size_t LUT = 0;
    static constexpr size_t RBUF = 3 * (size_t)SCAN_LUT_BYTES;
    static constexpr size_t TILES = RBUF + 2 * (size_t)RB * sizeof(float);
    static constexpr size_t STAGE = TILES + S2_SLOTS * S2_SLOT_BYTES;    // codebook staging rings (DSUB == 8)
    static constexpr size_t TOTAL = STAGE + (DSUB == 8 ? S2_PW * S2_STAGE_BYTES : 0);
};

__device__ __forceinline__ const TileDesc *slot_ptr(const unsigned char *tiles, uint32_t n)
{
    return reinterpret_cast<const TileDesc *>(tiles + (n & (S2_SLOTS - 1)) * S2_SLOT_BYTES);
}

// ---------------------------------------------------------------- builder (producer) side
template <int DSUB>
struct Resid {
    static constexpr int RB = Smem<DSUB>::RB;
    static constexpr int RPT = (RB + S2_PT - 1) / S2_PT;
    float vq[RPT], vc[RPT];
    // global loads for residual chunk `ch` of tile T into registers; the subtraction (q - centroid, or
    // q - 0 for dot) happens in store(), a whole build stage later, so the loads are never waited on here
    template <bool DOT>
    __device__ __forceinline__ void load(const ScanArgs &a, const TileDesc *T, uint32_t ch, int tid)
    {
        const uint32_t p = T->p;
        const int ng = (int)T->ng;
        const float *cenp = a.centroids + (size_t)p * a.dim;
#pragma unroll
        for (int u = 0; u < RPT; u++) {
            const int idx = tid + u * S2_PT;
            float rq = 0.f, rc = 0.f;
            if (idx < RB) {
                const int g = idx / (8 * DSUB), rem = idx - g * (8 * DSUB);
                const int ss = rem / DSUB, e = rem - ss * DSUB;
                const uint32_t i = ch * 8 + ss;
                if (g < ng && i < a.m) {
                    const uint32_t dimi = i * DSUB + e;
                    rq = __ldg(a.queries + (size_t)T->q[g] * a.dim + dimi);
                    if (!DOT) rc = __ldg(cenp + dimi);
                }
            }
            vq[u] = rq; vc[u] = rc;
        }
    }
    __device__ __forceinline__ void store(float *dst, int tid) const
    {
#pragma unroll
        for (int u = 0; u < RPT; u++) {
            const int idx = tid + u * S2_PT;
            if (idx < RB) {
                int at = idx;
                if constexpr (DSUB == 8) {      // 16-byte unit u -> u ^ ((u >> 3) & 1): conflict-free LDS.128 reads
                    const int unit = idx >> 2;
                    at = ((unit ^ ((unit >> 3) & 1)) << 2) | (idx & 3);
                }
                dst[at] = __fsub_rn(vq[u], vc[u]);
            }
        }
    }
};

// ---- codebook staging (DSUB == 8).  A builder warp's task needs CPT codes x 8 sub-spaces x 32 B of the
// codebook chunk = CPT * 256 contiguous bytes.  Instead of loading them into registers a few tasks ahead
// (each load exposes an L2 round trip), each warp streams them with cp.async
// (LDGSTS, 16 B per lane) into a private ring of D = 3072 / (CPT * 256) slots, D tasks ahead, and reads
// its (code, sub-space) entry back with two LDS.128 one task ahead.  16-byte unit u of a code's 256 B
// is stored at unit u ^ ((u >> 3) & 1) so that the eight lanes of a quarter-warp (sub-spaces 0..7, 32 B
// apart) hit eight different bank groups.
struct CbStage {
    uint32_t base;      // shared-space address of this warp's ring
    uint32_t so;        // byte offset of the slot holding the task whose entry is in `cur`
    float4 cur[2];      // codebook entry (this lane's code, sub-space) of the current task
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float4 lds128(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t stage_swz(int lane) { return (uint32_t)((lane ^ ((lane >> 3) & 1)) << 4); }

// issue the copy of task k of chunk ch (CPT codes) into the slot at byte offset `so`
template <int CPT>
__device__ __forceinline__ void stage_issue(const ScanArgs &a, const CbStage &cs, uint32_t so, uint32_t ch, int k,
                                            int pw, int lane)
{
    const unsigned char *src = reinterpret_cast<const unsigned char *>(a.cb_tiled) +
                               ((size_t)ch * 256 + CPT * (pw + S2_PW * k)) * 256 + lane * 16;
    const uint32_t dst = cs.base + so + stage_swz(lane);
    cp_async16(dst, src);
    if constexpr (CPT == 4) cp_async16(dst + 512, src + 512);
}

// start of a tile: tasks 0..D-1 of chunk 0 in flight, ring phase reset
template <int CPT>
__device__ __forceinline__ void stage_start(const ScanArgs &a, CbStage &cs, int pw, int lane)
{
    constexpr int SLOT = CPT * 256, D = S2_STAGE_BYTES / SLOT;
#pragma unroll
    for (int k = 0; k < D; k++) {
        stage_issue<CPT>(a, cs, k * SLOT, 0, k, pw, lane);
        cp_async_commit();
    }
    cs.so = 0;
}

// The residuals of this lane's sub-space for its 4 queries (DSUB == 8), packed for the f32x2 ops.  Loaded by the
// builder loop *before* it waits for the ring buffer, so the LDS latency hides behind the barrier.
struct ResidRegs {
    uint64_t pr[4][4];          // [query][dim pair]
};
template <int DSUB>
__device__ __forceinline__ void load_resid_regs(ResidRegs &rr, int rslot, bool two_halves, int lane)
{
    if constexpr (DSUB == 8) {
        extern __shared__ __align__(1024) unsigned char smem[];
        const int s = lane & 7;
        const int h = two_halves ? ((lane >> 3) & 1) : 0;
        const uint32_t base = (uint32_t)__cvta_generic_to_shared(smem + Smem<DSUB>::RBUF) +
                              (uint32_t)rslot * Smem<DSUB>::RB * 4 + (uint32_t)(4 * h) * 256 +
                              (uint32_t)(((2 * s) ^ (s >> 2)) << 4);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t at = base + j * 256;
            const float4 lo = lds128(at), hi = lds128(at ^ 16u);
            rr.pr[j][0] = pk2(lo.x, lo.y); rr.pr[j][1] = pk2(lo.z, lo.w);
            rr.pr[j][2] = pk2(hi.x, hi.y); rr.pr[j][3] = pk2(hi.z, hi.w);
        }
    }
}

// Build one 8-sub-space chunk of the distance table into ring buffer `b`.
//   HALVES == 2: lane -> (s = lane & 7, h = (lane >> 3) & 1, cc = lane >> 4); a warp task covers 2 codes
//                x 8 sub-spaces x both query halves; 16 tasks per warp.
//   HALVES == 1: lane -> (s = lane & 7, cq = lane >> 3); a warp task covers 4 codes x 8 sub-spaces for
//                queries 0-3; 8 tasks per warp.
// DSUB == 8: on entry `cs` has the copies of this chunk's first D tasks in flight (or landed) and, from the
// second chunk of a tile on, the entry of task 0 in cs.cur; `has_next` = the tile has another chunk, whose
// first D tasks are issued from here.  `rr` = this lane's residuals (load_resid_regs).
template <int DSUB, bool DOT, int HALVES>
__device__ __forceinline__ void build_chunk(const ScanArgs &a, uint32_t ch, int b, int rslot, CbStage &cs,
                                            const ResidRegs &rr, bool has_next, int pw, int lane)
{
    extern __shared__ __align__(1024) unsigned char smem[];      // declared here so every access is a plain
    unsigned char *const lut = smem + Smem<DSUB>::LUT;           // shared-space LDS/STS
    const float *const rsrc_chunk = reinterpret_cast<const float *>(smem + Smem<DSUB>::RBUF) + rslot * Smem<DSUB>::RB;
    constexpr int CPT = HALVES == 2 ? 2 : 4;
    constexpr int NTASK = 256 / CPT / S2_PW;                   // 16 or 8
    const int s = lane & 7;
    const int h = HALVES == 2 ? ((lane >> 3) & 1) : 0;
    const int csel = HALVES == 2 ? (lane >> 4) : (lane >> 3);
    const bool sub_ok = (ch * 8 + s) < a.m;
    const float *rsrc = rsrc_chunk + ((4 * h) * 8 + s) * DSUB;                // + j * 8 * DSUB per query
    unsigned char *dst = lut + b * SCAN_LUT_BYTES + h * SCAN_LUT_HALF + s * 16 + (CPT * pw + csel) * 128;
    constexpr int DST_STRIDE = CPT * S2_PW * 128;                              // bytes between tasks

    if constexpr (DSUB == 8) {
        constexpr int SLOT = CPT * 256, D = S2_STAGE_BYTES / SLOT;             // 6 or 3 tasks in flight
        static_assert(D >= 2 && D <= NTASK, "staging depth");
        const uint64_t (&pr)[4][4] = rr.pr;
        // this lane's entry inside a slot: code csel, sub-space s, swizzled 16-byte units 2s and 2s+1
        const uint32_t ent = cs.base + (uint32_t)csel * 256 + (uint32_t)(((2 * s) ^ (s >> 2)) << 4);
        if (ch == 0) {                          // first task of the tile: its copy is the oldest of D groups
            cp_async_wait<D - 1>();
            __syncwarp();
            cs.cur[0] = lds128(ent + cs.so); cs.cur[1] = lds128((ent + cs.so) ^ 16u);
        }
#pragma unroll
        for (int k = 0; k < NTASK; k++) {
            // entry of task k is in cs.cur, its slot (cs.so) is free: refill it with task k + D
            cp_async_wait<D - 2>();             // task k+1 has landed (this lane's part) ...
            __syncwarp();                       // ... and every lane's part; also orders last LDS before the refill
            if (k + D < NTASK) stage_issue<CPT>(a, cs, cs.so, ch, k + D, pw, lane);
            else if (has_next) stage_issue<CPT>(a, cs, cs.so, ch + 1, k + D - NTASK, pw, lane);
            cp_async_commit();                  // (possibly empty: keeps the group count per task at one)
            const uint32_t so_next = cs.so + SLOT == S2_STAGE_BYTES ? 0u : cs.so + SLOT;
            float4 n0 = cs.cur[0], n1 = cs.cur[1];
            if (k + 1 < NTASK || has_next) { n0 = lds128(ent + so_next); n1 = lds128((ent + so_next) ^ 16u); }
            const float4 c0 = cs.cur[0], c1 = cs.cur[1];
            float4 out;
            if constexpr (!DOT) {
                const uint64_t pc[4] = {pk2(c0.x, c0.y), pk2(c0.z, c0.w), pk2(c1.x, c1.y), pk2(c1.z, c1.w)};
                out = l2_tree8_packed_x4(pr, pc, a.fzero2);      // zero-padded codebook & residual => +0 past m
            } else {
                const float cv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
                float o[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    float rr[8];
#pragma unroll
                    for (int e = 0; e < 4; e++) upk2(pr[j][e], rr[2 * e], rr[2 * e + 1]);
                    o[j] = sub_ok ? subvec_dot_dist<8>(rr, cv) : 0.f;
                }
                out = make_float4(o[0], o[1], o[2], o[3]);
            }
            *reinterpret_cast<float4 *>(dst + k * DST_STRIDE) = out;
            cs.cur[0] = n0; cs.cur[1] = n1;
            cs.so = so_next;
        }
    } else {
        (void)cs; (void)has_next; (void)rr;
        const float *cbp = a.cb_tiled + (((size_t)ch * 256 + CPT * pw + csel) * 8 + s) * DSUB;
        for (int k = 0; k < NTASK; k++) {
            float cbv[DSUB], rr[DSUB], o[4] = {0.f, 0.f, 0.f, 0.f};
            load_vec<DSUB>(cbv, cbp + (size_t)k * CPT * S2_PW * 8 * DSUB);
            if (sub_ok) {
#pragma unroll
                for (int j = 0; j < 4; j++) {
#pragma unroll
                    for (int e = 0; e < DSUB; e++) rr[e] = rsrc[j * 8 * DSUB + e];
                    o[j] = DOT ? subvec_dot_dist<DSUB>(rr, cbv) : subvec_l2<DSUB>(rr, cbv);
                }
            }
            *reinterpret_cast<float4 *>(dst + k * DST_STRIDE) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
}

template <int DSUB, bool DOT>
__device__ __forceinline__ void producer_loop(const ScanArgs &a, uint32_t total, int tid)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *const lut = smem + Smem<DSUB>::LUT;
    float *const rbuf = reinterpret_cast<float *>(smem + Smem<DSUB>::RBUF);
    unsigned char *const tiles = smem + Smem<DSUB>::TILES;
    constexpr int RB = Smem<DSUB>::RB;
    const int lane = tid & 31, pw = tid >> 5;
    const uint32_t nch = a.nch;

    Resid<DSUB> res;
    CbStage cs;
    cs.base = (uint32_t)__cvta_generic_to_shared(smem + Smem<DSUB>::STAGE) + (uint32_t)pw * S2_STAGE_BYTES;
    cs.so = 0;
    cs.cur[0] = cs.cur[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    {   // first tile: residual chunk 0 and the first codebook copies
        const TileDesc *T0 = slot_ptr(tiles, 0);
        if (T0->ng) {
            if constexpr (DSUB == 8) {
                if (T0->ng > 4) stage_start<2>(a, cs, pw, lane); else stage_start<4>(a, cs, pw, lane);
            }
            res.template load<DOT>(a, T0, 0, tid);
            res.store(rbuf, tid);
        }
    }
    bar_sync(BAR_PROD, S2_PT);

    int b = 0;                 // ring buffer of the current stage
    uint32_t gs = 0;           // stages issued so far (only "< 2" matters)
    for (uint32_t n = 0;; n++) {
        const TileDesc *T = slot_ptr(tiles, n);
        const int ng = (int)T->ng;
        if (ng == 0) break;
        const TileDesc *Tn = slot_ptr(tiles, n + 1);
        const int ng_next = (int)Tn->ng;
        uint32_t t_claim = 0, t_word = 0;
        for (uint32_t ch = 0; ch <= nch; ch++) {
            // --- tile look-ahead (warp 0): claim at stage 0, read the descriptor at stage 1 ---
            if (pw == 0) {
                if (ch == 0) {
                    if (lane == 0) t_claim = atomicAdd(a.tile_counter, 1u);
                    t_claim = __shfl_sync(0xffffffffu, t_claim, 0);
                } else if (ch == 1) {
                    t_word = 0;
                    if (lane < (int)(sizeof(TileDesc) / 4) && t_claim < total)
                        t_word = __ldg(reinterpret_cast<const uint32_t *>(a.tile_desc + t_claim) + lane);
                }
            }
            // --- residual prefetch: next chunk of this tile, or chunk 0 of the next tile ---
            const bool res_here = ch + 1 < nch;
            const bool res_next = (ch == nch) && ng_next != 0;
            if (res_here) res.template load<DOT>(a, T, ch + 1, tid);
            else if (res_next) {
                res.template load<DOT>(a, Tn, 0, tid);
                if constexpr (DSUB == 8) {      // this stage builds nothing: start the next tile's codebook copies
                    if (ng_next > 4) stage_start<2>(a, cs, pw, lane); else stage_start<4>(a, cs, pw, lane);
                }
            }

            ResidRegs rr;
            if (ch < nch) load_resid_regs<DSUB>(rr, (int)(ch & 1), ng > 4, lane);
            if (gs >= 2) bar_sync(BAR_EMPTY + b, S2_NT);          // scanners are done with stage gs-2
            if (ch == nch) {                                       // all-zero row for the lagging lanes
                if (tid < 64)
                    reinterpret_cast<float *>(lut + b * SCAN_LUT_BYTES + (tid >> 5) * SCAN_LUT_HALF)[tid & 31] = 0.f;
            } else {
                const bool has_next = ch + 1 < nch;
                if (ng > 4) build_chunk<DSUB, DOT, 2>(a, ch, b, (int)(ch & 1), cs, rr, has_next, pw, lane);
                else build_chunk<DSUB, DOT, 1>(a, ch, b, (int)(ch & 1), cs, rr, has_next, pw, lane);
            }
            if (pw == 0 && ch == 1 && lane < (int)(sizeof(TileDesc) / 4))   // publish tile n+2 before FULL(stage 1)
                reinterpret_cast<uint32_t *>(const_cast<TileDesc *>(slot_ptr(tiles, n + 2)))[lane] = t_word;
            bar_arrive(BAR_FULL + b, S2_NT);
            if (res_here) res.store(rbuf + ((ch + 1) & 1) * RB, tid);
            else if (res_next) res.store(rbuf, tid);
            bar_sync(BAR_PROD, S2_PT);
            b = ring_next(b);
            gs++;
        }
    }
}

// ---------------------------------------------------------------- scanner (consumer) side
// R rows per thread (row = row0 + ct + r * 128), the 4 queries of half h.  R == 0: this half has no
// queries in the tile; the thread only keeps the barrier protocol going.
template <int DSUB, int R>
__device__ __forceinline__ int consume_tile(const ScanArgs &a, const TileDesc *T, bool next_exists, int b, int h,
                                            int ct)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const unsigned char *const lut_half = smem + Smem<DSUB>::LUT + h * SCAN_LUT_HALF;
    const uint32_t nch = a.nch;
    const uint32_t p = T->p, row0 = T->row0, nrows = T->nrows;
    const int ng = (int)T->ng;
    const int sig = ct & 7;                               // this lane's skew (== row % 8)
    const uint32_t n_p = a.part_n[p], npad = a.part_npad[p];
    const uint2 *cs = reinterpret_cast<const uint2 *>(a.codes + a.code_base[p]);   // [nch+1][npad]

    constexpr int RR = R > 0 ? R : 1;
    float acc[RR][4];
    bool valid[RR];
    uint2 wn[RR];
#pragma unroll
    for (int r = 0; r < RR; r++) {
#pragma unroll
        for (int g = 0; g < 4; g++) acc[r][g] = 0.f;
        const uint32_t row = row0 + ct + r * S2_CT;
        valid[r] = R > 0 && row < row0 + nrows && row < n_p;
        wn[r] = valid[r] ? __ldg(cs + row) : make_uint2(0u, 0u);
    }

    for (uint32_t it = 0; it <= nch; it++) {
        uint2 w[RR];
#pragma unroll
        for (int r = 0; r < RR; r++) w[r] = wn[r];
        if (R > 0 && it < nch) {                           // prefetch the next block of code bytes
#pragma unroll
            for (int r = 0; r < RR; r++) {
                const uint32_t row = row0 + ct + r * S2_CT;
                wn[r] = valid[r] ? __ldg(cs + (size_t)(it + 1) * npad + row) : make_uint2(0u, 0u);
            }
        }
        bar_sync(BAR_FULL + b, S2_NT);
        const int bp = b == 0 ? 2 : b - 1;                 // buffer of the previous stage
        if (R > 0) {
            const uint32_t base_cur = (uint32_t)b * SCAN_LUT_BYTES;
            const uint32_t base_prev = (uint32_t)bp * SCAN_LUT_BYTES;
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const uint32_t off = ((e < sig) ? base_prev : base_cur) + (((e - sig) & 7) << 4);
#pragma unroll
                for (int r = 0; r < RR; r++) {
                    const uint32_t word = (e < 4) ? w[r].x : w[r].y;
                    const uint32_t c = (word >> (8 * (e & 3))) & 0xffu;
                    const float4 v = *reinterpret_cast<const float4 *>(lut_half + off + (c << 7));
                    acc[r][0] = __fadd_rn(acc[r][0], v.x);
                    acc[r][1] = __fadd_rn(acc[r][1], v.y);
                    acc[r][2] = __fadd_rn(acc[r][2], v.z);
                    acc[r][3] = __fadd_rn(acc[r][3], v.w);
                }
            }
        }
        // the previous stage's buffer is free again; the builders wait for it iff they still have a stage
        // (this tile's or the next tile's) to put there
        if (it + 2 <= nch || next_exists) bar_arrive(BAR_EMPTY + bp, S2_NT);
        b = ring_next(b);
    }

    // ---- epilogue: metric post-processing, one f32 per (row, query) to HBM ----
    if (R > 0) {
        const float mcorr = (float)(a.m - 1);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int g = 4 * h + j;
            if (g < ng) {
                float *out = a.dist_out + T->out[g];
#pragma unroll
                for (int r = 0; r < RR; r++) {
                    if (valid[r]) {
                        float v = acc[r][j];
                        if (a.metric == LGPU_COSINE) v = __fmul_rn(v, 0.5f);
                        else if (a.metric == LGPU_DOT) v = __fsub_rn(v, mcorr);
                        out[row0 + ct + r * S2_CT] = v;
                    }
                }
            }
        }
    }
    return b;
}

template <int DSUB>
__device__ __forceinline__ void consumer_loop(const ScanArgs &a, int tid)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const unsigned char *const tiles = smem + Smem<DSUB>::TILES;
    const int cidx = tid - S2_PT;
    const int h = cidx >> 7, ct = cidx & (S2_CT - 1);
    int b = 0;
    for (uint32_t n = 0;; n++) {
        const TileDesc *T = slot_ptr(tiles, n);
        const int ng = (int)T->ng;
        if (ng == 0) break;
        const bool next_exists = slot_ptr(tiles, n + 1)->ng != 0;
        const int R = 4 * h < ng ? (int)((T->nrows + S2_CT - 1) / S2_CT) : 0;      // uniform per half
#define LGPU_CONSUME(RR) b = consume_tile<DSUB, RR>(a, T, next_exists, b, h, ct)
        if (R == 0) LGPU_CONSUME(0);
        else if (R <= 2) LGPU_CONSUME(2);
        else if (R <= 4) LGPU_CONSUME(4);
        else if (R <= 6) LGPU_CONSUME(6);
        else if (R <= 8) LGPU_CONSUME(8);
        else if (R <= 10) LGPU_CONSUME(10);
        else LGPU_CONSUME(12);
#undef LGPU_CONSUME
    }
}

// ---------------------------------------------------------------- kernel
template <int DSUB, bool DOT>
__global__ void __launch_bounds__(S2_NT, 1) scan2_kernel(ScanArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x;
    if (a.gate && *a.gate == 0) return;
    const uint32_t total = *a.total_tiles;
    unsigned char *const tiles = smem + Smem<DSUB>::TILES;

    // "stage -1" of the first tile: zero code-0 row in ring buffer 2 (both halves)
    if (tid < 64)
        reinterpret_cast<float *>(smem + 2 * SCAN_LUT_BYTES + (tid >> 5) * SCAN_LUT_HALF)[tid & 31] = 0.f;
    // tiles 0 and 1 of this CTA
    if (tid < 32) {
        uint32_t t0 = 0, t1 = 0;
        if (tid == 0) { t0 = atomicAdd(a.tile_counter, 1u); t1 = atomicAdd(a.tile_counter, 1u); }
        t0 = __shfl_sync(0xffffffffu, t0, 0);
        t1 = __shfl_sync(0xffffffffu, t1, 0);
        if (tid < (int)(sizeof(TileDesc) / 4)) {
            uint32_t w0 = 0, w1 = 0;
            if (t0 < total) w0 = __ldg(reinterpret_cast<const uint32_t *>(a.tile_desc + t0) + tid);
            if (t1 < total) w1 = __ldg(reinterpret_cast<const uint32_t *>(a.tile_desc + t1) + tid);
            reinterpret_cast<uint32_t *>(tiles)[tid] = w0;
            reinterpret_cast<uint32_t *>(tiles + S2_SLOT_BYTES)[tid] = w1;
        }
    }
    __syncthreads();

    if (tid < S2_PT) {
        if constexpr (S2_PREG < S2_CREG) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(S2_PREG));
        else if constexpr (S2_PREG > S2_CREG) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(S2_PREG));
        producer_loop<DSUB, DOT>(a, total, tid);
    } else {
        if constexpr (S2_PREG < S2_CREG) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(S2_CREG));
        else if constexpr (S2_PREG > S2_CREG) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(S2_CREG));
        consumer_loop<DSUB>(a, tid);
    }
}

template <int DSUB, bool DOT>
void launch2(const ScanArgs &a, int grid, cudaStream_t st)
{
    constexpr size_t smem = Smem<DSUB>::TOTAL;
    auto kern = scan2_kernel<DSUB, DOT>;
    LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    launch_k(kern, dim3(grid), dim3(S2_NT), smem, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

template <int DSUB>
void launch2_metric(const ScanArgs &a, int grid, cudaStream_t st)
{
    if (a.metric == LGPU_DOT) launch2<DSUB, true>(a, grid, st);
    else launch2<DSUB, false>(a, grid, st);
}

}  // namespace

bool scan_dsub_supported(uint32_t dsub)
{
    return dsub == 1 || dsub == 2 || dsub == 4 || dsub == 8 || dsub == 16 || dsub == 32;
}

void launch_scan2(const ScanArgs &a, uint32_t dsub, int grid, cudaStream_t st)
{
    if (!a.tile_desc || a.rows_tile != SCAN_ROWS_TILE_MID) {
        set_error("internal: the exact scan needs tile descriptors built with rows_tile 1536");
        throw Failure{LGPU_RUNTIME};
    }
    switch (dsub) {
    case 1: launch2_metric<1>(a, grid, st); break;
    case 2: launch2_metric<2>(a, grid, st); break;
    case 4: launch2_metric<4>(a, grid, st); break;
    case 8: launch2_metric<8>(a, grid, st); break;
    case 16: launch2_metric<16>(a, grid, st); break;
    case 32: launch2_metric<32>(a, grid, st); break;
    default:
        set_error("unsupported PQ sub-vector length (dim/num_sub_vectors must be 1,2,4,8,16 or 32)");
        throw Failure{LGPU_INVALID_INPUT};
    }
}

}  // namespace lgpu
