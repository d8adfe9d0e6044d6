// scan3.cu -- K2+K3 as a FILTER: the PQ code scan over 16-bit per-QUERY tables.
//
// The exact kernel (scan2.cu) has to build one f32 distance table per (query, probed partition), because
// lance's table is on the residual q - c_p [lance, recalled; SURVEY.md 8a rows a4-a5]: 20 480 tables per
// 1024-query batch of BASELINE config 2, and that build -- its shared-memory staging and its f32 arithmetic --
// not the scan, bounds the exact kernel.
// Algebraically (tables.cu has the derivation)
//     d(q, row r of partition p) = sum_i T_q[i][code_i(r)]  +  A(q,p)  +  R(r)
// with ONE table per query, T_q[i][c] = |q_i - codebook_i[c]|^2 (1 - q_i.codebook_i[c] for dot), a scalar per
// (query, probe) and a constant per stored row.  tables.cu quantises T_q to 16 bits,
//     T_q[i][c] in [min_i + step_q n, min_i + step_q (n + 1)),   n = n_q[i][c] in [0, floor(65535 / m)],
// so that the m entries of a row add up inside one 16-bit lane: this kernel accumulates EIGHT queries per
// 128-bit shared-memory load with four 32-bit integer adds, half the shared-memory wavefronts and a quarter
// of the arithmetic per (row, sub-space, query) of the f32 form, and builds no table at all.
// The result  L = step_q * sum n + (sum_i min_i + A) + R  is a rigorous LOWER bound of the exact distance with a
// known band (band_check3 in tables.cu); the caller keeps the kp best rows by L, proves the exact top-k is among
// them, re-scores those few rows in the oracle's arithmetic (pq_rescore_kernel) and redoes unproven queries with
// the exact kernel, so the reported ids and distances are bit-identical to the exact path.
//
// Pipeline: identical hand-over protocol to scan2.cu (tests/test_scan2_protocol.py models it): persistent CTAs,
// a ring of three shared chunk buffers, named barriers FULL/EMPTY between 8 stager warps and 8 scanner warps, the
// stage counter running on across tiles, tile descriptors claimed two tiles ahead.
//   tile    = (partition, <= 8 of the queries probing it, <= 1536 rows); two CTAs per SM
//   chunk   = 8 sub-spaces: shared [256 codes][8 sub-spaces][8 queries] u16 = 32 KB
//   stagers : thread c owns code c.  It loads the 16 bytes (8 sub-spaces) of each of the tile's queries for code c
//             from the L2-resident query tables (8 x LDG.128, issued a whole stage ahead), transposes 8x8 u16 in
//             registers (32 PRMT) and writes eight 16-byte units [sub-space][8 queries].  The global tables are
//             stored ROTATED -- position j of code c holds sub-space (j + c) mod 8 -- so that in step j the eight
//             lanes of a quarter-warp write eight different 16-byte slots: conflict-free without a per-lane
//             register rotation.
//   scanners: thread = rows row0 + ct + 256 r (r < 6); the skewed code stream (retile.cu) makes the eight lanes of
//             a quarter-warp read eight different sub-space slots, so every LDS.128 is conflict-free whatever the
//             codes are; accumulators are 4 x u32 per row (8 queries x u16).
// Algorithmic bytes per tile row and query: m code bytes (SURVEY.md 8d), as for the exact kernel.
#include "kernels.cuh"
#include "scan_common.cuh"

#include <math_constants.h>

namespace lgpu {

namespace {

constexpr int S3_PW = 8, S3_CW = 8;                 // stager / scanner warps
constexpr int S3_PT = S3_PW * 32, S3_CT = S3_CW * 32, S3_NT = S3_PT + S3_CT;
constexpr int S3_RMAX = 6;                          // rows per scanner thread
// two CTAs per SM (2 x 512 threads, 2 x 97 KB of shared memory): while one CTA sits in a tile's prologue /
// epilogue or at a barrier, the other keeps the shared-memory pipe busy.  64 registers per thread at launch,
// re-split by role: the stagers hold one 32-register slab, the scanners 6 rows x (4 accumulators + 2 + 2 code words)
constexpr int S3_PREG = 48, S3_CREG = 80;
static_assert(S3_PT * S3_PREG + S3_CT * S3_CREG <= 32768, "register budget of half an SM");
constexpr int S3_BUF = 32768;                       // one chunk buffer
constexpr int S3_SLOTS = 4, S3_SLOT_BYTES = 128;    // tile-descriptor ring
constexpr size_t S3_TILES = 3 * (size_t)S3_BUF;
constexpr int S3_SCR = 32;                          // words per bank of threshold scratch
// + two banks of threshold scratch + mbarriers + the candidate epilogue's per-query scalars
constexpr size_t S3_SMEM = S3_TILES + S3_SLOTS * S3_SLOT_BYTES + 2 * S3_SCR * 4 + 32 + SCAN_G * 16;
constexpr int S3_LIST_PER = CAND_CAP_MAX / S3_CT;  // list keys per scanner thread in a list-based tightening
constexpr int S3_LIST_STEPS = 10;
constexpr int BAR_SCAN = 8;                         // named barrier of the 256 scanner threads (candidate mode)
// FULL hand-over (stagers -> scanners) as mbarriers, one per ring buffer: a named barrier made the 8 scanner warps
// wait for EACH OTHER at every stage (bar.sync counts all of them), so a stage took as long as its slowest warp; with
// an mbarrier only the stagers arrive (one elected lane per warp) and every scanner warp goes on as soon as the
// buffer is full.  The scanners can then drift apart by at most two stages (the EMPTY barrier, which the stagers
// wait on, needs all of them).  LGPU_S3_NAMED_FULL=1 at build time restores the named barrier (A/B).
#ifndef LGPU_S3_NAMED_FULL
#define LGPU_S3_NAMED_FULL 0
#endif
constexpr size_t S3_MBAR_OFF = S3_TILES + S3_SLOTS * S3_SLOT_BYTES + 2 * S3_SCR * 4;   // 3 x 8 bytes, 8-byte aligned
constexpr size_t S3_QS_OFF = S3_MBAR_OFF + 32;     // [SCAN_G][step, cst, slack, -] f32
static_assert(S3_QS_OFF + SCAN_G * 16 == S3_SMEM, "shared-memory layout");
static_assert(SCAN3_ROWS_TILE == S3_CT * S3_RMAX, "rows_tile");
static_assert(S3_PT == 256, "one stager thread per code");

__device__ __forceinline__ int ring_next3(int b) { return b == 2 ? 0 : b + 1; }
__device__ __forceinline__ const TileDesc *slot3(const unsigned char *tiles, uint32_t n)
{
    return reinterpret_cast<const TileDesc *>(tiles + (n & (S3_SLOTS - 1)) * S3_SLOT_BYTES);
}
__device__ __forceinline__ uint4 lds128u(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128u(uint32_t addr, uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ uint32_t word_of(const uint4 &v, int w)
{
    return w == 0 ? v.x : (w == 1 ? v.y : (w == 2 ? v.z : v.w));
}

// ---------------------------------------------------------------- stager side
struct Slab {
    uint4 v[SCAN_G];            // code c of the tile's 8 queries: 8 rotated sub-space entries each
};
// Unused query slots of a tile (g >= ng) load query slot 0's entries again: an L1 hit, no branch, and sums that
// nobody reads but that still fit their 16-bit lane.
__device__ __forceinline__ void slab_load(Slab &s, const ScanArgs &a, const TileDesc *T, uint32_t ch, uint32_t c)
{
    const int ng = (int)T->ng;
    const uint32_t q0 = T->q[0];
#pragma unroll
    for (int g = 0; g < SCAN_G; g++) {
        const uint32_t q = g < ng ? T->q[g] : q0;
        s.v[g] = __ldg(a.qt + ((size_t)q * a.nch + ch) * 256 + c);
    }
}
// unit j of code c = sub-space (j + c) & 7: (query 0..7) x u16, written to [c][(j + c) & 7]
__device__ __forceinline__ void slab_store(const Slab &s, uint32_t buf_addr, uint32_t c)
{
    const uint32_t row = buf_addr + (c << 7);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int w = j >> 1;
        const uint32_t sel = (j & 1) ? 0x7632u : 0x5410u;
        uint4 o;
        o.x = __byte_perm(word_of(s.v[0], w), word_of(s.v[1], w), sel);
        o.y = __byte_perm(word_of(s.v[2], w), word_of(s.v[3], w), sel);
        o.z = __byte_perm(word_of(s.v[4], w), word_of(s.v[5], w), sel);
        o.w = __byte_perm(word_of(s.v[6], w), word_of(s.v[7], w), sel);
        sts128u(row + ((((uint32_t)j + c) & 7u) << 4), o);
    }
}

__device__ __forceinline__ void stager_loop(const ScanArgs &a, uint32_t total, int tid)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *const tiles = smem + S3_TILES;
    const uint32_t lut = (uint32_t)__cvta_generic_to_shared(smem);
    const int lane = tid & 31, pw = tid >> 5;
    const uint32_t nch = a.nch, c = (uint32_t)tid;

    // One slab in registers.  The loads of the next data stage are issued right after this stage's slab has been
    // written to shared memory, i.e. a whole scanner stage before they are needed: they land while the stagers
    // wait for the ring buffer to come free.
    Slab cur;
    {
        const TileDesc *T0 = slot3(tiles, 0);
        if (T0->ng) slab_load(cur, a, T0, 0, c);
    }
    int b = 0;
    uint32_t gs = 0;
    for (uint32_t n = 0;; n++) {
        const TileDesc *T = slot3(tiles, n);
        if (T->ng == 0) break;
        const TileDesc *Tn = slot3(tiles, n + 1);
        const bool next_tile = Tn->ng != 0;
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
            if (gs >= 2) bar_sync(BAR_EMPTY + b, S3_NT);           // scanners are done with stage gs-2
            if (ch == nch) {                                       // all-zero code-0 row for the lagging lanes
                if (tid < 32) reinterpret_cast<uint32_t *>(smem + b * S3_BUF)[tid] = 0u;
            } else {
                slab_store(cur, lut + (uint32_t)b * S3_BUF, c);
                // the next data stage: the next chunk of this tile, or chunk 0 of the next tile (which then
                // rides through the zero stage)
                if (ch + 1 < nch) slab_load(cur, a, T, ch + 1, c);
                else if (next_tile) slab_load(cur, a, Tn, 0, c);
            }
            if (pw == 0 && ch == 1 && lane < (int)(sizeof(TileDesc) / 4))   // publish tile n+2 before FULL(stage 1)
                reinterpret_cast<uint32_t *>(const_cast<TileDesc *>(slot3(tiles, n + 2)))[lane] = t_word;
#if LGPU_S3_NAMED_FULL
            bar_arrive(BAR_FULL + b, S3_NT);
#else
            __syncwarp();
            if (lane == 0) mbar_arrive(lut + (uint32_t)S3_MBAR_OFF + 8u * (uint32_t)b);
#endif
            bar_sync(BAR_PROD, S3_PT);
            b = ring_next3(b);
            gs++;
        }
    }
}

// ---------------------------------------------------------------- scanner side
// ---- tau_q from the list itself.  Tile-local bisection cannot get below the k-th smallest of ONE tile (the
// 100 k / rows_tile quantile); the list holds every row seen so far that was under the threshold of its time, so its
// k-th smallest key is the k-th smallest of everything scanned for the query.  Any k keys of the list give a valid tau
// (records still in flight read as 0xffffffff and only make the bound looser).  Triggered each time the list grew by
// k since the last time, i.e. about once per doubling of the rows seen.  Out of line: its S3_LIST_PER key registers
// must not take part in the register allocation of the gather loop.
__device__ __noinline__ uint32_t tighten_from_list(const uint32_t *keys, uint32_t *thr_q, uint32_t *last_q,
                                                   volatile uint32_t *sh, uint32_t ln, uint32_t tkey, uint32_t k, int ct)
{
    const int lane = ct & 31;
    uint32_t lk[S3_LIST_PER];
    uint32_t mn = 0xffffffffu, c0 = 0;
#pragma unroll
    for (int j = 0; j < S3_LIST_PER; j++) {
        const uint32_t i = (uint32_t)j * S3_CT + ct;
        lk[j] = i < ln ? __ldcg(keys + i) : 0xffffffffu;
    }
#pragma unroll
    for (int j = 0; j < S3_LIST_PER; j++) { mn = min(mn, lk[j]); c0 += lk[j] <= tkey ? 1u : 0u; }
    mn = __reduce_min_sync(0xffffffffu, mn); c0 = __reduce_add_sync(0xffffffffu, c0);
    if (lane == 0) { atomicMin(const_cast<uint32_t *>(sh + 15), mn); if (c0) atomicAdd(const_cast<uint32_t *>(sh + 16), c0); }
    bar_sync(BAR_SCAN, S3_CT);
    if (sh[16] >= k) {                          // invariant: count(list key <= hi) >= k
        float lo = key_f32(sh[15]), hi = key_f32(tkey);
#pragma unroll 1
        for (int it = 0; it < S3_LIST_STEPS; it++) {
            const uint32_t mid = f32_key(0.5f * lo + 0.5f * hi);
            uint32_t c = 0;
#pragma unroll
            for (int j = 0; j < S3_LIST_PER; j++) c += lk[j] <= mid ? 1u : 0u;
            c = __reduce_add_sync(0xffffffffu, c);
            if (lane == 0 && c) atomicAdd(const_cast<uint32_t *>(sh + 17 + it), c);
            bar_sync(BAR_SCAN, S3_CT);
            if (sh[17 + it] >= k) hi = key_f32(mid); else lo = key_f32(mid);
        }
        const uint32_t nk = f32_key(hi);
        if (nk < tkey) {
            if (ct == 0) atomicMin(thr_q, nk);
            tkey = nk;
        }
    }
    if (ct == 0) *last_q = ln;
    return tkey;
}

template <int R, bool LIST>
__device__ __forceinline__ int scan_tile(const ScanArgs &a, const TileDesc *T, bool next_exists, int b, int ct, uint32_t &ph)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t lut = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t nch = a.nch;
    const uint32_t p = T->p, row0 = T->row0, nrows = T->nrows;
    const int ng = (int)T->ng;
    const int sig = ct & 7;                               // this lane's skew (== row % 8)
    const uint32_t n_p = T->n_p, npad = T->npad;                                    // (copied into the descriptor)
    const uint2 *cs = reinterpret_cast<const uint2 *>(a.codes + ((uint64_t)T->code_base8 << 3));   // [nch+1][npad]

    uint32_t acc[R][4];
    bool valid[R];
    uint2 wn[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
#pragma unroll
        for (int g = 0; g < 4; g++) acc[r][g] = 0u;
        const uint32_t row = row0 + ct + r * S3_CT;
        valid[r] = row < row0 + nrows && row < n_p;
        wn[r] = valid[r] ? __ldg(cs + row) : make_uint2(0u, 0u);
    }

    for (uint32_t it = 0; it <= nch; it++) {
        uint2 w[R];
#pragma unroll
        for (int r = 0; r < R; r++) w[r] = wn[r];
        if (it < nch) {                                    // prefetch the next block of code bytes
#pragma unroll
            for (int r = 0; r < R; r++) {
                const uint32_t row = row0 + ct + r * S3_CT;
                wn[r] = valid[r] ? __ldg(cs + (size_t)(it + 1) * npad + row) : make_uint2(0u, 0u);
            }
        }
#if LGPU_S3_NAMED_FULL
        bar_sync(BAR_FULL + b, S3_NT);
#else
        mbar_wait(lut + (uint32_t)S3_MBAR_OFF + 8u * (uint32_t)b, (ph >> b) & 1u);
        ph ^= 1u << b;
#endif
        const int bp = b == 0 ? 2 : b - 1;                 // buffer of the previous stage
        const uint32_t base_cur = lut + (uint32_t)b * S3_BUF;
        const uint32_t base_prev = lut + (uint32_t)bp * S3_BUF;
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const uint32_t off = ((e < sig) ? base_prev : base_cur) + (uint32_t)(((e - sig) & 7) << 4);
#pragma unroll
            for (int r = 0; r < R; r++) {
                const uint32_t word = (e < 4) ? w[r].x : w[r].y;
                const uint32_t code = (word >> (8 * (e & 3))) & 0xffu;
                const uint4 v = lds128u(off + (code << 7));
                acc[r][0] += v.x; acc[r][1] += v.y; acc[r][2] += v.z; acc[r][3] += v.w;
            }
        }
        if (it + 2 <= nch || next_exists) bar_arrive(BAR_EMPTY + bp, S3_NT);
        b = ring_next3(b);
    }

    // ---- epilogue: lower bound L = step_q * sum + (base_q + A(q,p)) + R(row) per (row, query) ----
    const float scale = a.metric == LGPU_COSINE ? 0.5f : 1.0f;
    const uint64_t pos0 = T->part_off32;
    float rr[R];
#pragma unroll
    for (int r = 0; r < R; r++)
        rr[r] = (valid[r] && a.row_R) ? __ldg(a.row_R + pos0 + row0 + ct + r * S3_CT) : 0.f;
    if (a.cand == nullptr) {
        // dense mode: one f32 per (row, query) to HBM; the caller selects a shortlist from them
#pragma unroll
        for (int g = 0; g < SCAN_G; g++) {
            if (g < ng) {
                const uint32_t q = T->q[g];
                const float step = __ldg(a.qt_step + q);
                const float cst = __ldg(a.qt_base + q) + (a.probe_A ? __ldg(a.probe_A + T->slot[g]) : 0.f);
                float *out = a.dist_out + T->out[g];
#pragma unroll
                for (int r = 0; r < R; r++) {
                    if (valid[r]) {
                        const uint32_t s = (g & 1) ? (acc[r][g >> 1] >> 16) : (acc[r][g >> 1] & 0xffffu);
                        out[row0 + ct + r * S3_CT] = (fmaf(step, (float)s, cst) + rr[r]) * scale;
                    }
                }
            }
        }
        return b;
    }
    // candidate mode.  tau_q (global, atomicMin) is any value such that at least k rows of the query have L <= tau_q:
    // then the k-th smallest exact distance is <= tau_q + W + E and every row of the exact top-k has
    // L <= tau_q + W + 2E = tau_q + slack_q.  The CTA's 256 scanner threads tighten tau_q from the tile's own rows (an
    // upper bound of their k-th smallest L, by 8 counting bisections through shared counters) when the query has no
    // threshold yet or when this is one of its three nearest partitions -- that is where the small distances are;
    // every warp then appends the rows under the threshold.
    const int lane = ct & 31;
    const uint32_t k = a.topk;
    // The queries' scalars (step, base + A, slack) are loaded here for all of the tile's queries at once, beside the
    // row terms above, and read back from shared memory after each query's first barrier.  The epilogue runs its queries
    // one after the other behind scanner barriers, so a load inside the query loop would add one L2 round trip per
    // query that every scanner warp waits for, after the one for the threshold.  The slots are rewritten by the next tile's
    // epilogue only: every read of query g is before the second barrier of iteration g, and no thread passes the
    // last such barrier before all have read.
    float *const qsc = reinterpret_cast<float *>(smem + S3_QS_OFF);
    if (ct >= 32 && ct < 32 + ng) {
        const int g = ct - 32;
        const uint32_t q = T->q[g];
        qsc[4 * g + 0] = __ldg(a.qt_step + q);
        qsc[4 * g + 1] = __ldg(a.qt_base + q) + (a.probe_A ? __ldg(a.probe_A + T->slot[g]) : 0.f);
        qsc[4 * g + 2] = __ldg(a.slack + q);
    }
    // scratch, two banks alternating by query so that the reset for query g+1 cannot overtake a slow warp still
    // reading query g's counters: [0] threshold key, [1] min key, [2] max key, [3] valid rows, [4..12] counters of the
    // tile bisection; [13] list length, [14] list length at the last list tightening, [15] smallest list key,
    // [16..16+S3_LIST_STEPS] counters of the list bisection
#pragma unroll 1
    for (int g = 0; g < ng; g++) {
        volatile uint32_t *const sh =
            reinterpret_cast<volatile uint32_t *>(smem + S3_TILES + S3_SLOTS * S3_SLOT_BYTES) + (g & 1) * S3_SCR;
        const uint32_t q = T->q[g], slot = T->slot[g];
        if (ct < S3_SCR) {
            uint32_t v = 0u;
            if (ct == 0) v = __ldcg(a.thr + q);
            else if (ct == 1 || ct == 15) v = 0xffffffffu;
            else if (ct == 13) v = min(__ldcg(a.cand_cnt + q), a.cand_cap);
            else if (ct == 14) v = __ldcg(a.cand_last + q);
            sh[ct] = v;
        }
        bar_sync(BAR_SCAN, S3_CT);
        uint32_t tkey = sh[0];
        // ---- tau_q from the list itself.  Tile-local bisection cannot get below the k-th smallest of ONE tile (the
        // 100 k / rows_tile quantile); the list holds every row seen so far that was under the threshold of its time,
        // so its k-th smallest key is the k-th smallest of everything scanned for the query.  Any k keys of the list
        // give a valid tau (records still in flight read as 0xffffffff and only make the bound looser).  Triggered
        // each time the list grew by k since the last time, i.e. about once per doubling of the rows seen.
        if (LIST) {
            const uint32_t ln = sh[13], last = sh[14];
            if (tkey != CAND_NO_THR && ln >= 2u * k && ln >= last + k)
                tkey = tighten_from_list(a.cand_key + (size_t)q * a.cand_cap, a.thr + q, a.cand_last + q, sh, ln, tkey, k, ct);
        }
        const float step = qsc[4 * g + 0], cst = qsc[4 * g + 1], slack = qsc[4 * g + 2];
        float L[R];
        uint32_t nvalid = 0, kmin = 0xffffffffu, kmax = 0u;
#pragma unroll
        for (int r = 0; r < R; r++) {
            const uint32_t w = (g & 2) ? ((g & 4) ? acc[r][3] : acc[r][1]) : ((g & 4) ? acc[r][2] : acc[r][0]);
            const uint32_t s = (g & 1) ? (w >> 16) : (w & 0xffffu);
            L[r] = valid[r] ? (fmaf(step, (float)s, cst) + rr[r]) * scale : CUDART_INF_F;
            if (valid[r]) { const uint32_t kk = f32_key(L[r]); kmin = min(kmin, kk); kmax = max(kmax, kk); nvalid++; }
        }

        const uint32_t rank = slot - q * a.nprobes;
        // Tighten tau_q from this tile when it pays: always for a query without a threshold and for its three nearest
        // partitions (that is where the small distances are); otherwise only when this tile alone holds 2k or more
        // rows under the current threshold (one counting pass decides) -- without that a loose early threshold, set
        // by whichever far partition happened to finish first, would let whole near partitions through.
        bool bisect = tkey == CAND_NO_THR || rank < 3u;
        float cur = tkey == CAND_NO_THR ? CUDART_INF_F : key_f32(tkey);
        kmin = __reduce_min_sync(0xffffffffu, kmin); kmax = __reduce_max_sync(0xffffffffu, kmax);
        nvalid = __reduce_add_sync(0xffffffffu, nvalid);
        uint32_t cunder = 0;
        if (tkey != CAND_NO_THR) {
#pragma unroll
            for (int r = 0; r < R; r++) cunder += L[r] <= cur ? 1u : 0u;
            cunder = __reduce_add_sync(0xffffffffu, cunder);
        }
        if (lane == 0) {
            atomicMin(const_cast<uint32_t *>(sh + 1), kmin); atomicMax(const_cast<uint32_t *>(sh + 2), kmax);
            atomicAdd(const_cast<uint32_t *>(sh + 3), nvalid);
            if (cunder) atomicAdd(const_cast<uint32_t *>(sh + 4), cunder);
        }
        bar_sync(BAR_SCAN, S3_CT);
        {
            float lo = key_f32(sh[1]), hi = key_f32(sh[2]);
            const uint32_t under = sh[4];                    // rows of this tile with L <= current threshold
            if (tkey != CAND_NO_THR) { bisect = bisect ? under >= k : under >= 2u * k; if (cur < hi) hi = cur; }
            if (bisect && sh[3] >= k && hi < CUDART_INF_F && lo == lo && hi == hi) {
                // invariant: count(L <= hi) >= k
#pragma unroll 1
                for (int it = 0; it < 8; it++) {
                    const float mid = 0.5f * lo + 0.5f * hi;
                    uint32_t c = 0;
#pragma unroll
                    for (int r = 0; r < R; r++) c += L[r] <= mid ? 1u : 0u;
                    c = __reduce_add_sync(0xffffffffu, c);
                    if (lane == 0 && c) atomicAdd(const_cast<uint32_t *>(sh + 5 + it), c);
                    bar_sync(BAR_SCAN, S3_CT);
                    if (sh[5 + it] >= k) hi = mid; else lo = mid;
                }
                const uint32_t nk = f32_key(hi);
                if (nk < tkey) {
                    if (ct == 0) atomicMin(a.thr + q, nk);
                    tkey = nk;
                }
            }
        }
        const float lim = tkey == CAND_NO_THR ? CUDART_INF_F : key_f32(tkey) + slack;
        uint32_t npass = 0;
#pragma unroll
        for (int r = 0; r < R; r++) npass += (valid[r] && L[r] <= lim) ? 1u : 0u;
        const uint32_t wpass = __reduce_add_sync(0xffffffffu, npass);
        if (wpass) {
            uint32_t pre = npass;                          // inclusive scan over lanes
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, pre, o);
                if (lane >= o) pre += t;
            }
            uint32_t base = 0;
            if (lane == 31) base = atomicAdd(a.cand_cnt + q, wpass);
            base = __shfl_sync(0xffffffffu, base, 31);
            uint32_t at = base + pre - npass;
            CandRec *dst = a.cand + (size_t)q * a.cand_cap;
            uint32_t *dkey = a.cand_key + (size_t)q * a.cand_cap;
#pragma unroll
            for (int r = 0; r < R; r++) {
                if (valid[r] && L[r] <= lim) {
                    if (at < a.cand_cap) {
                        CandRec rec; rec.lb = L[r]; rec.p = p; rec.row = row0 + ct + r * S3_CT; rec.pad = 0u;
                        dst[at] = rec;
                        dkey[at] = f32_key(L[r]);
                    }
                    at++;
                }
            }
        }
    }
    return b;
}

template <bool LIST>
__device__ __forceinline__ void scanner_loop(const ScanArgs &a, int tid)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const unsigned char *const tiles = smem + S3_TILES;
    const int ct = tid - S3_PT;
    int b = 0;
    uint32_t ph = 0u;                                   // bit b: parity of ring buffer b's next FULL phase
    for (uint32_t n = 0;; n++) {
        const TileDesc *T = slot3(tiles, n);
        if (T->ng == 0) break;
        const bool next_exists = slot3(tiles, n + 1)->ng != 0;
        const int R = (int)((T->nrows + S3_CT - 1) / S3_CT);
#define LGPU_SCAN3(RR) b = scan_tile<RR, LIST>(a, T, next_exists, b, ct, ph)
        if (R <= 2) LGPU_SCAN3(2);
        else if (R <= 4) LGPU_SCAN3(4);
        else LGPU_SCAN3(6);
#undef LGPU_SCAN3
    }
}

// LIST: the scanners also tighten tau_q from the query's own candidate list (k > 32: tile-local thresholds alone would
// overflow the lists).  A separate instantiation, so that the list keys held in registers there do not cost the
// k <= 32 kernel (BASELINE config 2) spills inside its gather loop.
template <bool LIST>
__global__ void __launch_bounds__(S3_NT, 2) scan3_kernel(ScanArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x;
    const uint32_t total = *a.total_tiles;
    unsigned char *const tiles = smem + S3_TILES;

    // "stage -1" of the first tile: zero code-0 row in ring buffer 2
    if (tid < 32) reinterpret_cast<uint32_t *>(smem + 2 * S3_BUF)[tid] = 0u;
#if !LGPU_S3_NAMED_FULL
    if (tid == 0) {
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(smem) + (uint32_t)S3_MBAR_OFF;
        for (int i = 0; i < 3; i++) mbar_init(mb + 8u * i, S3_PW);      // one arrival per stager warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#endif
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
            reinterpret_cast<uint32_t *>(tiles + S3_SLOT_BYTES)[tid] = w1;
        }
    }
    __syncthreads();
    if (tid < S3_PT) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(S3_PREG));
        stager_loop(a, total, tid);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(S3_CREG));
        scanner_loop<LIST>(a, tid);
    }
}

}  // namespace

void launch_scan3(const ScanArgs &a, int grid, cudaStream_t st)
{
    if (!a.qt || !a.qt_step || !a.qt_base || !a.tile_desc || a.rows_tile != SCAN3_ROWS_TILE || !a.part_off ||
        (a.cand && (!a.thr || !a.slack || !a.cand_cnt || !a.cand_key || !a.cand_last || a.cand_cap > CAND_CAP_MAX || a.topk < 1 || a.topk > CAND_TOPK_MAX || a.nprobes < 1))) {
        set_error("internal: the filter scan needs query tables and tile descriptors built with rows_tile 1536");
        throw Failure{LGPU_RUNTIME};
    }
    const bool list = a.cand && a.topk > 32;
    auto kern = list ? scan3_kernel<true> : scan3_kernel<false>;
    LGPU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S3_SMEM));
    launch_k(kern, dim3(2 * grid), dim3(S3_NT), S3_SMEM, st, a); LGPU_COUNT_LAUNCH();   // two CTAs per SM
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
