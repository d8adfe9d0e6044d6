// select_large.cu -- K4 for SELECT_KMAX < k <= LGPU_K_MAX: per-query top-k by (_distance ASC, _rowid ASC) with no
// shared-memory bound on k (refine pools, deep pagination, range queries with a large limit).
//
// The small selects (select.cu) stage each query's survivors in one CTA's shared memory, which caps k at 2048.  Here
// every stage works from global memory and one query's candidates are spread over many CTAs (grid: slices x queries),
// so a single query over 10M rows still runs on every SM:
//   1. radix select of the k-th ordered key t (f32_key of the distance) in three histogram passes of 11 / 11 / 10
//      bits; each pass's CTAs build a shared-memory histogram of their slice (keys matching the prefix found so far)
//      and add it to the query's global one, and a one-CTA-per-query walk fixes the next digit;
//   2. ties: when more rows than still needed have key t, a radix select over the ids of just those rows (relative to
//      their minimum, 11 bits per pass) gives an id bound u.  Exactly min(k, valid) rows satisfy key < t or
//      (key == t and id <= u), whatever the tie counts (Hamming and 4-bit PQ distances tie in long runs);
//   3. those rows are appended to a [k] buffer per query; a query with at most k valid rows skips 1-2;
//   4. segmented sort by (key, id): bitonic sort of LS_CHUNK-entry chunks in shared memory, merge-path merges of runs
//      in global memory, then the outputs (ids, distances, positions, counts; unused slots UINT64_MAX / +inf).
// Every pass reads its candidates and applies the row filter (NaN dropped, -0 folded into +0, [lower, upper),
// allow-list) through one function, for_each_candidate, so the passes agree on the candidate set by construction.
// A walk that finds the digit's bin holding exactly the rows still needed finishes early, and each pass's CTAs return
// at once for a query that is done, so the id passes cost a launch when there are no ties to break.
#include "kernels.cuh"

#include <cooperative_groups.h>
#include <math_constants.h>

#include <algorithm>

namespace cg = cooperative_groups;

namespace lgpu {

namespace {

constexpr int LS_THREADS = 256;
constexpr uint32_t LS_BINS = 2048;            // 11-bit digits
constexpr uint32_t LS_CHUNK = 2048;           // entries one CTA sorts in shared memory
constexpr int LS_MERGE_ITEMS = 8;             // outputs per thread of a merge pass
constexpr int LS_ID_PASSES = 6;               // ceil(64 / 11): digits of a 64-bit id range

enum LkPhase : uint32_t { LK_KEY0 = 0, LK_KEY1 = 1, LK_KEY2 = 2, LK_RANGE = 3, LK_ID = 4, LK_DONE = 5 };

// one query's radix walk
struct alignas(16) LkState {
    uint32_t phase;           // LkPhase: the pass the query waits for
    uint32_t r;               // rows still to take among those matching the prefix
    uint32_t t;               // key prefix; final: the k-th key
    uint32_t cnt;             // rows appended by the compaction
    uint64_t idlo, idhi;      // min / max id of the rows with key t
    uint64_t pre;             // id digits fixed so far, relative to idlo
    uint64_t u;               // final: the id bound
    uint32_t shift, width;    // the next id digit: bits [shift, shift + width) of id - idlo
    uint32_t pad[2];
};

// scratch layout (select_large_scratch_bytes): state [B], hist [B][LS_BINS], then two sort buffers of [B][k] keys,
// ids and (with out_pos) positions
struct LkBuf {
    uint32_t *key;
    uint64_t *id;
    uint64_t *pos;
};
struct LkScratch {
    LkState *state;
    uint32_t *hist;
    LkBuf buf[2];
};

__host__ __device__ inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

LkScratch carve(void *p, uint32_t B, uint32_t k, bool pos)
{
    char *c = static_cast<char *>(p);
    LkScratch s{};
    s.state = reinterpret_cast<LkState *>(c); c += align256((size_t)B * sizeof(LkState));
    s.hist = reinterpret_cast<uint32_t *>(c); c += align256((size_t)B * LS_BINS * 4);
    for (int i = 0; i < 2; i++) {
        s.buf[i].key = reinterpret_cast<uint32_t *>(c); c += align256((size_t)B * k * 4);
        s.buf[i].id = reinterpret_cast<uint64_t *>(c); c += align256((size_t)B * k * 8);
        s.buf[i].pos = pos ? reinterpret_cast<uint64_t *>(c) : nullptr; c += pos ? align256((size_t)B * k * 8) : 0;
    }
    return s;
}

__device__ __forceinline__ bool skip_query(const SelectArgs &a, uint32_t q)
{
    return (a.gate && *a.gate == 0) || (a.only && !a.only[q]);
}

// Calls f(key, id, pos) for every candidate of query q in this CTA's slice that passes the row filter: not NaN, inside
// [lower, upper), an allowed id; -0 folded into +0 before the key is taken.  NEED: 0 = key only (ids are still read
// under an allow-list), 1 = key and id, 2 = key, id and position.  The slice is every nslices-th block of LS_THREADS
// consecutive candidates, so a warp's loads stay coalesced.
template <int NEED, class F>
__device__ __forceinline__ void for_each_candidate(const SelectArgs &a, uint32_t q, uint32_t slice, uint32_t nslices,
                                                   F &&f)
{
    const bool need_id = NEED >= 1 || a.allow;
    auto offer = [&](float v, uint64_t id_or_idx, const uint64_t *idsrc, uint64_t pos, bool id_given) {
        if (v == 0.f) v = 0.f;                                   // -0 and +0 tie
        if (v != v) return;                                      // FilterExec: _distance IS NOT NULL
        if (a.has_lower && !(v >= a.lower)) return;
        if (a.has_upper && !(v < a.upper)) return;
        uint64_t id = id_or_idx;
        if (need_id && !id_given && idsrc) id = idsrc[id_or_idx];
        if (a.allow && !(id < a.allow_bits && ((a.allow[id >> 5] >> (id & 31)) & 1u))) return;
        f(f32_key(v), id, pos);
    };
    const uint64_t first = (uint64_t)slice * LS_THREADS + threadIdx.x, step = (uint64_t)nslices * LS_THREADS;
    if (a.mode == 0) {
        for (uint32_t j = 0; j < a.nprobes; j++) {
            const uint32_t slot = q * a.nprobes + j;
            const uint64_t pp = a.probes[slot];
            if (pp >= a.nlist) continue;                         // unused probe slot
            const uint32_t p = (uint32_t)pp;
            const uint32_t n = a.part_n[p];
            const float *src = a.dist + a.seg_off[slot];
            const uint64_t rowbase = a.part_off[p];
            for (uint64_t r = first; r < n; r += step) offer(src[r], rowbase + r, a.row_ids, rowbase + r, false);
        }
    } else if (a.mode == 1) {
        const float *src = a.dense + (size_t)q * a.row_stride;
        for (uint64_t c = first; c < a.ncols; c += step) offer(src[c], a.col_ids ? c : a.col_base + c, a.col_ids, c, false);
    } else {
        const uint64_t ncols = a.ncols_q ? min((uint64_t)a.ncols_q[q], a.ncols) : a.ncols;
        for (uint64_t c = first; c < ncols; c += step) {
            if (a.list_cnt && c % a.inner >= a.list_cnt[c / a.inner * a.B + q]) continue;
            const uint64_t addr = (c / a.inner) * a.outer_stride + (uint64_t)q * a.row_stride + c % a.inner;
            uint64_t id;
            float v;
            if (a.cand_rec) { const TopkRecord r = a.cand_rec[addr]; id = r.id; v = r.dist; }
            else { id = a.cand_ids[addr]; v = a.dense[addr]; }
            if (id == UINT64_MAX) continue;                      // unused slot of a shorter list
            const uint64_t pos = NEED >= 2 ? (a.cand_pos ? a.cand_pos[addr] : c) : 0;
            offer(v, id, nullptr, pos, true);
        }
    }
}

__device__ __forceinline__ uint32_t key_digit_shift(uint32_t phase)
{
    return phase == LK_KEY0 ? 21 : (phase == LK_KEY1 ? 10 : 0);
}
__device__ __forceinline__ uint32_t key_digit_width(uint32_t phase) { return phase == LK_KEY2 ? 10 : 11; }

__global__ void lk_init_kernel(LkState *state, uint32_t B, uint32_t k)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    LkState s{};
    s.phase = LK_KEY0; s.r = k; s.t = 0; s.cnt = 0;
    s.idlo = UINT64_MAX; s.idhi = 0; s.pre = 0; s.u = UINT64_MAX;
    state[q] = s;
}

// one histogram pass: phase LK_KEY0..2 (digit of the key), LK_RANGE (min / max id of the rows with key t) or LK_ID
// (digit of id - idlo among the rows with key t).  Grid (nslices, B).
__global__ void __launch_bounds__(LS_THREADS) lk_hist_kernel(SelectArgs a, LkState *state, uint32_t *hist,
                                                            uint32_t phase, uint32_t q0)
{
    __shared__ uint32_t h[LS_BINS];
    __shared__ unsigned long long s_lo, s_hi;
    const uint32_t q = q0 + blockIdx.y;
    if (skip_query(a, q)) return;
    const LkState s = state[q];
    if (s.phase != phase) return;
    const uint32_t slice = blockIdx.x, nslices = gridDim.x;
    if (phase == LK_RANGE) {
        if (threadIdx.x == 0) { s_lo = UINT64_MAX; s_hi = 0; }
        __syncthreads();
        uint64_t lo = UINT64_MAX, hi = 0;
        for_each_candidate<1>(a, q, slice, nslices, [&](uint32_t key, uint64_t id, uint64_t) {
            if (key == s.t) { lo = min(lo, id); hi = max(hi, id); }
        });
        for (int o = 16; o > 0; o >>= 1) {
            lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(&s_lo, lo); atomicMax(&s_hi, hi); }
        __syncthreads();
        if (threadIdx.x == 0 && s_lo <= s_hi) {
            atomicMin(reinterpret_cast<unsigned long long *>(&state[q].idlo), s_lo);
            atomicMax(reinterpret_cast<unsigned long long *>(&state[q].idhi), s_hi);
        }
        return;
    }
    for (uint32_t i = threadIdx.x; i < LS_BINS; i += LS_THREADS) h[i] = 0;
    __syncthreads();
    if (phase == LK_ID) {
        const uint32_t top = s.shift + s.width;               // <= 64
        const uint32_t mask = (1u << s.width) - 1u;
        for_each_candidate<1>(a, q, slice, nslices, [&](uint32_t key, uint64_t id, uint64_t) {
            if (key != s.t) return;
            const uint64_t v = id - s.idlo;
            if (top < 64 && (v >> top) != (s.pre >> top)) return;
            atomicAdd(&h[(uint32_t)(v >> s.shift) & mask], 1u);
        });
    } else {
        const uint32_t shift = key_digit_shift(phase), top = shift + key_digit_width(phase);
        const uint32_t mask = (1u << key_digit_width(phase)) - 1u;
        for_each_candidate<0>(a, q, slice, nslices, [&](uint32_t key, uint64_t, uint64_t) {
            if (top < 32 && (key >> top) != (s.t >> top)) return;
            atomicAdd(&h[(key >> shift) & mask], 1u);
        });
    }
    __syncthreads();
    uint32_t *g = hist + (size_t)q * LS_BINS;
    for (uint32_t i = threadIdx.x; i < LS_BINS; i += LS_THREADS)
        if (h[i]) atomicAdd(&g[i], h[i]);
}

// the walk after a histogram pass, one CTA per query: the digit d whose bin holds the r-th row of the prefix, then
// the next phase.  Clears the histogram for the next pass.
__global__ void __launch_bounds__(LS_THREADS) lk_walk_kernel(SelectArgs a, LkState *state, uint32_t *hist,
                                                            uint32_t phase, uint32_t q0)
{
    constexpr int PER = LS_BINS / LS_THREADS;
    __shared__ uint32_t s_warp[LS_THREADS / 32];
    __shared__ uint32_t s_total;
    const uint32_t q = q0 + blockIdx.x;
    if (skip_query(a, q)) return;
    LkState *sp = state + q;
    // every thread reads phase and r before the first barrier; the one that finds the digit updates them after it
    const uint32_t ph = sp->phase, r = sp->r;
    if (ph != phase) return;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (phase == LK_RANGE) {
        if (tid == 0) {
            const uint64_t span = sp->idhi - sp->idlo;
            if (span == 0) { sp->u = sp->idlo; sp->phase = LK_DONE; }     // every tie has the same id
            else {
                const uint32_t nbits = 64 - __clzll((long long)span);
                sp->width = min(nbits, 11u); sp->shift = nbits - sp->width; sp->pre = 0; sp->phase = LK_ID;
            }
        }
        return;
    }
    uint32_t *g = hist + (size_t)q * LS_BINS;
    uint32_t v[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; i++) { v[i] = g[tid * PER + i]; sum += v[i]; }
    // exclusive prefix sum of the per-thread sums
    uint32_t incl = sum;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (int i = 0; i < w; i++) wbase += s_warp[i];
    if (tid == LS_THREADS - 1) s_total = wbase + incl;
    const uint32_t below0 = wbase + incl - sum;
    __syncthreads();
    const uint32_t total = s_total;
    if (phase == LK_KEY0 && total <= r) {                       // at most k valid rows: take them all
        if (tid == 0) { sp->t = 0xffffffffu; sp->u = UINT64_MAX; sp->phase = LK_DONE; }
    } else if (below0 < r && r <= below0 + sum) {               // this thread's bins hold the r-th row
        uint32_t below = below0, hd = 0;
        int sel = -1;
#pragma unroll
        for (int i = 0; i < PER; i++) {                         // (unrolled: v stays in registers)
            if (sel >= 0) continue;
            if (below + v[i] >= r) { sel = i; hd = v[i]; }
            else below += v[i];
        }
        const uint32_t d = tid * PER + sel, rr = r - below;
        if (phase == LK_ID) {
            uint64_t pre = sp->pre | ((uint64_t)d << sp->shift);
            if (hd == rr || sp->shift == 0) {                   // (at shift 0, hd > rr only for repeated ids)
                if (hd == rr) pre |= ((uint64_t)1 << sp->shift) - 1;
                sp->u = sp->idlo + pre; sp->phase = LK_DONE;
            } else {
                const uint32_t nw = min(sp->shift, 11u);
                sp->pre = pre; sp->shift -= nw; sp->width = nw;
            }
        } else {
            const uint32_t shift = key_digit_shift(phase);
            uint32_t t = sp->t | (d << shift);
            if (hd == rr) {                                     // every row of this digit is in: no tie to break
                t |= (1u << shift) - 1u;
                sp->u = UINT64_MAX; sp->phase = LK_DONE;
            } else {
                sp->phase = phase == LK_KEY2 ? (uint32_t)LK_RANGE : phase + 1;
            }
            sp->t = t;
        }
        sp->r = rr;
    }
#pragma unroll
    for (int i = 0; i < PER; i++) g[tid * PER + i] = 0;
}

// the rows with key < t or (key == t and id <= u), appended to the query's buffer (at most k of them)
template <bool POS>
__global__ void __launch_bounds__(LS_THREADS) lk_compact_kernel(SelectArgs a, LkState *state, LkBuf out, uint32_t q0)
{
    const uint32_t q = q0 + blockIdx.y;
    if (skip_query(a, q)) return;
    const uint32_t t = state[q].t;
    const uint64_t u = state[q].u;
    uint32_t *cnt = &state[q].cnt;
    const size_t base = (size_t)q * a.k;
    for_each_candidate<POS ? 2 : 1>(a, q, blockIdx.x, gridDim.x, [&](uint32_t key, uint64_t id, uint64_t pos) {
        if (!(key < t || (key == t && id <= u))) return;
        cg::coalesced_group g = cg::coalesced_threads();
        uint32_t slot = 0;
        if (g.thread_rank() == 0) slot = atomicAdd(cnt, g.size());
        slot = g.shfl(slot, 0) + g.thread_rank();
        if (slot < a.k) {                                       // (more than k only with repeated (key, id) pairs)
            out.key[base + slot] = key; out.id[base + slot] = id;
            if (POS) out.pos[base + slot] = pos;
        }
    });
}

__device__ __forceinline__ bool lk_less(uint32_t ka, uint64_t ia, uint32_t kb, uint64_t ib)
{
    return ka < kb || (ka == kb && ia < ib);
}
__device__ __forceinline__ uint32_t lk_count(const SelectArgs &a, const LkState *state, uint32_t q)
{
    return min(state[q].cnt, a.k);
}

// bitonic sort of chunk blockIdx.x (LS_CHUNK entries) of each query's buffer, in place.  Grid (chunks, B).
template <bool POS>
__global__ void __launch_bounds__(LS_THREADS) lk_chunk_sort_kernel(SelectArgs a, const LkState *state, LkBuf buf,
                                                                  uint32_t q0)
{
    __shared__ uint32_t sk[LS_CHUNK];
    __shared__ uint64_t si[LS_CHUNK];
    __shared__ uint64_t sp[POS ? LS_CHUNK : 1];
    const uint32_t q = q0 + blockIdx.y;
    if (skip_query(a, q)) return;
    const uint32_t cnt = lk_count(a, state, q), c0 = blockIdx.x * LS_CHUNK;
    if (c0 >= cnt) return;
    const uint32_t n = min(cnt - c0, LS_CHUNK);
    uint32_t n2 = 2;
    while (n2 < n) n2 <<= 1;
    const size_t base = (size_t)q * a.k + c0;
    for (uint32_t i = threadIdx.x; i < n2; i += LS_THREADS) {
        const bool have = i < n;
        sk[i] = have ? buf.key[base + i] : 0xffffffffu;
        si[i] = have ? buf.id[base + i] : UINT64_MAX;
        if (POS) sp[i] = have ? buf.pos[base + i] : UINT64_MAX;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= n2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < (n2 >> 1); i += LS_THREADS) {
                const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool asc = (lo & size) == 0;
                const uint32_t ka = sk[lo], kb = sk[hi];
                const uint64_t ia = si[lo], ib = si[hi];
                if (lk_less(kb, ib, ka, ia) == asc) {
                    sk[lo] = kb; sk[hi] = ka; si[lo] = ib; si[hi] = ia;
                    if (POS) { const uint64_t p = sp[lo]; sp[lo] = sp[hi]; sp[hi] = p; }
                }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < n; i += LS_THREADS) {
        buf.key[base + i] = sk[i]; buf.id[base + i] = si[i];
        if (POS) buf.pos[base + i] = sp[i];
    }
}

// one merge pass: the sorted runs [2 j w, 2 j w + w) and [2 j w + w, 2 (j + 1) w) of src into run j of dst (merge
// path: each thread finds where its LS_MERGE_ITEMS outputs start by a binary search on its diagonal).  Ties between
// the runs (repeated (key, id) pairs only) take the first run's entry first.  Grid (ceil(k / (LS_THREADS items)), B).
template <bool POS>
__global__ void __launch_bounds__(LS_THREADS) lk_merge_kernel(SelectArgs a, const LkState *state, LkBuf src, LkBuf dst,
                                                             uint32_t w, uint32_t q0)
{
    const uint32_t q = q0 + blockIdx.y;
    if (skip_query(a, q)) return;
    const uint32_t n = lk_count(a, state, q);
    const uint32_t g0 = (blockIdx.x * LS_THREADS + threadIdx.x) * LS_MERGE_ITEMS;
    if (g0 >= n) return;
    const uint32_t run0 = g0 / (2 * w) * (2 * w), o = g0 - run0;   // 2 w is a multiple of LS_MERGE_ITEMS
    const uint32_t la = min(w, n - run0), lb = n - run0 > w ? min(w, n - run0 - w) : 0;
    const size_t qa = (size_t)q * a.k + run0, qb = qa + w;
    const uint32_t *ka = src.key + qa, *kb = src.key + qb;
    const uint64_t *ia = src.id + qa, *ib = src.id + qb;
    uint32_t lo = o > lb ? o - lb : 0, hi = min(o, la);
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1, j = o - 1 - mid;
        if (!lk_less(kb[j], ib[j], ka[mid], ia[mid])) lo = mid + 1;    // a[mid] <= b[j]: a[mid] comes first
        else hi = mid;
    }
    uint32_t i = lo, j = o - lo;
    const size_t out = qa + o;
    const uint32_t m = min((uint32_t)LS_MERGE_ITEMS, la + lb - o);
    for (uint32_t e = 0; e < m; e++) {
        const bool take_a = i < la && (j >= lb || !lk_less(kb[j], ib[j], ka[i], ia[i]));
        const size_t from = take_a ? qa + i : qb + j;
        dst.key[out + e] = src.key[from]; dst.id[out + e] = src.id[from];
        if (POS) dst.pos[out + e] = src.pos[from];
        if (take_a) i++; else j++;
    }
}

// the outputs: the sorted rows, then unused slots (UINT64_MAX / +inf); the count.  Grid (ceil(k / LS_THREADS), B).
template <bool POS>
__global__ void __launch_bounds__(LS_THREADS) lk_write_kernel(SelectArgs a, const LkState *state, LkBuf buf,
                                                             uint32_t q0)
{
    const uint32_t q = q0 + blockIdx.y;
    if (skip_query(a, q)) return;
    const uint32_t n = lk_count(a, state, q), i = blockIdx.x * LS_THREADS + threadIdx.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) a.out_count[q] = n;
    if (i >= a.k) return;
    const size_t at = (size_t)q * a.k + i;
    const bool have = i < n;
    const uint64_t oid = have ? buf.id[at] : UINT64_MAX;
    const float od = have ? key_f32(buf.key[at]) : CUDART_INF_F;
    if (a.out_rec) { TopkRecord r; r.id = oid; r.dist = od; r.pad = 0u; a.out_rec[at] = r; }
    else { a.out_ids[at] = oid; a.out_dist[at] = od; }
    if (POS) a.out_pos[at] = have ? buf.pos[at] : UINT64_MAX;
}

// the whole pipeline for queries [q0, q0 + nq) (nq <= 65535: the queries are the grids' y dimension)
template <bool POS>
void run_large(const SelectArgs &a, const LkScratch &s, uint32_t q0, uint32_t nq, int sms, cudaStream_t st)
{
    const uint32_t k = a.k;
    // slices per query: enough CTAs to cover the SMs a few times over (mode 0's candidate count is only known on the
    // device), never more than one per LS_THREADS x 8 candidates of a dense row or list
    uint64_t slices = std::max<uint64_t>(1, (uint64_t)4 * sms / nq);
    if (a.mode != 0) slices = std::min<uint64_t>(slices, std::max<uint64_t>(1, a.ncols / (LS_THREADS * 8)));
    slices = std::min<uint64_t>(slices, 65535);
    const dim3 pass_grid((uint32_t)slices, nq);
    auto pass = [&](uint32_t phase) {
        lk_hist_kernel<<<pass_grid, LS_THREADS, 0, st>>>(a, s.state, s.hist, phase, q0); LGPU_COUNT_LAUNCH();
        lk_walk_kernel<<<nq, LS_THREADS, 0, st>>>(a, s.state, s.hist, phase, q0); LGPU_COUNT_LAUNCH();
    };
    pass(LK_KEY0); pass(LK_KEY1); pass(LK_KEY2);
    pass(LK_RANGE);
    for (int i = 0; i < LS_ID_PASSES; i++) pass(LK_ID);
    LkBuf b0 = s.buf[0], b1 = s.buf[1];
    lk_compact_kernel<POS><<<pass_grid, LS_THREADS, 0, st>>>(a, s.state, b0, q0); LGPU_COUNT_LAUNCH();
    lk_chunk_sort_kernel<POS><<<dim3(ceil_div(k, LS_CHUNK), nq), LS_THREADS, 0, st>>>(a, s.state, b0, q0);
    LGPU_COUNT_LAUNCH();
    const dim3 merge_grid(ceil_div(k, LS_THREADS * LS_MERGE_ITEMS), nq);
    for (uint32_t w = LS_CHUNK; w < k; w *= 2) {
        lk_merge_kernel<POS><<<merge_grid, LS_THREADS, 0, st>>>(a, s.state, b0, b1, w, q0); LGPU_COUNT_LAUNCH();
        std::swap(b0, b1);
    }
    lk_write_kernel<POS><<<dim3(ceil_div(k, LS_THREADS), nq), LS_THREADS, 0, st>>>(a, s.state, b0, q0);
    LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace

size_t select_large_scratch_bytes(uint32_t B, uint32_t k, bool pos)
{
    const size_t entry = 4 + 8 + (pos ? 8 : 0);
    return align256((size_t)B * sizeof(LkState)) + align256((size_t)B * LS_BINS * 4) +
           2 * ((size_t)B * k * entry + (pos ? 3 : 2) * 256);
}

void launch_select_large(const SelectArgs &a, cudaStream_t st)
{
    if (a.B == 0) return;
    LGPU_REQUIRE(a.k > SELECT_KMAX && a.k <= LGPU_K_MAX, "limit+offset (k) above 65536 (LGPU_K_MAX) is not supported");
    LGPU_REQUIRE(a.scratch && a.scratch_bytes >= select_large_scratch_bytes(a.B, a.k, a.out_pos != nullptr),
                 "the top-k select above k = 2048 needs its scratch buffer");
    const LkScratch s = carve(a.scratch, a.B, a.k, a.out_pos != nullptr);
    int dev = 0, sms = 0;
    LGPU_CUDA(cudaGetDevice(&dev));
    LGPU_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    lk_init_kernel<<<ceil_div(a.B, 256), 256, 0, st>>>(s.state, a.B, a.k); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaMemsetAsync(s.hist, 0, (size_t)a.B * LS_BINS * 4, st));
    for (uint32_t q0 = 0; q0 < a.B; q0 += 65535) {
        const uint32_t nq = std::min<uint32_t>(65535, a.B - q0);
        if (a.out_pos) run_large<true>(a, s, q0, nq, sms, st);
        else run_large<false>(a, s, q0, nq, sms, st);
    }
}

}  // namespace lgpu
