// select.cu -- K4: per-query top-k by (_distance ASC, _rowid ASC).
//
// Replaces the per-partition bounded heap + SortExec TopK(fetch=k) merge
// [lance, recalled; SURVEY.md 8a rows a8-a9; tie-break pinned by
// python/python/lancedb/query.py:1366-1368].  Also used to pick the
// nprobes nearest centroids (IvfModel::find_partitions' sort_to_indices) and for the
// flat / refine / multi-GPU merge paths.
//
// One CTA per query streams that query's candidate distances (coalesced float4),
// keeps only those not worse than the current k-th best, and stages survivors
// (ordered-uint distance key, row id) in shared memory; when `trigger` survivors have
// piled up it bitonic-sorts them, keeps k, and tightens the threshold.  The first sort
// happens after the first 1024 candidates, after which the pass rate collapses to
// ~k/seen, so a query costs one ~1024-element sort plus a small final sort.
// Integer work (ids, ordering) is exact; distances are passed through untouched.
#include "kernels.cuh"

#include <math_constants.h>

namespace lgpu {

namespace {

constexpr int SEL_THREADS = 256;
constexpr int SEL_ITER = SEL_THREADS * 4;

struct Stage {
    uint32_t *keys;
    uint64_t *ids;
    uint64_t *pos;   // may be null
};

__device__ __forceinline__ bool key_less(uint32_t ka, uint64_t ia, uint32_t kb, uint64_t ib)
{
    return ka < kb || (ka == kb && ia < ib);
}

// bitonic sort of the first n2 (power of two) staged entries, ascending
template <bool POS>
__device__ void bitonic_sort(Stage s, uint32_t n2)
{
    for (uint32_t size = 2; size <= n2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < (n2 >> 1); i += SEL_THREADS) {
                uint32_t lo = 2 * i - (i & (stride - 1));
                uint32_t hi = lo + stride;
                bool asc = (lo & size) == 0;
                uint32_t ka = s.keys[lo], kb = s.keys[hi];
                uint64_t ia = s.ids[lo], ib = s.ids[hi];
                bool gt = key_less(kb, ib, ka, ia);
                if (gt == asc) {
                    s.keys[lo] = kb; s.keys[hi] = ka;
                    s.ids[lo] = ib; s.ids[hi] = ia;
                    if (POS) { uint64_t pa = s.pos[lo]; s.pos[lo] = s.pos[hi]; s.pos[hi] = pa; }
                }
            }
            __syncthreads();
        }
    }
}

__device__ __forceinline__ bool allow_bit(const SelectArgs &a, uint64_t id)
{
    return id < a.allow_bits && ((a.allow[id >> 5] >> (id & 31)) & 1u);
}

__device__ __forceinline__ void write_entry(const SelectArgs &a, size_t at, bool have, uint64_t id, uint32_t key)
{
    const uint64_t oid = have ? id : UINT64_MAX;
    const float od = have ? key_f32(key) : CUDART_INF_F;
    if (a.out_rec) { TopkRecord r; r.id = oid; r.dist = od; r.pad = 0u; a.out_rec[at] = r; }
    else { a.out_ids[at] = oid; a.out_dist[at] = od; }
}

template <bool POS>
__global__ void __launch_bounds__(SEL_THREADS) select_kernel(SelectArgs a, uint32_t cap, uint32_t trigger)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    extern __shared__ __align__(16) unsigned char smem[];
    Stage st;
    st.ids = reinterpret_cast<uint64_t *>(smem);
    st.pos = POS ? st.ids + cap : nullptr;
    st.keys = reinterpret_cast<uint32_t *>(smem + (size_t)cap * 8 * (POS ? 2 : 1));
    __shared__ uint32_t s_cnt, s_tau;

    const uint32_t q = blockIdx.x;
    if (a.gate && *a.gate == 0) return;
    if (a.only && !a.only[q]) return;                       // fix-up pass: untouched query
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) { s_cnt = 0; s_tau = 0xffffffffu; }
    __syncthreads();

    auto in_range = [&](float v) -> bool {
        if (v != v) return false;                           // FilterExec: _distance IS NOT NULL
        if (a.has_lower && !(v >= a.lower)) return false;
        if (a.has_upper && !(v < a.upper)) return false;
        return true;
    };
    // sort what is staged, keep the k best, tighten the threshold.  Whether to compact is decided inside the barrier that
    // ends an iteration (__syncthreads_or: the last thread to arrive sees every append of the iteration), so the whole
    // CTA takes the same branch.  Reading s_cnt after a plain barrier does not: a warp that skips the compaction goes on
    // appending for the next iteration, a slower warp then reads a count at or above `trigger` and enters compact()
    // alone, and the CTA's barriers no longer pair up -- seen as wrong rows, now and then, when the staged count lands
    // right at the trigger (k = 432: 432 kept + about 432 of the next 1024 rows = 2 k)
    auto compact = [&]() {
        uint32_t cnt = s_cnt;
        uint32_t n2 = 2;
        while (n2 < cnt) n2 <<= 1;
        for (uint32_t i = cnt + tid; i < n2; i += SEL_THREADS) { st.keys[i] = 0xffffffffu; st.ids[i] = UINT64_MAX; }
        __syncthreads();
        bitonic_sort<POS>(st, n2);
        if (tid == 0) {
            uint32_t keep = cnt < a.k ? cnt : a.k;
            s_cnt = keep;
            if (keep == a.k && a.k > 0) s_tau = st.keys[a.k - 1];
        }
        __syncthreads();
    };
    // offer up to 4 candidates per thread; warp-aggregated staging
    auto offer4 = [&](const float v[4], const bool ok[4], const uint64_t idbase, const uint64_t *idsrc,
                      const uint64_t posbase) {
        const uint32_t tau = s_tau;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            float f = v[u];
            if (f == 0.f) f = 0.f;                           // -0 and +0 tie
            uint32_t key = f32_key(f);
            bool pass = ok[u] && in_range(f) && key <= tau;
            uint64_t id = 0;
            if (pass) {
                id = idsrc ? idsrc[idbase + u] : idbase + u;
                if (a.allow) pass = allow_bit(a, id);
            }
            unsigned mask = __ballot_sync(0xffffffffu, pass);
            if (mask) {
                uint32_t base = 0;
                if (lane == (__ffs(mask) - 1)) base = atomicAdd(&s_cnt, __popc(mask));
                base = __shfl_sync(0xffffffffu, base, __ffs(mask) - 1);
                if (pass) {
                    uint32_t slot = base + __popc(mask & ((1u << lane) - 1));
                    st.keys[slot] = key;
                    st.ids[slot] = id;
                    if (POS) st.pos[slot] = posbase + u;
                }
            }
        }
    };

    if (a.mode == 0) {
        for (uint32_t j = 0; j < a.nprobes; j++) {
            const uint32_t slot = q * a.nprobes + j;
            const uint64_t pp = a.probes[slot];
            if (pp >= a.nlist) continue;                   // unused probe slot (fewer than nprobes finite distances)
            const uint32_t p = (uint32_t)pp;
            const uint32_t n = a.part_n[p];
            const float *src = a.dist + a.seg_off[slot];
            const uint64_t rowbase = a.part_off[p];
            for (uint32_t r0 = 0; r0 < n; r0 += SEL_ITER) {
                uint32_t r = r0 + tid * 4;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                bool ok[4];
                if (r < n) {
                    float4 t = *reinterpret_cast<const float4 *>(src + r);   // segment padded to 4
                    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
                }
#pragma unroll
                for (int u = 0; u < 4; u++) ok[u] = r + u < n;
                offer4(v, ok, rowbase + r, a.row_ids, rowbase + r);
                if (__syncthreads_or(s_cnt >= trigger)) compact();
            }
        }
    } else if (a.mode == 1) {
        const float *src = a.dense + (size_t)q * a.row_stride;
        const bool aligned = ((a.row_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.dense) & 15) == 0);
        for (uint64_t c0 = 0; c0 < a.ncols; c0 += SEL_ITER) {
            uint64_t c = c0 + (uint64_t)tid * 4;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            bool ok[4];
            if (aligned && c + 3 < a.ncols) {
                float4 t = *reinterpret_cast<const float4 *>(src + c);
                v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
            } else {
#pragma unroll
                for (int u = 0; u < 4; u++) if (c + u < a.ncols) v[u] = src[c + u];
            }
#pragma unroll
            for (int u = 0; u < 4; u++) ok[u] = c + u < a.ncols;
            offer4(v, ok, a.col_ids ? c : a.col_base + c, a.col_ids, c);
            if (__syncthreads_or(s_cnt >= trigger)) compact();
        }
    } else {
        const uint64_t ncols = a.ncols_q ? min((uint64_t)a.ncols_q[q], a.ncols) : a.ncols;
        for (uint64_t c0 = 0; c0 < ncols; c0 += SEL_ITER) {
            uint64_t c = c0 + (uint64_t)tid * 4;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            bool ok[4];
            uint64_t idv[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                ok[u] = false; idv[u] = UINT64_MAX;
                if (c + u < ncols && (!a.list_cnt || (c + u) % a.inner < a.list_cnt[(c + u) / a.inner * a.B + q])) {
                    uint64_t cc = c + u;
                    uint64_t addr = (cc / a.inner) * a.outer_stride + (uint64_t)q * a.row_stride + cc % a.inner;
                    if (a.cand_rec) { const TopkRecord r = a.cand_rec[addr]; idv[u] = r.id; v[u] = r.dist; }
                    else { idv[u] = a.cand_ids[addr]; v[u] = a.dense[addr]; }
                    ok[u] = idv[u] != UINT64_MAX;           // unused slot of a shorter list
                }
            }
            // ids differ per entry: stage them through the id "source" one at a time
            const uint32_t tau = s_tau;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                float f = v[u];
                if (f == 0.f) f = 0.f;
                uint32_t key = f32_key(f);
                bool pass = ok[u] && in_range(f) && key <= tau;
                if (pass && a.allow) pass = allow_bit(a, idv[u]);
                unsigned mask = __ballot_sync(0xffffffffu, pass);
                if (mask) {
                    uint32_t base = 0;
                    if (lane == (__ffs(mask) - 1)) base = atomicAdd(&s_cnt, __popc(mask));
                    base = __shfl_sync(0xffffffffu, base, __ffs(mask) - 1);
                    if (pass) {
                        uint32_t slot = base + __popc(mask & ((1u << lane) - 1));
                        st.keys[slot] = key;
                        st.ids[slot] = idv[u];
                        if (POS) {
                            uint64_t cc = c + u;
                            uint64_t addr = (cc / a.inner) * a.outer_stride + (uint64_t)q * a.row_stride + cc % a.inner;
                            st.pos[slot] = a.cand_pos ? a.cand_pos[addr] : cc;
                        }
                    }
                }
            }
            if (__syncthreads_or(s_cnt >= trigger)) compact();
        }
    }
    __syncthreads();
    compact();
    const uint32_t cnt = s_cnt;
    for (uint32_t i = tid; i < a.k; i += SEL_THREADS) {
        bool have = i < cnt;
        write_entry(a, (size_t)q * a.k + i, have, st.ids[i], st.keys[i]);
        if (POS) a.out_pos[(size_t)q * a.k + i] = have ? st.pos[i] : UINT64_MAX;
    }
    if (tid == 0) a.out_count[q] = cnt;
}

// ---------------------------------------------------------------------------------
// k <= 32: four warps per query; every warp keeps the k best of its share in registers, lane i holding its i-th best.
// Candidates stream through 8 per lane per iteration (two float4 loads in flight) and only the ones not worse than the
// warp's current k-th best are inserted (ballot loop).  After warm-up almost nothing passes, so a query costs ~1 compare
// per candidate.  The four queues are merged through shared memory.
#ifndef SELW_WARPS_V
#define SELW_WARPS_V 4
#endif
constexpr int SELW_WARPS = SELW_WARPS_V;       // power of two

template <bool POS>
__global__ void __launch_bounds__(SELW_WARPS * 32) select_warp_kernel(SelectArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    __shared__ uint32_t m_key[SELW_WARPS - 1][32];
    __shared__ uint64_t m_id[SELW_WARPS - 1][32];
    __shared__ uint64_t m_pos[SELW_WARPS - 1][POS ? 32 : 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x;
    if (a.gate && *a.gate == 0) return;
    if (a.only && !a.only[q]) return;                       // fix-up pass: untouched query
    const uint32_t k = a.k;
    uint32_t qk = 0xffffffffu;                              // the warp's queue, sorted ascending over the lanes
    uint64_t qid = UINT64_MAX, qpos = UINT64_MAX;
    uint32_t tau_k = 0xffffffffu;                           // (key, id) of the k-th best so far
    uint64_t tau_id = UINT64_MAX;
    const int tau_lane = (int)k - 1;

    auto in_range = [&](float v) -> bool {
        if (v != v) return false;
        if (a.has_lower && !(v >= a.lower)) return false;
        if (a.has_upper && !(v < a.upper)) return false;
        return true;
    };
    // offer one candidate per lane (pass == false for lanes without one)
    auto offer = [&](bool pass, uint32_t key, uint64_t id, uint64_t pos) {
        unsigned m = __ballot_sync(0xffffffffu, pass);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t ck = __shfl_sync(0xffffffffu, key, src);
            const uint64_t cid = __shfl_sync(0xffffffffu, id, src);
            if (!key_less(ck, cid, tau_k, tau_id)) continue;          // threshold moved meanwhile
            const uint64_t cpos = POS ? __shfl_sync(0xffffffffu, pos, src) : 0;
            // the queue is sorted: `at` entries are smaller; lanes >= at shift up by one
            const int at = __popc(__ballot_sync(0xffffffffu, key_less(qk, qid, ck, cid)));
            const uint32_t uk = __shfl_up_sync(0xffffffffu, qk, 1);
            const uint64_t uid = __shfl_up_sync(0xffffffffu, qid, 1);
            const uint64_t upos = POS ? __shfl_up_sync(0xffffffffu, qpos, 1) : 0;
            if (lane == at) { qk = ck; qid = cid; if (POS) qpos = cpos; }
            else if (lane > at) { qk = uk; qid = uid; if (POS) qpos = upos; }
            if (lane >= (int)k) { qk = 0xffffffffu; qid = UINT64_MAX; }
            tau_k = __shfl_sync(0xffffffffu, qk, tau_lane);
            tau_id = __shfl_sync(0xffffffffu, qid, tau_lane);
        }
    };
    auto offer4 = [&](const float4 t, uint64_t n_left, uint64_t idbase, const uint64_t *idsrc, uint64_t posbase) {
        const float v[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
        for (int u = 0; u < 4; u++) {
            float f = v[u];
            if (f == 0.f) f = 0.f;                          // -0 and +0 tie
            const uint32_t key = f32_key(f);
            bool pass = (uint64_t)u < n_left && in_range(f) && key <= tau_k;
            uint64_t id = 0;
            if (pass) {
                id = idsrc ? idsrc[idbase + u] : idbase + u;
                if (a.allow) pass = allow_bit(a, id);
            }
            offer(pass, key, id, posbase + u);
        }
    };
    // one warp-iteration = 256 consecutive values of `src` starting at r0 (n values in total)
    // (ids from idsrc[idbase + r], or idbase + r without idsrc; positions posbase + r)
    auto scan256 = [&](const float *src, uint64_t r0, uint64_t n, bool vec, uint64_t posbase, uint64_t idbase,
                       const uint64_t *idsrc) {
        const uint64_t ra = r0 + (uint64_t)lane * 4, rb = ra + 128;
        float4 ta = make_float4(0.f, 0.f, 0.f, 0.f), tb = ta;
        if (vec) {
            if (ra < n) ta = *reinterpret_cast<const float4 *>(src + ra);   // rows padded to 4 floats
            if (rb < n) tb = *reinterpret_cast<const float4 *>(src + rb);
        } else {
            float *pa = reinterpret_cast<float *>(&ta), *pb = reinterpret_cast<float *>(&tb);
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (ra + u < n) pa[u] = src[ra + u];
                if (rb + u < n) pb[u] = src[rb + u];
            }
        }
        offer4(ta, ra < n ? n - ra : 0, idbase + ra, idsrc, posbase + ra);
        offer4(tb, rb < n ? n - rb : 0, idbase + rb, idsrc, posbase + rb);
    };

    if (a.mode == 0) {
        uint32_t itc = 0;                                   // iteration counter across segments
        for (uint32_t j = 0; j < a.nprobes; j++) {
            const uint32_t slot = q * a.nprobes + j;
            const uint64_t pp = a.probes[slot];
            if (pp >= a.nlist) continue;                   // unused probe slot (fewer than nprobes finite distances)
            const uint32_t p = (uint32_t)pp;
            const uint32_t n = a.part_n[p];
            const float *src = a.dist + a.seg_off[slot];
            const uint64_t rowbase = a.part_off[p];
            for (uint32_t r0 = 0; r0 < n; r0 += 256, itc++)
                if ((itc & (SELW_WARPS - 1)) == (uint32_t)w) scan256(src, r0, n, true, rowbase, rowbase, a.row_ids);
        }
    } else if (a.mode == 1) {
        const float *src = a.dense + (size_t)q * a.row_stride;
        const bool aligned = ((a.row_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.dense) & 15) == 0);
        for (uint64_t c0 = (uint64_t)w * 256; c0 < a.ncols; c0 += 256 * SELW_WARPS) {
            const bool vec = aligned && c0 + 256 <= a.ncols;
            scan256(src, c0, a.ncols, vec, 0, a.col_ids ? 0 : a.col_base, a.col_ids);
        }
    } else {
        const uint64_t ncols = a.ncols_q ? min((uint64_t)a.ncols_q[q], a.ncols) : a.ncols;
        for (uint64_t c0 = (uint64_t)w * 32; c0 < ncols; c0 += 32 * SELW_WARPS) {
            const uint64_t cc = c0 + lane;
            bool pass = false;
            uint32_t key = 0;
            uint64_t id = UINT64_MAX, pos = cc;
            const uint64_t l = cc / a.inner, e = cc - l * a.inner;     // list, entry
            if (cc < ncols && (!a.list_cnt || e < a.list_cnt[l * a.B + q])) {
                const uint64_t addr = l * a.outer_stride + (uint64_t)q * a.row_stride + e;
                float f;
                if (a.cand_rec) { const TopkRecord r = a.cand_rec[addr]; id = r.id; f = r.dist; }
                else { id = a.cand_ids[addr]; f = a.dense[addr]; }
                if (f == 0.f) f = 0.f;
                key = f32_key(f);
                pass = id != UINT64_MAX && in_range(f) && key <= tau_k;
                if (pass && a.allow) pass = allow_bit(a, id);
                if (POS && a.cand_pos) pos = a.cand_pos[addr];
            }
            offer(pass, key, id, pos);
        }
    }
    // merge the four queues: warps 1..3 publish, warp 0 inserts
    if (w > 0) {
        m_key[w - 1][lane] = qk; m_id[w - 1][lane] = qid;
        if (POS) m_pos[w - 1][lane] = qpos;
    }
    __syncthreads();
    if (w > 0) return;
#pragma unroll
    for (int o = 0; o < SELW_WARPS - 1; o++) {
        const uint32_t ck = m_key[o][lane];
        const uint64_t cid = m_id[o][lane];
        offer(cid != UINT64_MAX || ck != 0xffffffffu, ck, cid, POS ? m_pos[o][lane] : 0);
    }
    const bool have = qid != UINT64_MAX || qk != 0xffffffffu;
    const uint32_t total = __popc(__ballot_sync(0xffffffffu, have));
    if (lane < (int)k) {
        write_entry(a, (size_t)q * k + lane, have, qid, qk);
        if (POS) a.out_pos[(size_t)q * k + lane] = have ? qpos : UINT64_MAX;
    }
    if (lane == 0) a.out_count[q] = min(total, k);
}

__global__ void pack_records_kernel(const uint64_t *__restrict__ ids, const float *__restrict__ dist, uint64_t n,
                                    TopkRecord *__restrict__ out)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    TopkRecord r; r.id = ids[i]; r.dist = dist[i]; r.pad = 0u;
    out[i] = r;
}

}  // namespace

__global__ void count_below_kernel(const uint32_t *__restrict__ cnt, uint32_t B, uint32_t k, uint32_t *__restrict__ flags)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < B) flags[q] = cnt[q] < k ? 1u : 0u;
}

void launch_count_below(const uint32_t *cnt, uint32_t B, uint32_t k, uint32_t *flags, cudaStream_t st)
{
    if (B == 0) return;
    count_below_kernel<<<(B + 255) / 256, 256, 0, st>>>(cnt, B, k, flags); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_pack_records(const uint64_t *ids, const float *dist, uint64_t n, TopkRecord *out, cudaStream_t st)
{
    if (n == 0) return;
    pack_records_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ids, dist, n, out); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

void launch_select(const SelectArgs &a, cudaStream_t st)
{
    if (a.B == 0) return;
    if (a.k > SELECT_KMAX) { launch_select_large(a, st); return; }   // select_large.cu
    LGPU_REQUIRE(a.k >= 1, "limit+offset (k) must be at least 1");
    // above k = 32 the warp queues' serial inserts (k ln(n/k) per warp) dominate: the shared-memory stage + bitonic
    // kernel is the faster one there
    if (a.k <= 32) {
        if (a.out_pos) launch_k(select_warp_kernel<true>, dim3(a.B), dim3(SELW_WARPS * 32), 0, st, a);
        else launch_k(select_warp_kernel<false>, dim3(a.B), dim3(SELW_WARPS * 32), 0, st, a);
        LGPU_COUNT_LAUNCH();
        LGPU_CUDA(cudaGetLastError());
        return;
    }
    uint32_t trigger = a.k * 2 < 512 ? 512 : a.k * 2;
    uint32_t cap = 2;
    while (cap < trigger + SEL_ITER) cap <<= 1;
    const bool pos = a.out_pos != nullptr;
    size_t smem = (size_t)cap * (pos ? 20 : 12);
    if (pos) {
        LGPU_CUDA(cudaFuncSetAttribute(select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        launch_k(select_kernel<true>, dim3(a.B), dim3(SEL_THREADS), smem, st, a, cap, trigger); LGPU_COUNT_LAUNCH();
    } else {
        LGPU_CUDA(cudaFuncSetAttribute(select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        launch_k(select_kernel<false>, dim3(a.B), dim3(SEL_THREADS), smem, st, a, cap, trigger); LGPU_COUNT_LAUNCH();
    }
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
