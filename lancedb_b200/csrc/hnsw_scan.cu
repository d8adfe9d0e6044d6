// hnsw_scan.cu -- IVF_HNSW_SQ: the graph search of every probe slot, one warp per slot, over IVF_SQ's codes.
//
// The search (include/lancedb_b200.h, IVF_HNSW_SQ; the CPU statement is tests/hnsw_sq_oracle.c): a greedy descent
// through the upper levels, then the level-0 loop over W (the ef' best rows seen, each expanded or not) and R (the kk
// best evaluated rows that pass the row filter), both kept sorted in shared memory by the key (d, position):
//     key = f32 bits of d << 32 | position        (d >= 0, so the bits order like the floats; positions < 2^31)
// Bit 31 of a W key marks the row expanded; comparisons mask it off.
//
// Persistent CTAs: each warp claims one probe slot at a time from a counter.  Per expansion the warp loads the row's
// <= 2m level-0 neighbours (a lane per neighbour), drops those its visited cache has seen, and scores the rest eight
// lanes per neighbour with 16-byte loads of the row's and the query's codes: |k - q| per byte (vabsdiffu4) squared and
// summed by dp4a into a u32, exact modulo 2^32 as in sq_scan.cu, then one round to f32.  A group of eight lanes per
// neighbour keeps every lane's loads 16-byte wide at any dim (dim_pad is a multiple of 64) while scoring four
// neighbours at once; a lane per neighbour would read each row with 32 different strides.
//
// The whole batch is then merged into W and into R at once.  That is exact because the result of offering a batch
// to a bounded sorted list does not depend on the order of its members, and a row that was evicted (or refused) can
// never re-enter (the threshold only tightens).  The visited cache is lossy (a direct-mapped table of positions): a
// row it forgets is scored and offered again, and W and R reject it as a duplicate, so only work changes.
#include "kernels.cuh"

namespace lgpu {

namespace {

constexpr uint32_t HNSW_VIS = 1024;              // visited-cache entries per warp
constexpr uint32_t HNSW_BATCH = 128;             // 2 x LGPU_HNSW_MAX_M
constexpr uint32_t HNSW_FLAG = 1u << 31;
constexpr uint32_t HNSW_MAX_WARPS = 8;
constexpr unsigned FULL = 0xffffffffu;

__host__ __device__ constexpr size_t hnsw_warp_smem(uint32_t efp, uint32_t kk)
{
    return (size_t)8 * (efp + kk + HNSW_BATCH) + 4 * (HNSW_VIS + 2 * HNSW_BATCH);
}

__device__ __forceinline__ uint64_t masked(uint64_t k) { return k & ~(uint64_t)HNSW_FLAG; }
__device__ __forceinline__ uint32_t vis_slot(uint32_t pos) { return (pos * 2654435761u) >> 22; }   // 10 bits

__device__ __forceinline__ uint32_t sqd4(uint32_t a, uint32_t b, uint32_t acc)
{
    const uint32_t d = __vabsdiffu4(a, b);
    return __dp4a(d, d, acc);
}

// bk[i] = key of row bpos[i] (i < c) for the query codes qc; rows at pc + pos * dim_pad
__device__ void score_batch(const uint8_t *__restrict__ pc, const uint8_t *__restrict__ qc, uint32_t dim_pad,
                            const uint32_t *bpos, uint64_t *bk, uint32_t c, int lane)
{
    const uint32_t g = lane >> 3, li = lane & 7;
    for (uint32_t i0 = 0; i0 < c; i0 += 4) {
        const uint32_t i = i0 + g;
        uint32_t s = 0;
        if (i < c) {
            const uint8_t *row = pc + (uint64_t)bpos[i] * dim_pad;
            for (uint32_t o = li * 16; o < dim_pad; o += 128) {
                const uint4 x = __ldg(reinterpret_cast<const uint4 *>(row + o));
                const uint4 y = __ldg(reinterpret_cast<const uint4 *>(qc + o));
                s = sqd4(x.x, y.x, s); s = sqd4(x.y, y.y, s); s = sqd4(x.z, y.z, s); s = sqd4(x.w, y.w, s);
            }
        }
        s += __shfl_xor_sync(FULL, s, 4);
        s += __shfl_xor_sync(FULL, s, 2);
        s += __shfl_xor_sync(FULL, s, 1);
        if (i < c && li == 0) bk[i] = (uint64_t)__float_as_uint(__uint2float_rn(s)) << 32 | bpos[i];
    }
    __syncwarp();
}

// Merge the batch bk[0..c) -- the members whose bit is set in ok[] -- into the sorted list arr[0..n) of capacity cap:
// arr becomes the cap smallest of the union, a key already in arr or repeated in the batch entering once.  sra:
// scratch [HNSW_BATCH].  Returns the new length; *first = the index of the first inserted key (>= cap: none).
__device__ uint32_t merge_batch(uint64_t *arr, uint32_t n, uint32_t cap, const uint64_t *bk, uint32_t c,
                                const uint32_t (&ok)[4], uint32_t *sra, uint32_t *first, int lane)
{
    bool v[4];
    uint32_t ra[4];
    uint64_t key[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const uint32_t i = lane + 32 * j;
        v[j] = i < c && (ok[j] >> lane & 1u);
        ra[j] = 0; key[j] = 0;
        if (v[j]) {
            key[j] = bk[i];
            uint32_t lo = 0, hi = n;                           // first index with masked(arr) >= key
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (masked(arr[mid]) < key[j]) lo = mid + 1; else hi = mid;
            }
            ra[j] = lo;
            if (lo >= cap || (lo < n && masked(arr[lo]) == key[j])) v[j] = false;
            for (uint32_t t = 0; t < i && v[j]; t++)
                if (bk[t] == key[j] && (ok[t >> 5] >> (t & 31) & 1u)) v[j] = false;
        }
    }
    uint32_t vm[4], nv = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) { vm[j] = __ballot_sync(FULL, v[j]); nv += __popc(vm[j]); }
    *first = cap;
    if (nv == 0) return n;
    uint32_t fin[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        fin[j] = cap;
        if (!v[j]) continue;
        uint32_t rb = 0;
        for (uint32_t t = 0; t < c; t++)
            if ((vm[t >> 5] >> (t & 31) & 1u) && bk[t] < key[j]) rb++;
        sra[rb] = ra[j];
        fin[j] = ra[j] + rb;
    }
    __syncwarp();
    const uint32_t lo_min = sra[0];
    // entries at t >= lo_min move right by the number of inserted keys with rank <= t, from the top down
    for (int hi = (int)n; hi > (int)lo_min; hi -= 32) {
        const int t = hi - 1 - lane;
        uint64_t val = 0;
        uint32_t dst = cap;
        if (t >= (int)lo_min) {
            val = arr[t];
            uint32_t a = 0, b = nv;                            // count of sra[] <= t
            while (a < b) { const uint32_t mid = (a + b) >> 1; if (sra[mid] <= (uint32_t)t) a = mid + 1; else b = mid; }
            dst = (uint32_t)t + a;
        }
        __syncwarp();
        if (dst < cap) arr[dst] = val;
        __syncwarp();
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
        if (v[j] && fin[j] < cap) arr[fin[j]] = key[j];
    __syncwarp();
    *first = lo_min;
    return min(cap, n + nv);
}

// the row filter of R: distance_range and the allow bitmap (d is never NaN)
__device__ __forceinline__ bool passes(const HnswArgs &a, uint64_t key, uint64_t off)
{
    const float d = __uint_as_float((uint32_t)(key >> 32));
    if (a.has_lower && !(d >= a.lower)) return false;
    if (a.has_upper && !(d < a.upper)) return false;
    if (!a.allow) return true;
    const uint64_t id = __ldg(a.row_ids + off + (uint32_t)key);
    return id < a.allow_bits && (__ldg(a.allow + (id >> 5)) >> (id & 31) & 1u);
}

// compact the lanes' candidates (fresh[j]: nb[j] is one) into bpos; returns the count
__device__ __forceinline__ uint32_t compact(const bool (&fresh)[4], const uint32_t (&nb)[4], uint32_t *bpos, int lane)
{
    uint32_t c = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const uint32_t bal = __ballot_sync(FULL, fresh[j]);
        if (fresh[j]) bpos[c + __popc(bal & ((1u << lane) - 1u))] = nb[j];
        c += __popc(bal);
    }
    __syncwarp();
    return c;
}

__global__ void __launch_bounds__(HNSW_MAX_WARPS * 32, 1) hnsw_search_kernel(HnswArgs a)
{
    pdl_entry();
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *base = smem + (size_t)warp * hnsw_warp_smem(a.efp, a.kk);
    uint64_t *W = reinterpret_cast<uint64_t *>(base);
    uint64_t *R = W + a.efp;
    uint64_t *bk = R + a.kk;
    uint32_t *vis = reinterpret_cast<uint32_t *>(bk + HNSW_BATCH);
    uint32_t *bpos = vis + HNSW_VIS;
    uint32_t *sra = bpos + HNSW_BATCH;
    const uint32_t m = a.m, m2 = 2 * a.m;
    for (;;) {
        uint32_t s = 0;
        if (lane == 0) s = atomicAdd(a.counter, 1u);
        s = __shfl_sync(FULL, s, 0);
        if (s >= a.slots) break;
        const uint32_t q = s / a.nprobes;
        if (a.only && !__ldg(a.only + q)) continue;
        const uint64_t p = __ldg(a.probes + s);
        uint32_t rn = 0;
        uint64_t off = 0;
        if (p < a.nlist && __ldg(a.part_off + p + 1) > __ldg(a.part_off + p)) {
            off = __ldg(a.part_off + p);
            const uint8_t *pc = a.codes + off * a.dim_pad, *qc = a.qcodes + (uint64_t)q * a.dim_pad;
            for (uint32_t i = lane; i < HNSW_VIS; i += 32) vis[i] = LGPU_HNSW_NONE;
            // upper levels: greedy descent from the entry row
            uint32_t cur = __ldg(a.entry + p);
            if (lane == 0) bpos[0] = cur;
            __syncwarp();
            score_batch(pc, qc, a.dim_pad, bpos, bk, 1, lane);
            uint64_t ck = bk[0];
            for (int L = __ldg(a.top_level + p); L >= 1; L--) {
                for (;;) {
                    const uint32_t *nbl = a.upper_adj + ((uint64_t)__ldg(a.upper_index + off + cur) + L - 1) * m;
                    bool fresh[4]; uint32_t nb[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const uint32_t i = lane + 32 * j;
                        nb[j] = i < m ? __ldg(nbl + i) : LGPU_HNSW_NONE;
                        fresh[j] = nb[j] != LGPU_HNSW_NONE;
                    }
                    const uint32_t c = compact(fresh, nb, bpos, lane);
                    score_batch(pc, qc, a.dim_pad, bpos, bk, c, lane);
                    uint64_t best = ck;
                    for (uint32_t i = lane; i < c; i += 32) best = min(best, bk[i]);
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(FULL, best, o));
                    __syncwarp();
                    if (best >= ck) break;
                    ck = best; cur = (uint32_t)best;
                }
            }
            // level 0
            if (lane == 0) {
                W[0] = ck;
                vis[vis_slot(cur)] = cur;
                if (passes(a, ck, off)) { R[0] = ck; rn = 1; }
            }
            rn = __shfl_sync(FULL, rn, 0);
            __syncwarp();
            uint32_t wn = 1, cursor = 0;
            for (;;) {
                for (;;) {                                     // the first unexpanded entry from `cursor`
                    const uint32_t t = cursor + lane;
                    const uint32_t bal = __ballot_sync(FULL, t < wn && !((uint32_t)W[t] & HNSW_FLAG));
                    if (bal) { cursor += __ffs(bal) - 1; break; }
                    cursor += 32;
                    if (cursor >= wn) break;
                }
                if (cursor >= wn) break;
                const uint32_t node = (uint32_t)W[cursor] & ~HNSW_FLAG;
                __syncwarp();
                if (lane == 0) W[cursor] |= HNSW_FLAG;
                const uint32_t *nbl = a.adj0 + (off + node) * m2;
                bool fresh[4]; uint32_t nb[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t i = lane + 32 * j;
                    nb[j] = i < m2 ? __ldg(nbl + i) : LGPU_HNSW_NONE;
                    fresh[j] = nb[j] != LGPU_HNSW_NONE && vis[vis_slot(nb[j])] != nb[j];
                }
                const uint32_t c = compact(fresh, nb, bpos, lane);
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (fresh[j]) vis[vis_slot(nb[j])] = nb[j];
                __syncwarp();
                if (c == 0) continue;
                score_batch(pc, qc, a.dim_pad, bpos, bk, c, lane);
                uint32_t ok[4], first;
#pragma unroll
                for (int j = 0; j < 4; j++) ok[j] = __ballot_sync(FULL, lane + 32 * j < c);
                wn = merge_batch(W, wn, a.efp, bk, c, ok, sra, &first, lane);
                cursor = min(cursor, first);
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t i = lane + 32 * j;
                    ok[j] = __ballot_sync(FULL, i < c && passes(a, i < c ? bk[i] : 0, off));
                }
                rn = merge_batch(R, rn, a.kk, bk, c, ok, sra, &first, lane);
            }
        }
        uint64_t *oi = a.out_ids + (uint64_t)s * a.kk, *op = a.out_pos + (uint64_t)s * a.kk;
        float *od = a.out_dist + (uint64_t)s * a.kk;
        for (uint32_t i = lane; i < a.kk; i += 32) {
            if (i < rn) {
                const uint64_t k = R[i];
                oi[i] = __ldg(a.row_ids + off + (uint32_t)k);
                od[i] = __uint_as_float((uint32_t)(k >> 32));
                op[i] = off + (uint32_t)k;
            } else {
                oi[i] = UINT64_MAX; od[i] = __int_as_float(0x7f800000); op[i] = UINT64_MAX;
            }
        }
        __syncwarp();
    }
}

}  // namespace

void launch_hnsw_search(const HnswArgs &a, int num_sms, cudaStream_t st)
{
    if (a.slots == 0) return;
    if (a.m == 0 || a.m > LGPU_HNSW_MAX_M || a.kk == 0 || a.kk > a.efp || a.efp > LGPU_HNSW_EF_MAX ||
        a.dim_pad % 64) {
        set_error("internal: HNSW search arguments out of range");
        throw Failure{LGPU_RUNTIME};
    }
    const size_t per_warp = hnsw_warp_smem(a.efp, a.kk);
    int max_smem = 0, dev = 0;
    LGPU_CUDA(cudaGetDevice(&dev));
    LGPU_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const uint32_t warps = (uint32_t)std::min<size_t>(HNSW_MAX_WARPS, (size_t)max_smem / per_warp);
    const size_t smem = warps * per_warp;
    LGPU_CUDA(cudaFuncSetAttribute(hnsw_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    LGPU_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hnsw_search_kernel, warps * 32, smem));
    const uint32_t grid = std::min<uint32_t>(ceil_div(a.slots, warps), (uint32_t)std::max(1, per_sm) * num_sms);
    launch_k(hnsw_search_kernel, dim3(grid), dim3(warps * 32), smem, st, a); LGPU_COUNT_LAUNCH();
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
