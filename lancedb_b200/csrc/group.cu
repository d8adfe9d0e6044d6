// group.cu -- batch preparation between the coarse step and the scan: regroup the
// B x nprobes probe slots by partition so the scan kernel can process, per partition,
// groups of up to 8 queries against one read of that partition's codes.  This is the
// structural change versus the reference, which plans and runs each query vector
// independently (rust/lancedb/src/table/query.rs:201-215, 334-381: "B independent
// plans + UnionExec"); all of it is index arithmetic and exact.
#include "kernels.cuh"

namespace lgpu {

namespace {

__device__ __forceinline__ uint64_t pad4(uint64_t n) { return (n + 3) & ~3ull; }

// one thread per query: count probes per partition, lay the query's distance segments
// out back to back (each padded to 4 floats).  Two launches: `first` handles every query's NEAREST probe only, the
// second the others, so that inside a partition the queries for which it is the nearest come first in the query
// list -- they end up in the partition's first tile group, and those groups are scanned first (tile_desc_kernel):
// the filter scan's per-query thresholds settle on each query's best partition before the bulk of its tiles run.
__global__ void group_count_kernel(GroupArgs a, int first)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    if (a.gate && *a.gate == 0) return;
    if (first) {
        const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
        if (q >= a.B) return;
        const bool take = !a.only || a.only[q];         // fix-up pass: only flagged queries get tiles
        const uint32_t slot = q * a.nprobes;
        const uint64_t pp = a.probes[slot];
        a.slot_pos[slot] = (take && pp < a.nlist) ? atomicAdd(&a.part_cnt[(uint32_t)pp], 1u) : 0xffffffffu;
        return;
    }
    // a warp per query, a lane per probe (32 at a time): the loads and atomics of a query's probes are in flight
    // together (one thread per query walked them one after the other: 20 dependent round trips), and the
    // segment offsets come from a warp scan
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= a.B) return;
    const bool take = !a.only || a.only[q];
    uint64_t off = 0, rows = 0;
    for (uint32_t j0 = 0; j0 < a.nprobes; j0 += 32) {
        const uint32_t j = j0 + lane;
        const bool in = j < a.nprobes;
        const uint32_t slot = q * a.nprobes + (in ? j : 0u);
        // a query with fewer than nprobes finite centroid distances (NaN / Inf input, zero cosine query)
        // leaves UINT64_MAX in its unused probe slots: those behave as empty partitions
        const uint64_t pp = in ? a.probes[slot] : UINT64_MAX;
        const bool valid = pp < a.nlist;
        const uint32_t p = valid ? (uint32_t)pp : 0u;
        const uint32_t n = valid ? a.part_n[p] : 0u;
        if (in && j > 0) a.slot_pos[slot] = (take && valid) ? atomicAdd(&a.part_cnt[p], 1u) : 0xffffffffu;
        const uint64_t mine = pad4(n);
        uint64_t pre = mine;                                // inclusive warp scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += t;
        }
        if (in) a.seg_local[slot] = off + pre - mine;
        off += __shfl_sync(0xffffffffu, pre, 31);
        uint64_t r = n;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        rows += r;
    }
    if (lane == 0) {
        a.qtot[q] = off;
        if (!a.only) atomicAdd(a.scanned_rows, (unsigned long long)rows);
    }
}

// single CTA: exclusive scans over queries (segment bases) and partitions (query-list and tile offsets).  Every thread
// sums a contiguous run of elements, one 1024-wide block scan combines the runs, the thread then writes its run back:
// one block scan per array whatever B / nlist are (a chunked form needs one per chunk).
template <class Get, class Put>
__device__ __forceinline__ uint64_t block_exclusive_scan(uint32_t n, uint64_t *s_part, int tid, Get &&get, Put &&put)
{
    const uint32_t per = (n + 1023) / 1024;
    const uint32_t b = min(n, (uint32_t)tid * per), e = min(n, b + per);
    uint64_t sum = 0;
    // runs of up to 16 elements are read into registers first, all loads in flight (a rolled `sum += get(i)` waited for
    // one L2 round trip per element, twice per array), and written back from the registers
    constexpr int RUN = 16;
    uint64_t v[RUN];
    const bool in_regs = per > 4 && per <= RUN;              // short runs: the rolled loop is cheaper than 16 predicated slots
    if (in_regs) {
#pragma unroll
        for (int j = 0; j < RUN; j++) v[j] = b + j < e ? get(b + j) : 0ull;
#pragma unroll
        for (int j = 0; j < RUN; j++) sum += v[j];
    } else {
        for (uint32_t i = b; i < e; i++) sum += get(i);
    }
    // warp scan by shuffles, then the 32 warp totals by warp 0: three barriers per array (the shared-memory
    // Hillis-Steele form took twenty)
    const int lane = tid & 31, w = tid >> 5;
    uint64_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_part[w] = inc;
    __syncthreads();
    if (w == 0) {
        uint64_t v = s_part[lane], wi = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        s_part[32 + lane] = wi - v;                        // exclusive prefix of the warp totals
        if (lane == 31) s_part[64] = wi;                    // grand total
    }
    __syncthreads();
    uint64_t run = s_part[32 + w] + inc - sum;
    if (in_regs) {
#pragma unroll
        for (int j = 0; j < RUN; j++) { if (b + j < e) put(b + j, run); run += v[j]; }
    } else {
        for (uint32_t i = b; i < e; i++) { const uint64_t x = get(i); put(i, run); run += x; }
    }
    const uint64_t total = s_part[64];
    __syncthreads();
    return total;
}

__global__ void group_scan_kernel(GroupArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    __shared__ uint64_t s_part[1024];
    const int tid = threadIdx.x;
    if (a.gate && *a.gate == 0) {                       // nothing flagged: no tiles for the exact kernel
        if (tid == 0) { *a.total_tiles = 0; *a.tile_counter = 0; }
        return;
    }
    // queries: qtot -> exclusive prefix (in place)
    block_exclusive_scan(a.B, s_part, tid, [&](uint32_t i) { return a.qtot[i]; }, [&](uint32_t i, uint64_t v) { a.qtot[i] = v; });
    // partitions: query-list offsets, then tile offsets
    block_exclusive_scan(a.nlist, s_part, tid, [&](uint32_t p) { return (uint64_t)a.part_cnt[p]; },
                         [&](uint32_t p, uint64_t v) { a.qlist_off[p] = (uint32_t)v; });
    // tiles are numbered in two classes: A = the first query group of every probed partition (all its row blocks),
    // B = the remaining groups; both partition-major
    const uint64_t tiles_a = block_exclusive_scan(
        a.nlist, s_part, tid,
        [&](uint32_t p) { return a.part_cnt[p] ? (uint64_t)scan_nrb(a.part_n[p], a.rows_tile) : 0ull; },
        [&](uint32_t p, uint64_t v) { a.tile_off[p] = (uint32_t)v; });
    const uint64_t tiles_b = block_exclusive_scan(
        a.nlist, s_part, tid,
        [&](uint32_t p) {
            const uint32_t groups = (a.part_cnt[p] + SCAN_G - 1) / SCAN_G;
            return groups > 1 ? (uint64_t)(groups - 1) * scan_nrb(a.part_n[p], a.rows_tile) : 0ull;
        },
        [&](uint32_t p, uint64_t v) { a.tile_off_b[p] = (uint32_t)(tiles_a + v); });
    if (tid == 0) {
        a.tile_off[a.nlist] = (uint32_t)tiles_a;
        a.tile_off_b[a.nlist] = (uint32_t)(tiles_a + tiles_b);
        *a.total_tiles = (uint32_t)(tiles_a + tiles_b);
        *a.tile_counter = 0;
    }
}

__global__ void group_fill_kernel(GroupArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    if (a.gate && *a.gate == 0) return;
    uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= a.B * a.nprobes) return;
    uint32_t q = slot / a.nprobes;
    a.seg_off[slot] = a.qtot[q] + a.seg_local[slot];
    if (a.slot_pos[slot] != 0xffffffffu)           // (implies a valid partition id, see group_count_kernel)
        a.qlist[a.qlist_off[(uint32_t)a.probes[slot]] + a.slot_pos[slot]] = slot;
}

// 8 threads per tile (one per query slot of the group): tile t -> (partition, query group, row block),
// Tiles are numbered partition-major.
__global__ void tile_desc_kernel(GroupArgs a)
{
    pdl_entry();                                       // PDL: let the next grid in, wait for the previous one
    if (a.gate && *a.gate == 0) return;
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t t = gid / SCAN_G, g = gid % SCAN_G;
    const uint32_t total = *a.total_tiles;
    if (t >= total || t >= a.max_tiles) return;
    const bool class_a = t < a.tile_off[a.nlist];
    const uint32_t *off = class_a ? a.tile_off : a.tile_off_b;
    uint32_t lo = 0, hi = a.nlist - 1;          // smallest p with off[p+1] > t
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (off[mid + 1] > t) hi = mid; else lo = mid + 1;
    }
    const uint32_t p = lo;
    const uint32_t n_p = a.part_n[p];
    const uint32_t nrb = scan_nrb(n_p, a.rows_tile), rbr = scan_rb_rows(n_p, nrb);
    const uint32_t local = t - off[p];
    const uint32_t grp = class_a ? 0u : 1u + local / nrb, rb = class_a ? local : local % nrb;
    const uint32_t ng = min((uint32_t)SCAN_G, a.part_cnt[p] - grp * SCAN_G);
    const uint32_t row0 = rb * rbr;
    TileDesc *d = a.tile_desc + t;
    if (g == 0) {
        d->p = p; d->row0 = row0; d->nrows = row0 < n_p ? min(rbr, n_p - row0) : 0; d->ng = ng;
        d->n_p = n_p; d->npad = a.part_npad[p];
        d->code_base8 = (uint32_t)(a.code_base[p] >> 3); d->part_off32 = (uint32_t)a.part_off[p];
    }
    if (g < ng) {
        const uint32_t e = a.qlist[a.qlist_off[p] + grp * SCAN_G + g];
        d->q[g] = e / a.nprobes;
        d->slot[g] = e;
        d->out[g] = (uint32_t)a.seg_off[e];
    } else {
        d->q[g] = 0xffffffffu;
        d->slot[g] = 0;
        d->out[g] = 0;
    }
}

}  // namespace

void launch_group(const GroupArgs &a, cudaStream_t st)
{
    if (a.B == 0) return;
    LGPU_CUDA(cudaMemsetAsync(a.part_cnt, 0, sizeof(uint32_t) * a.nlist, st));
    if (!a.only) LGPU_CUDA(cudaMemsetAsync(a.scanned_rows, 0, sizeof(unsigned long long), st));
    launch_k(group_count_kernel, dim3((a.B + 127) / 128), dim3(128), 0, st, a, 1); LGPU_COUNT_LAUNCH();
    launch_k(group_count_kernel, dim3((a.B + 3) / 4), dim3(128), 0, st, a, 0); LGPU_COUNT_LAUNCH();       // a warp per query
    launch_k(group_scan_kernel, dim3(1), dim3(1024), 0, st, a); LGPU_COUNT_LAUNCH();
    uint32_t slots = a.B * a.nprobes;
    launch_k(group_fill_kernel, dim3((slots + 255) / 256), dim3(256), 0, st, a); LGPU_COUNT_LAUNCH();
    if (a.tile_desc && a.max_tiles) {
        uint64_t threads = (uint64_t)a.max_tiles * SCAN_G;
        launch_k(tile_desc_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st, a); LGPU_COUNT_LAUNCH();
    }
    LGPU_CUDA(cudaGetLastError());
}

}  // namespace lgpu
