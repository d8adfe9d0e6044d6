// kernels.cuh -- kernel argument blocks and host launchers shared by the C-ABI layer.
#pragma once

#include "common.cuh"

#include <cuda_fp16.h>

namespace lgpu {

// ---------------- scan (K2+K3) geometry ------------------------------------------
constexpr int SCAN_G = 8;                         // queries per tile
constexpr uint32_t SCAN_ROWS_TILE_MID = 4 * 32 * 12;   // exact kernel (scan2.cu): 2 x 128 scanner threads x 12 rows
constexpr uint32_t SCAN3_ROWS_TILE = 8 * 32 * 6;       // filter kernel (scan3.cu): 256 scanner threads x 6 rows
constexpr int SCAN_LUT_HALF = 32768;              // exact kernel: [256 c][8 s][4 g] f32
constexpr int SCAN_LUT_BYTES = 2 * SCAN_LUT_HALF; // [2 h] halves

__host__ __device__ __forceinline__ uint32_t scan_nrb(uint32_t n, uint32_t rows_tile)
{
    return (n + rows_tile - 1) / rows_tile;
}
__host__ __device__ __forceinline__ uint32_t scan_rb_rows(uint32_t n, uint32_t nrb)
{
    return nrb ? (((n + nrb - 1) / nrb + 31u) & ~31u) : 0u;
}

// One scan tile, precomputed by the regroup step (group.cu) so the persistent scan CTAs fetch a tile with a
// single 128-byte read: partition p, rows [row0, row0+nrows), ng (1..8) queries q[] (probe slots slot[]) whose
// distances go to dist_out + out[g].  ng == 0 marks "no tile" inside the kernel's shared-memory copy.
struct alignas(16) TileDesc {
    uint32_t p, row0, nrows, ng;
    uint32_t q[SCAN_G];
    uint32_t slot[SCAN_G];        // probe slot (q * nprobes + j) of each query
    uint32_t out[SCAN_G];         // offset (floats) of the slot's distance segment; sub-batches keep it < 2^32
    // the partition's constants, copied in by the regroup step: read from the shared-memory copy of the descriptor, a
    // tile's first code-word load and its row-constant load go out at once instead of behind a dependent global read
    uint32_t n_p, npad;           // rows / padded rows of partition p
    uint32_t code_base8;          // code_base[p] / 8
    uint32_t part_off32;          // part_off[p] (row position of the partition's first row)
};
static_assert(sizeof(TileDesc) == 128, "TileDesc layout");

// The tiles of one chunk of consecutive partitions [p0, p0 + n) of a row-major IVF index whose codes are staged through
// HBM (IVF_SQ, IVF_RQ and binary IVF_FLAT with codes in pinned host memory): the regroup numbers each partition's tiles
// in two contiguous ranges, so the chunk's tiles are [a[0], a[n]) and [b[0], b[n]) (a = tile_off + p0, b = tile_off_b +
// p0, device).  The staged rows start at row `row_shift` of the index: a tile's row r of partition p is read at
// part_off[p] + r - row_shift of the staging buffer, while the per-row terms keep their absolute row.  a == nullptr: the
// whole tile queue (*total_tiles tiles) over the index's own rows.
struct TileRange {
    const uint32_t *a, *b;
    uint32_t n;
    uint32_t row_shift;
};
// tiles the scan claims: the chunk's, or the whole queue's
__device__ __forceinline__ uint32_t tile_range_total(const TileRange &r, const uint32_t *total_tiles)
{
    return r.a ? (r.a[r.n] - r.a[0]) + (r.b[r.n] - r.b[0]) : *total_tiles;
}
// the tile descriptor of claim t < tile_range_total
__device__ __forceinline__ uint32_t tile_range_at(const TileRange &r, uint32_t t)
{
    if (!r.a) return t;
    const uint32_t a0 = r.a[0], na = r.a[r.n] - a0;
    return t < na ? a0 + t : r.b[0] + (t - na);
}

// one surviving row of the filter scan's candidate mode
struct alignas(16) CandRec {
    float lb;                     // lower bound L of the row's distance
    uint32_t p, row;              // partition and row inside it
    uint32_t pad;
};
constexpr uint32_t CAND_NO_THR = 0xffffffffu;
constexpr uint32_t CAND_TOPK_MAX = 128;      // largest k (or k * refine_factor) the candidate mode serves (LGPU_CAND_KMAX lowers it)
constexpr uint32_t CAND_CAP_MAX = 2048;      // largest per-query candidate list

struct ScanArgs {
    // index (device)
    const float *centroids;       // [nlist][dim]
    const float *cb_tiled;        // [nch][256][8][dsub]
    const unsigned char *codes;   // skewed code streams, see retile.cu
    const uint64_t *code_base;    // [nlist] byte offset of partition p's stream block
    const uint32_t *part_n;       // [nlist]
    const uint32_t *part_npad;    // [nlist] rows rounded up to 32
    uint32_t dim, m, nch, metric, nlist;
    uint32_t rows_tile;           // SCAN_ROWS_TILE_MID (exact) or SCAN3_ROWS_TILE (filter)
    unsigned long long fzero2;    // packed (+0.f, +0.f); opaque to ptxas on purpose (scan_common.cuh)
    // batch (device)
    const float *queries;         // [B][dim] (normalised for cosine)
    const uint32_t *total_tiles;  // [1]
    uint32_t *tile_counter;       // [1], zeroed before launch
    float *dist_out;
    const TileDesc *tile_desc;    // [total_tiles]
    const uint32_t *gate;         // optional [1] (exact kernel as fix-up pass): 0 = nothing to do
    // filter pass (scan3.cu, tables.cu); unused by the exact kernel
    const uint4 *qt;              // [B][nch][256] x (8 x u16): quantised per-query tables, rotated (tables.cu)
    const float *qt_step;         // [B] quantisation step
    const float *qt_base;         // [B] sum_i min_i (- (m - 1) for dot)
    const float *probe_A;         // [B*nprobes] |q - c_p|^2 - |q|^2   (nullptr for dot)
    const float *row_R;           // [nrows] 2 * codeword(row) . c_p  (nullptr for dot)
    const uint64_t *part_off;     // [nlist+1]
    // filter pass, candidate mode (cand != nullptr): instead of one f32 per (row, query) in dist_out, the scanners
    // keep a running per-query threshold and append only the rows that can still be among the exact top-k
    uint32_t nprobes, topk;       // probe slots per query; k (the number of neighbours the threshold is for)
    uint32_t *thr;                // [B] ordered-uint key (f32_key) of tau_q, CAND_NO_THR = none yet; atomicMin
    const float *slack;           // [B] scale (W + 2E): a row survives iff L <= tau_q + slack_q
    uint32_t *cand_cnt;           // [B] appended candidates (may exceed cand_cap: the overflow is dropped and flagged)
    CandRec *cand;                // [B][cand_cap]
    uint32_t cand_cap;
    uint32_t *cand_key;           // [B][cand_cap] f32_key(lb) of every appended record, 0xffffffff where none is yet: what
                                  // the scanners re-read to tighten tau_q from the list itself (scan3.cu)
    uint32_t *cand_last;          // [B] list length at the query's last list-based tightening
};
bool scan_dsub_supported(uint32_t dsub);
// exact kernel (scan2.cu): residual -> f32 table chunk -> sequential code scan, bit-identical to the oracle;
// needs a.tile_desc built with rows_tile == SCAN_ROWS_TILE_MID
void launch_scan2(const ScanArgs &a, uint32_t dsub, int grid, cudaStream_t st);
// filter kernel (scan3.cu): lower bounds from 16-bit per-query tables; rows_tile == SCAN3_ROWS_TILE
void launch_scan3(const ScanArgs &a, int grid, cudaStream_t st);

// ---------------- IVF_SQ scan (sq_scan.cu) ----------------------------------------------
constexpr uint32_t SQ_ROWS_TILE = 256;            // rows per tile: 8 warps x 32 rows
constexpr uint32_t SQ_K_CHUNK = 64;               // code bytes per K step of a warp; stored rows are padded to it
struct SqScanArgs {
    const uint8_t *codes;         // [nrows][dim_pad] row codes, partitions contiguous, zero padding
    const uint32_t *xx;           // [nrows] sum of the squared codes of each row
    const uint8_t *qcodes;        // [B][dim_pad] query codes (launch_sq_encode)
    const uint32_t *qq;           // [B]
    uint32_t dim_pad;
    const uint32_t *total_tiles;  // [1]
    uint32_t *tile_counter;       // [1], zeroed before launch
    const TileDesc *tile_desc;    // built with rows_tile == SQ_ROWS_TILE
    float *dist_out;              // segment of slot e at out[e]: (float) sum_i (k_i - q_i)^2 of row r at out[e] + r
    int out_u32;                  // 1: write the exact u32 sums instead (lgpu_debug_sq_distances)
    TileRange range;              // optional: one staged chunk's tiles, `codes` its staging buffer
};
// qc[b] = the codes of query b (sat_u8(((double)q - lo) * 255 / (hi - lo)), zero-padded to dim_pad), qq[b] = |qc[b]|^2
void launch_sq_encode(const float *Q, uint32_t B, uint32_t dim, uint32_t dim_pad, double lo, double hi, uint8_t *qc,
                      uint32_t *qq, cudaStream_t st);
// xx[r] = sum of the squared codes of row r of codes [n][dim_pad]
void launch_sq_row_norms(const uint8_t *codes, uint64_t n, uint32_t dim_pad, uint32_t *xx, cudaStream_t st);
void launch_sq_scan(const SqScanArgs &a, int grid, cudaStream_t st);

// ---------------- IVF_HNSW_SQ graph search (hnsw_scan.cu) ---------------------------------
struct HnswArgs {
    const uint8_t *codes;         // IVF_SQ's [nrows][dim_pad] row codes
    const uint8_t *qcodes;        // [B][dim_pad] query codes (launch_sq_encode)
    uint32_t dim_pad;
    const uint64_t *probes;       // [slots] partition of each probe slot (>= nlist: unused)
    uint32_t slots, nprobes, nlist;
    const uint64_t *part_off;     // [nlist + 1]
    const uint64_t *row_ids;
    const uint8_t *levels;        // the graph, lgpu_ivf_hnsw_sq_desc's layout
    const uint32_t *adj0, *upper_index, *upper_adj, *entry;
    const uint8_t *top_level;
    uint32_t m, efp, kk;          // efp: W's capacity, kk: R's (kk <= efp <= LGPU_HNSW_EF_MAX)
    int has_lower, has_upper;     // the row filter R applies
    float lower, upper;
    const uint32_t *allow;
    uint64_t allow_bits;
    const uint32_t *only;         // optional [B]: slots of other queries are skipped
    uint32_t *counter;            // [1], zeroed before launch
    uint64_t *out_ids;            // [slots][kk]: R of each slot, ascending by (d, position), padded with UINT64_MAX
    float *out_dist;              //   and +inf
    uint64_t *out_pos;            //   (the rows' global positions, for refine)
};
void launch_hnsw_search(const HnswArgs &a, int num_sms, cudaStream_t st);

// ---------------- IVF_RQ scan (rq_scan.cu) ----------------------------------------------
constexpr uint32_t RQ_ROWS_TILE = 256;            // rows per tile: 8 warps x 32 rows
constexpr uint32_t RQ_K_BITS = 256;               // code bits per K step (one b1 MMA); stored rows are padded to it
struct alignas(16) RqSlot {                       // one probe slot's 4-bit query grid
    float lo, delta;                              // min q', fl(fl(max q' - lo) / 15)
    uint32_t S;                                   // sum of the 4-bit codes u
    float qq;                                     // lance_l2(rq, rc_p)
};
struct RqScanArgs {
    const uint32_t *codes;        // [nrows][wpr] sign bits, partitions contiguous, zero padding
    const float *add, *scale;     // [nrows] |o|^2, -2 |o|^2 / sum |o_i|
    const uint32_t *popc;         // [nrows] set bits of each row
    const uint32_t *planes;       // [slots][4][wpr] bit-planes of u (launch_rq_planes)
    const RqSlot *slots;          // [slots]
    uint32_t dim, wpr;            // wpr = 32-bit words per row (dim_pad / 32, a multiple of 8)
    int cosine;                   // report fl(0.5 est)
    const uint32_t *total_tiles;  // [1]
    uint32_t *tile_counter;       // [1], zeroed before launch
    const TileDesc *tile_desc;    // built with rows_tile == RQ_ROWS_TILE; slot[] addresses planes / slots
    float *dist_out;              // segment of slot e at out[e]: the estimate of row r at out[e] + r
    int out_ip;                   // 1: write the exact u32 ip = sum_i b_i u_i instead (lgpu_debug_rq_distances)
    TileRange range;              // optional: one staged chunk's tiles, `codes` its staging buffer
};
// out[v][i] = lance_dot(P row i, x[v]): the rotation of n vectors by P [dim][dim]
void launch_rq_rotate(const float *P, const float *x, uint32_t n, uint32_t dim, float *out, cudaStream_t st);
// per probe slot e (query e / nprobes, partition probes[e]; slots without a partition are skipped): the 4-bit grid of
// q' = rq - rc_p as planes [e][4][wpr] and slot_out[e]
void launch_rq_planes(const float *rq, const float *rc, const uint64_t *probes, uint32_t slots, uint32_t nprobes,
                      uint32_t nlist, uint32_t dim, uint32_t wpr, uint32_t *planes, RqSlot *slot_out, cudaStream_t st);
// clear the padding bits of codes [n][wpr] and count each row's set bits
void launch_rq_row_prep(uint32_t *codes, uint64_t n, uint32_t dim, uint32_t wpr, uint32_t *popc, cudaStream_t st);
void launch_rq_scan(const RqScanArgs &a, int grid, cudaStream_t st);

// ---------------- binary IVF_FLAT scan (ivf_ham_scan.cu) --------------------------------
constexpr uint32_t HAM_ROWS_TILE = 512;           // rows per tile: 8 warps x 32 rows x 2 passes (not tuned)
struct HamScanArgs {
    const uint8_t *rows;          // [nrows][nbytes_pad] packed rows, partitions contiguous, zero padding
    const uint32_t *row_pop;      // [nrows] popc of each row
    const uint8_t *queries;       // [B][nbytes_pad] packed queries of the sub-batch (launch_ham_pack)
    const uint32_t *qpop;         // [B]
    uint32_t nbytes_pad;          // a multiple of 32
    const uint32_t *total_tiles;  // [1]
    uint32_t *tile_counter;       // [1], zeroed before launch
    const TileDesc *tile_desc;    // built with rows_tile == HAM_ROWS_TILE; q[] addresses queries / qpop
    float *dist_out;              // segment of slot e at out[e]: popc(q XOR x) of row r at out[e] + r, as f32
    int out_u32;                  // 1: write the u32 distances instead (lgpu_debug_ivf_hamming_scan)
    TileRange range;              // optional: one staged chunk's tiles, `rows` its staging buffer
};
void launch_ivf_ham_scan(const HamScanArgs &a, int grid, cudaStream_t st);
// One chunk of a row-major IVF index's codes (rows [part_off[p0], part_off[p1]), row_bytes each, a multiple of 16) from
// pinned host memory (src: the mapped alias of the whole store) into the staging buffer dst, which holds row
// part_off[p0] at byte 0: only the partitions some probe slot scans (part_cnt[p] > 0), the others skipped at once.
// *moved (optional) += the bytes copied.  Reads the offsets and counts on the device: no host synchronisation.
void launch_codes_copy_gated(const uint8_t *src, uint8_t *dst, uint64_t row_bytes, const uint64_t *part_off,
                             const uint32_t *part_cnt, uint32_t p0, uint32_t p1, uint64_t chunk_bytes,
                             unsigned long long *moved, int num_sms, cudaStream_t st);
// probes[q][j] = j for q < B, j < nlist: every partition, for nprobes >= nlist (no coarse step, no top-nprobes select)
void launch_ham_all_probes(uint64_t *probes, uint32_t B, uint32_t nlist, cudaStream_t st);

// ---------------- 4-bit IVF_PQ scan (pq4_scan.cu) ----------------------------------------
constexpr uint32_t PQ4_ROWS_TILE = 2048;          // rows per tile: 256 threads x 2 groups of 4 rows
struct alignas(8) Pq4Slot {                       // one probe slot's table quantiser
    float qmin, qmax;
};
struct Pq4ScanArgs {
    const uint32_t *codes;        // per partition [m/2][npad] packed code bytes at byte code_base[p] (launch_pq4_relayout)
    const uint8_t *tables;        // [slots][m][16] u8 tables (launch_pq4_tables)
    const Pq4Slot *slots;         // [slots]
    uint32_t m, metric;
    const uint32_t *total_tiles;  // [1]
    uint32_t *tile_counter;       // [1], zeroed before launch
    const TileDesc *tile_desc;    // built with rows_tile == PQ4_ROWS_TILE; slot[] addresses tables / slots
    float *dist_out;              // segment of slot e at out[e]: the distance of row r at out[e] + r (padded to 4 floats)
    int out_u32;                  // 1: write the exact u32 sums S instead (lgpu_debug_pq4_sums)
};
// dynamic shared memory of the scan kernel for m sub-vectors
size_t pq4_scan_smem(uint32_t m);
// per probe slot e (query e / nprobes, partition probes[e]; slots without a partition are skipped): the u8 tables
// [e][m][16] and slot_out[e]; codebook [m][dsub][16] (element-major: element t of codeword j of sub-space i at
// (i dsub + t) 16 + j)
void launch_pq4_tables(const float *Q, const float *centroids, const float *codebook, const uint64_t *probes,
                       uint32_t slots, uint32_t nprobes, uint32_t nlist, uint32_t m, uint32_t dsub, int metric,
                       uint8_t *tables, Pq4Slot *slot_out, cudaStream_t st);
void launch_pq4_scan(const Pq4ScanArgs &a, int grid, cudaStream_t st);
// codes (layout: lgpu_codes_layout, m/2 bytes per row) -> out, per partition [m/2][part_npad[p]] at code_base[p]
void launch_pq4_relayout(const uint8_t *codes, int layout, const uint64_t *part_off, uint32_t nlist, uint64_t nrows,
                         uint32_t m, const uint64_t *code_base, const uint32_t *part_npad, uint8_t *out, cudaStream_t st);

// ---------------- tiny batches: one CTA per (query, probed partition) pair (small.cu) ----------------
struct SmallScanArgs {
    const float *centroids; const float *cb_tiled; const unsigned char *codes; const uint64_t *code_base;
    const uint32_t *part_n; const uint32_t *part_npad;
    uint32_t dim, m, nch, metric, nlist, nprobes;
    const float *queries;         // [B][dim] (normalised for cosine)
    const uint64_t *probes;       // [B*nprobes]
    uint64_t seg_stride;          // floats per probe slot in dist_out (>= the largest partition, multiple of 4)
    uint64_t *seg_off;            // [B*nprobes], written here: slot * seg_stride
    float *dist_out;
};
size_t small_scan_smem(uint32_t m, uint32_t dim);
void launch_small_scan(const SmallScanArgs &a, uint32_t dsub, uint32_t slots, cudaStream_t st);

// ---------------- batch preparation (grouping probes by partition) ----------------
struct GroupArgs {
    const uint64_t *probes;       // [B*nprobes] partition ids (u64 from the selector)
    uint32_t B, nprobes, nlist, rows_tile;
    const uint32_t *part_n;
    const uint32_t *part_npad;    // (tile descriptors) padded rows per partition
    const uint64_t *code_base;    // (tile descriptors) byte offset of each partition's code blocks, multiple of 8
    const uint64_t *part_off;     // (tile descriptors) row position of each partition's first row, < 2^32
    uint32_t *part_cnt;           // [nlist] zeroed before
    uint32_t *slot_pos;           // [B*nprobes]
    uint64_t *seg_local;          // [B*nprobes] offset inside the query's block
    uint64_t *qtot;               // [B]
    uint64_t *seg_off;            // [B*nprobes]
    uint32_t *qlist_off;          // [nlist]
    uint32_t *tile_off;           // [nlist+1] first tile of each partition's first query group (class A)
    uint32_t *tile_off_b;         // [nlist+1] first tile of each partition's remaining groups (class B, after all of A)
    uint32_t *qlist;              // [B*nprobes]
    uint32_t *total_tiles;        // [1]
    uint32_t *tile_counter;       // [1]
    unsigned long long *scanned_rows;  // [1] sum over probe slots of n_p (roofline bytes / m)
    const uint32_t *only;         // optional [B]: regroup only the flagged queries (fix-up pass)
    const uint32_t *gate;         // optional [1]: 0 = no query is flagged, the whole fix-up pass returns at once
    TileDesc *tile_desc;          // optional [max_tiles] tile descriptors for the streaming scan kernel
    uint32_t max_tiles;           // capacity of tile_desc (host bound on the tile count)
};
void launch_group(const GroupArgs &a, cudaStream_t st);

// ---------------- exact distance matrix (K1 coarse, flat v1) ----------------------
// D[q][c] for q < B, c < N.  mode 0: L2 (squared), 1: dot distance 1 - x.y,
// 2: cosine 1 - x.y/|x|/|y| (xnorm[B] = |x|, ysqrt[N] = |y| required).
// `only` (optional, [B]): rows whose flag is 0 are skipped (used by the tensor-core paths' fix-up pass).
// The stored rows C (and V, X below) are float or __half: fp16 rows are converted to f32 in registers, so the distances
// are those of the rows' exact f32 upcast, bit for bit.
template <class T>
void launch_dist_matrix(const float *Q, const T *C, uint32_t B, uint64_t N, uint32_t d, int mode,
                        const float *xnorm, const float *ysqrt, float *D, uint64_t ldD, cudaStream_t st,
                        const uint32_t *only = nullptr, const uint32_t *gate = nullptr);
// coarse step after the tensor-core GEMM, one kernel: from S[B][ld] = |x|^2 - 2 bf16(q).bf16(x) (N columns) to the k
// columns with the smallest EXACT l2 distance (lance lane order), ascending by (distance, column); flags[q] = 1 when
// the candidate band overflowed and the caller must redo the query with the exact kernels
void launch_coarse_finish(const float *S, uint64_t ld, uint32_t B, uint32_t N, const float *Q, const float *C,
                          const float *qn2, const float *qerr, float xmax, float xerr, uint32_t d, uint32_t k,
                          uint64_t *out_ids, float *out_dist,
                          uint32_t *out_cnt, uint32_t *flags, uint32_t *gate, cudaStream_t st,
                          const uint64_t *list_pos = nullptr, const uint32_t *list_cnt = nullptr);
// list mode (list_pos / list_cnt given, N == ld == the list capacity): S[q] holds the list_cnt[q] scores the GEMM's
// filtering epilogue admitted for query q and list_pos[q] their columns; a list longer than its capacity flags the query
// row norms |x| = sqrt(dot(x,x)) in lance order; out[n]
template <class T>
void launch_row_norms(const T *X, uint64_t n, uint32_t d, float *out, cudaStream_t st);
// out[q] = x[q] / |x[q]|
void launch_normalize(const float *X, uint32_t B, uint32_t d, float *out, cudaStream_t st);
// exact distances of (query, stored row) pairs: out[q][c] = dist(Q[q], V[pos[q][c]]),
// pos == UINT64_MAX => +inf
template <class T>
void launch_pair_distance(const float *Q, const T *V, const uint64_t *pos, uint32_t B, uint32_t nc,
                          uint32_t d, int metric, float *out, cudaStream_t st);
// the same out[q][c], bit for bit, with the rows in pinned host memory: V is their mapped device alias, rows `stride`
// floats apart (a multiple of 4, 16-byte aligned).  Reads whole rows over PCIe into shared memory (dist.cu)
void launch_refine_host(const float *Q, const float *V, uint32_t stride, const uint64_t *pos, uint32_t B, uint32_t nc,
                        uint32_t d, int metric, float *out, int num_sms, cudaStream_t st);

// ---------------- top-k select (K4) ------------------------------------------------
constexpr uint32_t SELECT_KMAX = 2048;
// one top-k entry as it crosses NVLink in the partition-sharded search (SURVEY.md 8e): a single ncclAllGather of
// [B][k] of these per rank, consumed in place by the merge (select mode 2)
struct alignas(16) TopkRecord {
    uint64_t id;      // _rowid, UINT64_MAX = unused slot
    float dist;       // _distance
    uint32_t pad;
};
static_assert(sizeof(TopkRecord) == 16, "TopkRecord layout");
struct SelectArgs {
    int mode;                     // 0: IVF distance segments, 1: dense row (ids = column / col_ids),
                                  // 2: strided candidate lists with per-entry ids
    // mode 0
    const float *dist;            // dist_out
    const uint64_t *seg_off;      // [B*nprobes]
    const uint64_t *probes;       // [B*nprobes]
    uint32_t nprobes, nlist;      // probe ids >= nlist are unused slots
    const uint32_t *part_n;
    const uint64_t *part_off;     // [nlist+1] storage row offsets
    const uint64_t *row_ids;      // [nrows]
    // mode 1 / 2
    const float *dense;           // values
    uint64_t ncols;               // candidates per query
    uint64_t row_stride;          // mode 1: ld; mode 2: stride between queries
    uint64_t inner, outer_stride; // mode 2: col -> (col/inner)*outer_stride + q*row_stride + col%inner
    const uint64_t *col_ids;      // mode 1: optional id per column (NULL => col_base + column index)
    uint64_t col_base;            // mode 1: the id of column 0 when col_ids is NULL (a chunk of a streamed column)
    const uint64_t *cand_ids;     // mode 2: id per entry (same addressing as dense)
    const uint64_t *cand_pos;     // mode 2: optional pos per entry
    const uint32_t *ncols_q;      // mode 2: optional [B] candidates of each query (<= ncols)
    const uint32_t *list_cnt;     // mode 2: optional [ncols / inner][B] valid entries of list l (columns l * inner ..)
                                  // of query q at l * B + q; the entries of a list past its count are not read
    const TopkRecord *cand_rec;   // mode 2: optional packed (id, dist) entries instead of dense + cand_ids
    // common
    uint32_t B, k;
    int has_lower, has_upper;
    float lower, upper;
    uint64_t *out_ids;            // [B][k]
    float *out_dist;              // [B][k]
    uint32_t *out_count;          // [B]
    TopkRecord *out_rec;          // optional [B][k]: packed output instead of out_ids / out_dist
    uint64_t *out_pos;            // optional [B][k] storage position (mode 0) / column (mode 1)
    const uint32_t *only;         // optional [B]: queries whose flag is 0 are left untouched
    const uint32_t *gate;         // optional [1]: 0 = no query is flagged (the kernel returns at once)
    // prefilter (query.rs:489-507): optional row-id allow-list bitmap; a candidate whose id has bit 0 (or is
    // >= allow_bits) is dropped before it can enter the top-k
    const uint32_t *allow;
    uint64_t allow_bits;
    // k > SELECT_KMAX (select_large.cu): device scratch of at least select_large_scratch_bytes(B, k, out_pos != NULL)
    void *scratch;
    size_t scratch_bytes;
};
// k <= SELECT_KMAX: select.cu; SELECT_KMAX < k <= LGPU_K_MAX: launch_select_large
void launch_select(const SelectArgs &a, cudaStream_t st);
// the global-memory radix top-k (select_large.cu): same contract as the small selects, any k in (SELECT_KMAX, LGPU_K_MAX]
void launch_select_large(const SelectArgs &a, cudaStream_t st);
size_t select_large_scratch_bytes(uint32_t B, uint32_t k, bool pos);
// flags[q] = cnt[q] < k (maximum_nprobes widening: the queries that did not find k rows)
void launch_count_below(const uint32_t *cnt, uint32_t B, uint32_t k, uint32_t *flags, cudaStream_t st);
// rec[i] = (ids[i], dist[i]) for i < n
void launch_pack_records(const uint64_t *ids, const float *dist, uint64_t n, TopkRecord *out, cudaStream_t st);

// ---------------- live-row bitmaps of handles with deleted rows (rowmask.cu) ----------------
// *out = max(*out, ids[0..n))
void launch_rowmask_max(const uint64_t *ids, uint64_t n, unsigned long long *out, cudaStream_t st);
// set the bits of ids[0..n) (ids null: of first .. first + n - 1) below nbits
void launch_rowmask_set(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t first, uint64_t n, cudaStream_t st);
// *count += the rows i < n whose id (ids[i], ids null: i) is below nbits, set in mark and clear in live
void launch_rowmask_revived(const uint32_t *mark, const uint32_t *live, uint64_t nbits, const uint64_t *ids, uint64_t n,
                            unsigned long long *count, cudaStream_t st);
// clear the bits of ids[0..n) below nbits; *count += the bits this call found set
void launch_rowmask_clear(uint32_t *bits, uint64_t nbits, const uint64_t *ids, uint64_t n, unsigned long long *count,
                          cudaStream_t st);
// out[i] = a[i] & b[i] for i < words
void launch_rowmask_and(const uint32_t *a, const uint32_t *b, uint64_t words, uint32_t *out, cudaStream_t st);

// ---------------- tensor-core shortlist (gemm.cu) ------------------------------------
bool gemm_shape_supported(uint32_t d);
// X f32 [n][d] -> bf16 [n][d]; norm2[n] = |x|^2 (f32) if norm2 != nullptr; err[n] = |bf16(x) - x| if err != nullptr
void launch_to_bf16(const float *X, uint64_t n, uint32_t d, void *Xb, float *norm2, cudaStream_t st, float *err = nullptr);
// the operands of the fp16 form (F16Dist): queries Q f32 [B][d] -> Qh fp16 [B][d], qn2[q] = |q|^2 (f32),
// qerr[q] = |h(q) - q| (inf when a component overflows fp16); stored fp16 rows X [n][d] -> norm2[n] = |x|^2 (f32),
// err[n] = |h(x) - x| (h: the value the MMA consumes)
void launch_to_f16(const float *Q, uint32_t B, uint32_t d, void *Qh, float *qn2, float *qerr, cudaStream_t st);
void launch_f16_row_terms(const void *X, uint64_t n, uint32_t d, float *norm2, float *err, cudaStream_t st);
// E_q, the error band of the tensor-core scores: |S[q][x] - (|q - x|^2 - |q|^2)| <= E_q for every row x of the operand,
// S[q][x] = |x|^2 - 2 bf16(q).bf16(x) (f32 accumulation), with r_q = |bf16(q) - q| (qerr), r_X = max_x |bf16(x) - x|
// (xerr) and xmax >= max_x |x|:
//   E_q = 2 ((|q| + r_q) r_X + r_q xmax)(1 + 2^-10) + 4 d 2^-24 (|q| + xmax)^2.
// bf16(q).bf16(x) - q.x = bf16(q).(bf16(x) - x) + (bf16(q) - q).x and |bf16(q)| <= |q| + r_q; 2^-10 covers the f32
// arithmetic of the r's and of E_q itself, the last term the f32 sums (|x|^2, the accumulation, the exact re-score).
// Both operands round: r can reach 2^-8 of the norm each, so E_q reaches ~2^-6 |q| xmax on adversarial data.  Every
// consumer (band check, sample thresholds, coarse finishing kernel) takes its band from here.  A non-finite query (or
// one whose |q|^2 overflows) makes E_q inf or NaN: every consumer then hands the query to the exact kernels.  The
// operand's xmax and xerr are finite by construction: an operand without a finite bound gets no tensor-core copy.
__device__ __forceinline__ float tc_band(float qnorm2, float qerr, float xmax, float xerr, uint32_t d)
{
    const float qn = sqrtf(qnorm2), s = qn + xmax;
    return 2.0f * 1.0009765625f * ((qn + qerr) * xerr + qerr * xmax) + 4.0f * (float)d * 5.9604645e-8f * s * s;
}
// out[q][x] = xnorm2[x] - 2 * bf16(Q[q]) . bf16(X[x])   (wgmma + TMA), q < B, x < N; f16: Qb and Xb are fp16
// (F16Dist, gemm.cu)
// optional filtering epilogue: instead of writing the dense score matrix, append the columns whose score
// is <= thr[q] to the query's candidate list (count may exceed cap: those appends are dropped)
struct GemmFilter {
    const float *thr;             // [B]; nullptr = dense output
    uint32_t *count;              // [B], zeroed by the caller
    uint64_t *cand_pos;           // [B][cap] column (storage row) of each candidate
    uint64_t *cand_ids;           // [B][cap] its id (gemm_filter_id)
    const uint64_t *col_ids;      // optional
    uint64_t col_base;            // without col_ids, the id of column 0 (a chunk of a streamed column)
    uint32_t cap;
    float *cand_s;                // optional [B][cap]: the admitted score itself (coarse step: second-level threshold)
    // optional row filter: a column passing the threshold is admitted only if the bit of its id (gemm_filter_id) is
    // set, id < allow_bits (a prefilter, deleted rows)
    const uint32_t *allow;
    uint64_t allow_bits;
};
// the id of column x: col_ids[x], or col_base + x
__device__ __forceinline__ uint64_t gemm_filter_id(const GemmFilter &f, uint64_t x)
{
    return f.col_ids ? f.col_ids[x] : f.col_base + x;
}
// whether column x passes the row filter of a filter that has one (tested only for columns under the threshold)
__device__ __forceinline__ bool gemm_filter_admits(const GemmFilter &f, uint64_t x)
{
    const uint64_t id = gemm_filter_id(f, x);
    return id < f.allow_bits && ((__ldg(f.allow + (id >> 5)) >> (id & 31)) & 1u);
}
void launch_gemm_dist(const void *Qb, const void *Xb, const float *xnorm2, uint32_t B, uint64_t N, uint32_t d,
                      float *out, uint64_t ld_out, int num_sms, cudaStream_t st, const GemmFilter *filter = nullptr,
                      bool f16 = false);
// the binary (Hamming) form of the same kernel: the GemmFilter fields plus popc(q) of every query
struct HamFilter : GemmFilter {
    const int *qpop;              // [B]
};
// out[q][x] = popc(Q[q] XOR X[x]) as f32 (exact), Q / X packed bits [B | N][nbytes_pad] (zero-padded to a multiple of
// 32 bytes), xpop / qpop = popc of each row (wgmma m64n128k256 .and.popc + TMA).  With a filter (thr, count, cand_pos,
// cand_ids, cand_s, cap required): nothing dense is written; every column with distance <= thr[q] is appended as
// (position, id, distance) to the query's list (count may exceed cap: those appends are dropped).
void launch_ham_gemm(const void *Qp, const void *Xp, const uint32_t *xpop, const uint32_t *qpop, uint32_t B, uint64_t N,
                     uint32_t nbytes_pad, float *out, uint64_t ld_out, int num_sms, cudaStream_t st,
                     const GemmFilter *filter = nullptr);

// ---------------- binary vectors, SIMT side (hamming.cu) --------------------------------
// dst[r] = src row r (src rows `src_stride` bytes apart, nbytes used) zero-padded to nbytes_pad; pop[r] = its popcount.
// dst null: pop alone (rows already packed: nbytes = nbytes_pad)
void launch_ham_pack(const uint8_t *src, uint64_t src_stride, uint32_t nbytes, uint64_t n, uint8_t *dst,
                     uint32_t nbytes_pad, uint32_t *pop, cudaStream_t st);
// D[q][x] = popc(Q[q] XOR X[x]) as f32 for x < N (LOP3 + POPC over 32-bit words; rows padded to a multiple of 32
// bytes).  With qlist / qcount (device): only the *qcount queries qlist[0..) are computed (the fix-up of overflowed
// queries; nothing runs when the count is 0), otherwise queries 0..B-1.
void launch_ham_dense(const uint8_t *Q, const uint8_t *X, uint32_t B, uint64_t N, uint32_t nbytes_pad, float *D,
                      uint64_t ldD, int num_sms, cudaStream_t st, const uint32_t *qlist = nullptr,
                      const uint32_t *qcount = nullptr);
// the flagged queries of each chunk of `chunk` queries: list[c chunk + i], i < count[c], = chunk-local index (one block)
void launch_ham_flag_list(const uint32_t *flags, uint32_t B, uint32_t chunk, uint32_t *list, uint32_t *count,
                          cudaStream_t st);
// thr[q] = dist[q][k-1] when cnt[q] >= k, else +inf (the sample's k-th smallest distance, an upper bound of the k-th
// smallest over all rows)
void launch_ham_threshold(const float *dist, const uint32_t *cnt, uint32_t B, uint32_t k, float *thr, cudaStream_t st);

// ---------------- multivector (MaxSim) columns, tensor-core score (gemm.cu F16MaxSim, F16RowMaxSim) -----------
// M[q][col_row[x] - row_base] = f32_key(max over the columns x of that document of the similarity) by atomicMax (M
// zeroed by the caller); Q [B][d] fp16 of the normalised query vectors, d a multiple of 8.  rows false (F16MaxSim):
// X [N][d] fp16 of the normalised stored vectors, similarity fp16(Q[q]) . X[x].  rows true (F16RowMaxSim): X [N][d]
// the stored fp16 vectors themselves, similarity (fp16(Q[q]) . X[x]) / vnorm[x].
struct MaxSimOut : GemmFilter {   // (GemmFilter's fields stay unset)
    const uint32_t *col_row;      // [N] document (row) of each column
    uint32_t *M;                  // [B][ldM]
    uint64_t ldM;
    uint32_t row_base;
    const float *vnorm;           // [N] |v| of each column (the per-column term; F16MaxSim does not use it)
};
void launch_maxsim_gemm(const void *Qh, const void *Xh, uint32_t B, uint64_t N, uint32_t d, const MaxSimOut &out,
                        bool rows, int num_sms, cudaStream_t st);
// out[n][d] = fp16(x / |x|) (|x| = sqrt(lance dot)) unless out is null; bad[n] = 1 (and the row zeroed) when |x| is 0
// or not finite or a component is not finite.  X: f32, or fp16 rows (the same arithmetic on their exact f32 upcast)
template <class T>
void launch_mv_normalize_f16(const T *X, uint64_t n, uint32_t d, void *out, uint32_t *bad, cudaStream_t st);
// the per-query error band of the approximate MaxSim distance: |approx - exact| <= mv_band(nq, d), or mv_band_f16(nq, d)
// for an fp16 handle's F16RowMaxSim score (multivec.cu)
float mv_band_host(uint32_t nq, uint32_t d);
float mv_band_f16_host(uint32_t nq, uint32_t d);
// A[b - qa][r] = sum over query b's vectors i of (1 - key_f32(M[i - i_base][r])), NaN when some M entry is 0 (empty row)
void launch_mv_approx_sum(const uint32_t *M, uint64_t ldM, const uint32_t *q_off, uint32_t qa, uint32_t qb,
                          uint32_t i_base, uint64_t N, float *A, uint64_t ldA, int num_sms, cudaStream_t st);
// thr[b] = dist[b][k-1] + 2 E_b when cnt[b] >= k, else +inf; E_b = mv_band(nq_b, d), or mv_band_f16 when f16
void launch_mv_threshold(const float *dist, const uint32_t *cnt, const uint32_t *q_off, uint32_t qa, uint32_t B,
                         uint32_t k, uint32_t d, bool f16, float *thr, cudaStream_t st);
// every row r with A[b][r] <= thr[b] that passes the row filter (allow null: none; the bit of its id col_ids[r], or r
// without ids, set and below allow_bits) is appended to cand[b][.] (count[b] zeroed by the caller, may exceed cap)
void launch_mv_admit(const float *A, uint64_t ldA, uint32_t B, uint64_t N, const float *thr, uint32_t cap,
                     uint32_t *count, uint32_t *cand, const uint64_t *col_ids, const uint32_t *allow,
                     uint64_t allow_bits, cudaStream_t st);
// flags[b] = count[b] > cap or a vector of query b is bad; vflags[i] = flags of the query of vector i; *gate = any flag
void launch_mv_flags(const uint32_t *count, uint32_t cap, const uint32_t *qbad, const uint32_t *q_off, uint32_t qa,
                     uint32_t B, uint32_t *flags, uint32_t *vflags, uint32_t *gate, cudaStream_t st);
// exact re-score (dist.cu): for slot s < min(count[b], cap): out[b][s] = MaxSim distance of query b and row cand[b][s]
// in the oracle's arithmetic, ids[b][s] = its id; other slots NaN / UINT64_MAX.  V: the stored vectors, float or
// __half (converted in registers: the bits of their exact f32 upcast)
template <class T>
void launch_mv_rescore(const float *Q, const uint32_t *q_off, uint32_t qa, const float *xnorm, const T *V,
                       const float *ysqrt, const uint64_t *offsets, const uint64_t *row_ids, uint32_t d, uint32_t B,
                       const uint32_t *cand, const uint32_t *count, uint32_t cap, float *out, uint64_t *ids,
                       cudaStream_t st);
// the same values when V is the mapped device alias of pinned host memory: each candidate row is read over PCIe in
// 16-byte cp.async requests staged in shared memory (dist.cu mv_rescore_host_kernel)
template <class T>
void launch_mv_rescore_host(const float *Q, const uint32_t *q_off, uint32_t qa, const float *xnorm, const T *V,
                            const float *ysqrt, const uint64_t *offsets, const uint64_t *row_ids, uint32_t d, uint32_t B,
                            const uint32_t *cand, const uint32_t *count, uint32_t cap, float *out, uint64_t *ids,
                            int num_sms, cudaStream_t st);
// dst[0, n) = src[0, n) elements (float, __half, or the bytes of packed binary rows) when *gate (device) != 0; nothing
// otherwise (multivec.cu)
template <class T>
void launch_mv_copy_gated(const T *src, T *dst, uint64_t n, const uint32_t *gate, int num_sms, cudaStream_t st);

// ---------------- multivector (MaxSim) columns, exact path (multivec.cu) ----------------------
// M[i][r] = min over row r0 + r's stored vectors j of P[i][j - offsets[r0]] (NaN skipped; NaN if none), for the nqv
// query vectors of P [nqv][ldP] and the nr rows r0..r0+nr-1 (offsets: device [nrows+1])
// gate (optional, device): 0 = nothing to do (the fix-up pass with no flagged query)
void launch_mv_rowmin(const float *P, uint64_t ldP, uint32_t nqv, const uint64_t *offsets, uint64_t r0, uint32_t nr,
                      float *M, uint64_t ldM, int num_sms, cudaStream_t st, const uint32_t *gate = nullptr);
// for queries b in [b_lo, b_hi) (q_off: device [B+1] vector offsets): D[b - qa][col0 + r] = running sum over the
// query's vectors i in [i0, i1) of M[i - i0][r], in order of i, started at 0.0f at the query's first vector
void launch_mv_rowsum(const float *M, uint64_t ldM, const uint32_t *q_off, uint32_t b_lo, uint32_t b_hi, uint32_t qa,
                      uint32_t i0, uint32_t i1, uint32_t nr, float *D, uint64_t ldD, uint64_t col0, int num_sms,
                      cudaStream_t st, const uint32_t *only = nullptr, const uint32_t *gate = nullptr);
// (only: optional [B] per-query flags indexed like q_off, queries whose flag is 0 are skipped)
// filtering epilogue on an existing dense score matrix D[B][ld] (see gemm.cu)
void launch_filter_dense(const float *D, uint64_t ld, uint32_t B, uint64_t N, const GemmFilter &flt, cudaStream_t st);
// thr[q] = k-th smallest sample score + 2 E_q (+inf: fewer than k scores; NaN: E_q is not finite, see tc_band)
void launch_sample_threshold(const float *approx, const uint32_t *cnt, const float *qnorm2, const float *qerr, float xmax,
                             float xerr, uint32_t d, uint32_t B, uint32_t k, float *thr, cudaStream_t st);
// the same threshold straight from dense sample scores D[B][ld] (ns <= 4096 columns; false = shape not handled)
bool launch_sample_kth_threshold(const float *D, uint64_t ld, uint32_t ns, const float *qnorm2, const float *qerr, float xmax,
                                 float xerr, uint32_t d, uint32_t B, uint32_t k, float *thr, cudaStream_t st);
// flags[q] = count[q] > cap, or thr[q] is NaN (thr optional)
void launch_overflow_flags(const uint32_t *count, uint32_t cap, const float *thr, uint32_t B, uint32_t *flags,
                           cudaStream_t st);
// flags[q] = 1 when the approximate shortlist of query q cannot be proven to contain the exact top-k:
// approx[q][0..kp) ascending, cnt[q] entries valid; proven iff E_q is finite and cnt < kp or
// approx[kp-1] > approx[k-1] + 2E_q (tc_band)
void launch_band_check(const float *approx, const uint32_t *cnt, const float *qnorm2, const float *qerr, float xmax,
                       float xerr, uint32_t d, uint32_t B, uint32_t k, uint32_t kp, uint32_t *flags, cudaStream_t st);

// ---------------- filter + verify form of the PQ scan (tables.cu, scan3.cu) -------------
// Quantised per-query tables.  qt[q][ch][c] = 8 x u16, position j = n_q[i][c] for sub-space i = 8 ch + ((j + c) & 7):
//   T_q[i][c] in [min_i + step n, min_i + step (n + 1)),  n <= qmax = floor(65535 / m)   (0 for i >= m)
// step[q] = max_i (max_c T - min_c T) / qmax, base[q] = sum_i min_i (- (m - 1) for dot),
// sbound[q] = sum_i max_c |T|, bad[q] = 1 when the table is not finite (the query takes the exact path).
// mm: scratch [B][8 nch][2].
void launch_query_tables_q16(const float *Q, const float *cb_tiled, const float *cb_n2, uint32_t B, uint32_t dim,
                             uint32_t m, uint32_t nch, uint32_t dsub, int metric, float *mm, uint4 *qt, float *step,
                             float *base, float *sbound, uint32_t *bad, cudaStream_t st);
// out[e] = |cb_tiled entry e|^2 for the nch * 256 * 8 tiled codebook entries (open time)
void launch_cb_norms(const float *cb_tiled, uint32_t nch, uint32_t dsub, float *out, cudaStream_t st);
// R[row] = 2 * codeword(row) . centroid(partition(row)); *rmax_bits = float bits of max |R|
void launch_row_const(const unsigned char *codes, const uint64_t *code_base, const uint32_t *part_npad,
                      const uint64_t *part_off, uint32_t nlist, uint64_t nrows, const float *centroids,
                      const float *cb_tiled, uint32_t dim, uint32_t m, uint32_t dsub, float *R, int *rmax_bits,
                      cudaStream_t st);
// exact PQ distances (oracle order) of (query, storage row) pairs; pos == UINT64_MAX -> +inf
void launch_pq_rescore(const float *Q, const uint64_t *pos, uint32_t B, uint32_t nc, const unsigned char *codes,
                       const uint64_t *code_base, const uint32_t *part_npad, const uint64_t *part_off, uint32_t nlist,
                       const float *centroids, const float *cb_tiled, uint32_t dim, uint32_t m, uint32_t dsub, int metric,
                       const uint32_t *ncols_q, float *out, cudaStream_t st);   // ncols_q: optional [B] pairs of each query (<= nc)
// probe_A[slot] = coarse_dist[slot] - |q|^2, amax[q] = max_j coarse + |q|^2, qn2[q] = |q|^2
// (probe_A / amax may be null: dot has no residual).  Sets bad[q] = 1 when |q|^2, amax[q] or base[q] + probe_A of one
// of the query's probes is not finite: its lower bounds or its band would be, so only the exact path can serve it.
void launch_probe_terms(const float *probe_dist, const float *Q, uint32_t B, uint32_t nprobes, uint32_t dim,
                        float *probe_A, float *amax, float *qn2, const float *base, uint32_t *bad, cudaStream_t st);
// The band of the filter scan (the error budget is above band_check3_kernel in tables.cu): the exact distance of a row
// lies in [L - E, L + W + E] (times the metric scale), with
//   W = m step (1 + 2^-10)
//   E = 2^-15 ceil(m/96) (sbound + amax + rmax + 2 (|q|^2 + CB2) [+ m for dot]) + 2^-126.
// For l2 and cosine every term scales with the data (E(2^j x) = 4^j E(x) in the normal range); dot's entries
// 1 - q_i.b hold a constant 1 each, hence its m.  2^-126 is the underflow floor: 2^18 of the 2^-150 absolute errors
// of subnormal products, quotients and conversions, more than the filter, the oracle and the coarse step make per row.
// Every consumer (band_check3, cand_prepare) takes its band from here.
struct ScanBand { float W, E; };
__device__ __forceinline__ ScanBand scan_band(float step, float sbound, float amax, float rmax, float qn2, float cb2,
                                              uint32_t m, bool dot)
{
    const float mag = sbound + amax + rmax + 2.0f * (qn2 + cb2) + (dot ? (float)m : 0.f);
    ScanBand b;
    b.W = (float)m * step * 1.0009765625f;
    // separate roundings (no contraction into an fmaf): the band the host-side restatement computes, bit for bit
    b.E = __fadd_rn(__fmul_rn(3.0517578125e-5f * (float)((m + 95u) / 96u), mag), 1.17549435e-38f);
    return b;
}
// W[q], E[q] = scan_band of every query (lgpu_debug_filter_bounds)
void launch_scan_band(const float *step, const float *sbound, const float *amax, const int *rmax_bits, const float *qn2,
                      float cb2, uint32_t m, bool dot, uint32_t B, float *W, float *E, cudaStream_t st);
// the band of every query, for the candidate mode: slack[q] = scale (W + 2E) (scan_band); also resets
// thr[q] = CAND_NO_THR, cand_cnt[q] = cand_last[q] = 0 and every key of cand_key to 0xffffffff
void launch_cand_prepare(const float *step, const float *sbound, const float *amax, const int *rmax_bits, const float *qn2,
                         float cb2, float scale, uint32_t m, bool dot, uint32_t B, float *slack, uint32_t *thr,
                         uint32_t *cand_cnt, uint32_t *cand_last, uint32_t *cand_key, uint32_t cand_cap, cudaStream_t st);
// candidate mode, after the scan: per query, drop the candidates above the final threshold, re-score the survivors
// exactly (oracle arithmetic, as launch_pq_rescore), and write the k best by (_distance, _rowid) -- ids, distances,
// count and (optional) storage positions.  flags[q] = 1 when the query must be redone by the exact kernels (list
// overflow, or bad[q]); such a query's outputs are overwritten by the fix-up pass.
struct FinalizeArgs {
    const float *Q;               // [B][dim] (normalised for cosine)
    const CandRec *cand; const uint32_t *cand_cnt; uint32_t cand_cap;
    const uint32_t *cand_key;     // [B][cand_cap] keys of the records (coalesced copy of CandRec::lb)
    const uint32_t *thr; const float *slack; const uint32_t *bad;
    const unsigned char *codes; const uint64_t *code_base; const uint32_t *part_npad; const uint64_t *part_off;
    const uint64_t *row_ids; const float *centroids; const float *cb_tiled;
    uint32_t B, dim, m, dsub, k; int metric;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count; uint64_t *out_pos; uint32_t *flags;
    unsigned long long *stats;    // optional [4]: candidates appended, survivors re-scored, queries flagged, queries
    // scratch of the three finalize kernels
    uint2 *work;                  // [B * cand_cap] survivors to re-score: (query, candidate index << 16 | survivor slot)
    uint32_t *work_cnt;           // [2]: survivors; gate word of the fix-up pass (set when a query is flagged)
    uint32_t *surv_cnt;           // [B] survivors per query
    float *ex_dist; uint64_t *ex_id; uint64_t *ex_pos;   // [B][cand_cap] exact distance / row id / storage position
    int num_sms;
};
void launch_cand_finalize(const FinalizeArgs &a, cudaStream_t st);
// flags[q] = 1 when the shortlist of q (lower bounds `lb` ascending, [B][kp], cnt valid) cannot be proven to hold
// the exact top-k: proven iff cnt < kp or lb[kp-1] > lb[k-1] + scale (W + 2E), W and E from scan_band; also 1 when
// bad[q].  amax / rmax_bits may be null (dot).  cb2 = sum_i max_c |codebook_i[c]|^2.  surv (optional, [B]): the length
// of the ascending prefix lb <= lb[k-1] + scale (W + 2E) -- the only rows that can be among the exact top-k, hence the
// only ones to re-score.
void launch_band_check3(const float *lb, const uint32_t *cnt, const float *step, const float *sbound, const float *amax,
                        const int *rmax_bits, const uint32_t *bad, const float *qn2, float cb2, float scale, uint32_t m,
                        bool dot, uint32_t B, uint32_t k, uint32_t kp, uint32_t *flags, uint32_t *gate, uint32_t *surv,
                        cudaStream_t st);

// ---------------- index build (build.cu) ----------------------------------------------
// codes[row][i] = argmin_c entry(row's residual sub-vector i, codebook_i[c]) (ties: lowest c); X normalised for cosine
void launch_pq_encode(const float *X, const uint32_t *parts, const float *centroids, const float *codebook,
                      uint64_t n, uint32_t dim, uint32_t m, int metric, unsigned char *codes, cudaStream_t st);

// ---------------- index training (kmeans.cu) ----------------------------------------------
// one Lloyd update: rows bucketed by `assign` (u64 centre id per row, >= k = unassigned), every non-empty centre replaced
// by the mean of its rows (f64 sums in ascending row order).  counts [k], offsets [k+1], cursor [k], rows [n]: scratch
void launch_kmeans_update(const uint64_t *assign, const float *x, uint64_t n, uint32_t dim, uint32_t k, uint32_t *counts,
                          uint32_t *offsets, uint32_t *cursor, uint32_t *rows, float *centroids, cudaStream_t st);
// *out = sum of the finite dist[i]
void launch_kmeans_inertia(const float *dist, uint64_t n, double *out, cudaStream_t st);
// one Lloyd update of all m PQ codebooks: codebook[i][c] = mean of the sub-vectors i of the rows with codes[row][i] == c
void launch_pq_update(const float *x, const unsigned char *codes, uint64_t n, uint32_t dim, uint32_t m, double *sums,
                      uint32_t *counts, float *codebook, cudaStream_t st);

// ---------------- index re-layout (open time) --------------------------------------
void launch_retile_codes(const unsigned char *codes, int layout, const uint64_t *part_off, uint32_t nlist,
                         uint64_t nrows, uint32_t m, uint32_t nch, const uint64_t *code_base,
                         const uint32_t *part_npad, unsigned char *out, cudaStream_t st);
void launch_retile_codebook(const float *codebook, uint32_t m, uint32_t dsub, uint32_t nch, float *out,
                            cudaStream_t st);

}  // namespace lgpu
