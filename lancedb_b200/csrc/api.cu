// api.cu -- the extern "C" boundary (include/lancedb_b200.h): handle management,
// workspaces, and the host-side orchestration of one batched vector query:
//   [cosine: normalise] -> K1 exact centroid distances -> select nprobes ->
//   regroup probe slots by partition -> K2+K3 fused LUT build + code scan ->
//   K4 top-k by (_distance,_rowid) -> [refine: exact re-rank] .
// Everything runs on one stream per call with no host round trip in between.
// The reference-side equivalent is NativeTable::create_plan + execute_plan
// (rust/lancedb/src/table/query.rs:131-328, :121).
#include "kernels.cuh"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <unordered_set>
#include <vector>

#include <dlfcn.h>
#include <nccl.h>
#include <pthread.h>
#include <unistd.h>

namespace lgpu {

static thread_local std::string g_err;
static thread_local float g_stage_ms[7] = {0, 0, 0, 0, 0, 0, 0};
static thread_local uint64_t g_scanned_bytes = 0;
static thread_local uint64_t g_filter_stats[4] = {0, 0, 0, 0};
void set_error(const std::string &msg) { g_err = msg; }

// every kernel the library launches (eagerly, into a stream capture, or through a graph replay) is counted
static std::atomic<uint64_t> g_kernel_launches{0};
static thread_local bool g_capturing = false;        // launches made while capturing are counted per replay instead
static thread_local uint64_t g_captured_launches = 0;
bool pdl_enabled()
{
    static int v = -1;
    if (v < 0) { const char *e = getenv("LGPU_NO_PDL"); v = (e && e[0] == '1') ? 0 : 1; }
    return v == 1;
}

void count_launches(uint64_t n)
{
    if (g_capturing) g_captured_launches += n;
    else g_kernel_launches.fetch_add(n, std::memory_order_relaxed);
}

static std::atomic<int> g_profiling{-1};
static bool profiling_enabled()
{
    int v = g_profiling.load(std::memory_order_relaxed);
    if (v < 0) {
        const char *e = getenv("LGPU_PROFILE");
        int want = (e && e[0] == '1') ? 1 : 0;
        g_profiling.compare_exchange_strong(v, want);     // lgpu_set_profiling may have won the race: keep its value
        v = g_profiling.load(std::memory_order_relaxed);
    }
    return v == 1;
}
static size_t workspace_budget()
{
    static size_t v = 0;
    if (!v) {
        const char *e = getenv("LGPU_WS_BYTES");
        v = e ? (size_t)strtoull(e, nullptr, 10) : ((size_t)8 << 30);
        if (v < ((size_t)1 << 20)) v = (size_t)1 << 20;
    }
    return v;
}

// bumped by every device (re)allocation in the process.  A captured CUDA graph bakes workspace pointers in, so a
// graph is only replayed while the epoch still equals the one recorded at capture (Workspace::graph_epoch): any
// entry point, on any thread, that grows a buffer invalidates every captured graph (they re-capture on next use).
static std::atomic<uint64_t> g_alloc_epoch{0};

struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    void ensure(size_t n)
    {
        if (n <= bytes) return;
        g_alloc_epoch++;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        size_t want = n + n / 8;
        LGPU_CUDA(cudaMalloc(&p, want));
        bytes = want;
    }
    template <class T> T *as() { return reinterpret_cast<T *>(p); }
    ~DevBuf() { if (p) cudaFree(p); }
};

struct Workspace {
    cudaStream_t stream = nullptr;     // private stream (host-buffer entry points)
    // side stream of the filter scan's front: the coarse step and the regrouping run here while the per-query tables
    // are built on the search stream.  Created at the device's greatest priority, so that as SMs free up the block
    // scheduler hands them to this short critical chain before the waiting table CTAs (a per-stream property)
    cudaStream_t front = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int stats_mode = 0;                 // profiling: 1 = the last sub-batch ran the candidate mode, 2 = the dense filter
    uint32_t stages_marked = 0;         // profiling: bit s = ev[s] was recorded by the profiled sub-batch (IvfStage)
    bool front_open = false;            // an EAGER fork onto `front` has not been joined yet (a call failed half-way)
    cudaEvent_t done = nullptr;        // last use, for cross-stream reuse
    cudaEvent_t ev[8] = {};
    DevBuf q, qn, xnorm, D, probes, probe_dist, probe_cnt;
    DevBuf part_cnt, slot_pos, seg_local, qtot, seg_off, qlist_off, tile_off, tile_off_b, qlist, scalars, tile_desc, allow;
    DevBuf dist_out, out_ids, out_dist, out_count;
    DevBuf t_ids, t_dist, t_pos, t_cnt, t_exact;
    DevBuf widen;                       // maximum_nprobes widening: queries that found fewer than k rows
    DevBuf qb, qn2, qerr, flags;        // tensor-core shortlist: bf16 queries, |q|^2, |bf16(q) - q|, unproven-query flags
    // CUDA graph of one host-buffer search (lgpu_search): the ~15 launches of a batch replayed as one
    cudaGraphExec_t graph = nullptr;
    uint64_t graph_key[4] = {0, 0, 0, 0};
    uint64_t graph_epoch = 0;           // g_alloc_epoch when `graph` was captured
    uint64_t graph_kernels = 0;         // kernel launches one replay stands for
    int graph_state = 0;                // 0: next call runs eagerly (warm-up), 1: capture, 2: replay, -1: disabled
    DevBuf sbound, probe_A, amax;       // tensor-core shortlists: thresholds / counters; filter scan: bounds, per-probe scalars
    DevBuf qt, qt_mm, qt_step, qt_base, qt_bad;   // filter scan (scan3.cu): quantised per-query tables
    DevBuf s_ids, s_lb, s_pos, s_cnt, s_exact;    // filter scan (dense mode): shortlist by lower bound, exact re-score
    DevBuf c_stats;                               // candidate-mode counters (profiling only)
    DevBuf c_work, c_wcnt, c_surv, c_exd, c_exi, c_exp;   // candidate mode: survivor work list and exact results
    DevBuf c_thr, c_slack, c_cnt, c_rec, c_key, c_last;          // filter scan (candidate mode): thresholds, bands, candidate lists
    DevBuf hq, hq_pop, h_sample, h_list, h_cnt;   // binary search: padded queries, popc(q), sample distances, fix-up list
    DevBuf mv_qoff, mv_P, mv_M;         // multivector search: query vector offsets, pairwise cosd block, per-row minima
    DevBuf mv_qh, mv_qbad, mv_Mk, mv_A; // ... tensor-core path: fp16 queries, bad vectors, max-similarity keys, approx dist
    DevBuf mv_kd, mv_ki, mv_kc, mv_thr, mv_cnt, mv_cand, mv_flags, mv_vflags, mv_gate, mv_ex, mv_exid;   // shortlist
    DevBuf sq_q, sq_qq;                 // IVF_SQ search: query codes [B][dim_pad], their squared sums
    DevBuf rq_q, rq_planes, rq_slots;   // IVF_RQ search: rotated queries [B][dim], per-slot bit-planes and grids
    DevBuf pq4_tab, pq4_slots;          // 4-bit IVF_PQ search: per-slot u8 tables [slots][m][16] and quantisers
    Workspace()
    {
        LGPU_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        int least = 0, greatest = 0;
        LGPU_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        LGPU_CUDA(cudaStreamCreateWithPriority(&front, cudaStreamNonBlocking, greatest));
        LGPU_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        LGPU_CUDA(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
        LGPU_CUDA(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
        for (auto &e : ev) LGPU_CUDA(cudaEventCreate(&e));
    }
    ~Workspace()
    {
        if (graph) cudaGraphExecDestroy(graph);
        if (stream) cudaStreamDestroy(stream);
        if (front) cudaStreamDestroy(front);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
        if (done) cudaEventDestroy(done);
        for (auto &e : ev) if (e) cudaEventDestroy(e);
    }
};

struct WorkspacePool {
    std::mutex mu;
    std::vector<Workspace *> free_list;
    Workspace *take()
    {
        {
            std::lock_guard<std::mutex> g(mu);
            if (!free_list.empty()) { Workspace *w = free_list.back(); free_list.pop_back(); return w; }
        }
        return new Workspace();
    }
    void give(Workspace *w) { std::lock_guard<std::mutex> g(mu); free_list.push_back(w); }
    ~WorkspacePool() { for (auto *w : free_list) delete w; }
};

}  // namespace lgpu

using namespace lgpu;

// ---- live-handle registry: every entry point resolves its handle through it, so a handle that was closed (or
// that belongs to the parent of a fork()) is rejected instead of dereferenced, and close waits for the calls
// still inside the handle (BaseTable is Send + Sync: rust/lancedb/src/table.rs:549; queries are re-executable
// from any tokio worker: rust/lancedb/src/query.rs:954-955).
namespace lgpu {
static std::mutex g_live_mu;
static std::condition_variable g_live_cv;
static std::unordered_set<const void *> g_live;
static std::atomic<bool> g_cuda_touched{false};   // this process has created a CUDA context through the library
static std::atomic<bool> g_fork_poisoned{false};  // we are the child of a fork() taken after that
// fork(): the reference rebuilds its tokio runtime in the child (python/src/runtime.rs:68-81); a CUDA context has
// the same constraint and cannot be rebuilt, so the child drops every handle and refuses GPU work.
static void atfork_prepare() { g_live_mu.lock(); }
static void atfork_parent() { g_live_mu.unlock(); }
static void atfork_child()
{
    g_live.clear();                                  // the parent's handles are not valid here (leaked, never freed)
    if (g_cuda_touched.load()) g_fork_poisoned.store(true);
    g_live_mu.unlock();
}
static void register_handle(const void *h)
{
    static std::once_flag once;
    std::call_once(once, [] { pthread_atfork(atfork_prepare, atfork_parent, atfork_child); });
    std::lock_guard<std::mutex> g(g_live_mu);
    g_live.insert(h);
}
template <class H> struct HandleRef {
    H *h;
    HandleRef(H *p, const char *what) : h(nullptr)
    {
        std::lock_guard<std::mutex> g(g_live_mu);
        if (!p || !g_live.count(p)) {
            set_error(std::string(what) + " handle is null, closed, or was opened in another process (fork)");
            throw Failure{LGPU_INVALID_INPUT};
        }
        p->refs.fetch_add(1);
        h = p;
    }
    ~HandleRef()
    {
        if (h && h->refs.fetch_sub(1) == 1) { std::lock_guard<std::mutex> g(g_live_mu); g_live_cv.notify_all(); }
    }
    H *operator->() const { return h; }
};
// unregister and wait until no call is inside the handle any more; false = it was not a live handle
template <class H> static bool retire_handle(H *p)
{
    std::unique_lock<std::mutex> g(g_live_mu);
    if (!p || !g_live.erase(p)) return false;
    g_live_cv.wait(g, [&] { return p->refs.load() == 0; });
    return true;
}
// every *_close: unregister, drain the handle's device, free it.  A null or closed handle, or a parent-process
// handle in a fork child, is left alone.
template <class H> static void close_handle(H *p)
{
    if (!retire_handle(p)) return;
    cudaSetDevice(p->device);
    cudaDeviceSynchronize();
    delete p;
}
}  // namespace lgpu

// micro-batcher of concurrent single-vector calls (SURVEY.md 8b "Threading": many tokio workers each with one query
// vector).  Callers with identical parameters that arrive within a short window ride one batched search: the first
// arrival leads -- waits for the window (or a full batch), takes the queue, runs lgpu_search on the gathered
// queries, scatters the rows -- the others sleep on the condition variable until their row is filled in.
namespace lgpu {
struct PendingQuery {
    const float *q; uint64_t *ids; float *dist; uint32_t *cnt;
    int status = LGPU_OK; bool done = false; std::string err;
};
struct Coalescer {
    std::mutex mu;
    std::condition_variable cv;
    struct Lane { lgpu_search_params params; std::vector<PendingQuery *> queue; bool leader = false; };
    std::vector<Lane *> lanes;                           // one per distinct parameter set seen (a handful)
    ~Coalescer() { for (auto *l : lanes) delete l; }
};
}  // namespace lgpu

struct lgpu_index {
    std::atomic<int> refs{0};
    Coalescer coalescer;
    int device = 0, num_sms = 0;
    uint32_t dim = 0, nlist = 0, m = 0, dsub = 0, nch = 0;
    uint32_t max_nrb = 1;          // row blocks (of 1536 rows) of the largest partition: bounds the tile count
    int metric = 0;
    uint64_t nrows = 0, device_bytes = 0;
    DevBuf centroids, cb_tiled, codes, code_base, part_n, part_npad, part_off, row_ids, vectors;
    DevBuf row_R, rmax_bits;            // filter scan: per-row constant 2 b.c and max |R| (tables.cu)
    DevBuf cb_n2;                       // filter scan: |b|^2 of every tiled codebook entry
    float cb2 = 0.f;                    // sum_i max_c |codebook_i[c]|^2 (error budget of the filter's table entries)
    bool has_tables = false;
    DevBuf cent_b, cent_n2;             // bf16 centroids + |c|^2 for the tensor-core coarse step
    DevBuf cent_sb, cent_sn2;           // every COARSE_SAMPLE_STRIDE-th centroid (bf16 + |c|^2): the threshold sample
    uint32_t cent_ns = 0;               // rows of the sample (0: none)
    float cent_max = 0.f, cent_err = 0.f;   // max |c|, max |bf16(c) - c| (the error band, kernels.cuh tc_band)
    bool has_tc = false;
    bool has_vectors = false;
    // IVF_SQ (lgpu_ivf_sq_open): `codes` holds [nrows][dim_pad] u8 row codes, `sq_xx` the sum of each row's squared codes
    bool is_sq = false;
    uint32_t dim_pad = 0;
    double sq_lo = 0.0, sq_hi = 0.0;
    DevBuf sq_xx;
    // IVF_RQ (lgpu_ivf_rq_open): `codes` holds [nrows][rq_wpr] u32 sign bits; the rotation, the rotated centroids and
    // the per-row factors and popcounts
    bool is_rq = false;
    uint32_t rq_wpr = 0;
    DevBuf rq_rot, rq_rc, rq_add, rq_scale, rq_popc;
    // 4-bit IVF_PQ (lgpu_index_open with nbits = 4): `codes` holds per partition [m/2][npad] packed bytes, `pq4_cb` the
    // codebook [m][dsub][16] (element-major); no filter tables
    bool is_pq4 = false;
    DevBuf pq4_cb;
    std::vector<uint64_t> pad_prefix;   // prefix sums of pad4(n_p) sorted descending
    std::vector<uint32_t> h_part_n;
    WorkspacePool pool;
};

// a binary IVF_FLAT index (lgpu_ivf_binary_open): the IVF partition arrays of lgpu_index (part_n, part_off, row_ids,
// pad_prefix, ...; `dim` = nbytes), with `centroids` holding the packed centroids [nlist][nbytes_pad] and `codes` the
// packed rows [nrows][nbytes_pad] in partition order, both zero-padded, and their popcounts
struct lgpu_ivf_binary : lgpu_index {
    uint32_t nbytes = 0, nbytes_pad = 0;
    DevBuf cent_pop, row_pop;
};

struct lgpu_flat {
    std::atomic<int> refs{0};
    int device = 0;
    uint64_t nrows = 0;
    uint32_t dim = 0;
    DevBuf vectors, row_ids, ysqrt;
    DevBuf vec_b, vec_n2;               // bf16 rows + |x|^2 for the tensor-core path
    float vec_max = 0.f, vec_err = 0.f;     // max |x|, max |bf16(x) - x|
    int num_sms = 0;
    bool has_tc = false;
    bool has_ids = false, has_norms = false;
    std::mutex mu;
    WorkspacePool pool;
};

// a packed binary vector column (fixed_size_list<uint8, nbytes>) searched by Hamming distance
struct lgpu_binary {
    std::atomic<int> refs{0};
    int device = 0, num_sms = 0;
    uint64_t nrows = 0;
    uint32_t nbytes = 0, nbytes_pad = 0;   // caller's row bytes; stored row bytes (multiple of 32)
    DevBuf vectors, pop, row_ids;          // [nrows][nbytes_pad] zero-padded rows, popc of each row, optional ids
    DevBuf sample, sample_pop;             // every (nrows / nsample)-th row: the threshold sample of the list path
    uint64_t nsample = 0;                  // 0: no sample (nrows <= HAM_SAMPLE)
    bool has_ids = false;
    WorkspacePool pool;
};

// a multivector column (list<fixed_size_list<float, dim>>) searched by late interaction (MaxSim over cosine)
struct lgpu_multivec {
    std::atomic<int> refs{0};
    int device = 0, num_sms = 0;
    uint64_t nrows = 0, total = 0;         // rows; stored vectors T = offsets[nrows]
    uint32_t dim = 0;
    uint64_t max_row = 0;                  // largest n_r
    DevBuf vectors, ysqrt, offsets, row_ids;   // [T][dim] f32, |v| = sqrt(dot(v, v)) per vector, [nrows+1], optional ids
    DevBuf vec_h, col_row;                 // tensor-core path: fp16 normalised vectors [T][dim], row of each vector [T]
    bool tc_ok = false;                    // the tensor-core path may run (see multivec_search_device)
    std::vector<uint64_t> h_offsets;       // host copy: the row chunks of a search are cut on the host
    bool has_ids = false;
    WorkspacePool pool;
};

// ---- NCCL, bound at run time (dlopen): single-GPU hosts need no libnccl, and inside a process that already
// loaded one (torch) the same library instance is used ----
namespace lgpu {
struct NcclApi {
    void *lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    std::string error;
};
static NcclApi &nccl_api()
{
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {getenv("LGPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            if (!n || !*n) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) { api.error = "libnccl.so.2 not found (set LGPU_NCCL_LIB)"; return; }
        auto sym = [&](const char *n) { void *f = dlsym(api.lib, n); if (!f) api.error = std::string("missing NCCL symbol ") + n; return f; };
        api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
        api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
        api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
        api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
        api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    });
    if (!api.error.empty()) { set_error("NCCL unavailable: " + api.error); throw Failure{LGPU_RUNTIME}; }
    return api;
}
#define LGPU_NCCL(expr)                                                                          \
    do {                                                                                         \
        ncclResult_t _r = (expr);                                                                \
        if (_r != ncclSuccess) {                                                                 \
            ::lgpu::set_error(std::string(#expr) + ": " + ::lgpu::nccl_api().GetErrorString(_r)); \
            throw ::lgpu::Failure{LGPU_RUNTIME};                                                 \
        }                                                                                        \
    } while (0)
}  // namespace lgpu

// one rank of a partition-sharded search group (SURVEY.md 8e): an NCCL communicator plus the gather buffers
struct lgpu_comm {
    std::atomic<int> refs{0};
    int device = 0, rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    std::mutex mu;                       // collectives of one communicator are issued one call at a time
    DevBuf send, recv;                   // [B][k] / [world][B][k] TopkRecord
    DevBuf l_ids, l_dist, l_cnt;         // the local (per-shard) top-k before the exchange
    cudaEvent_t ev[3] = {};              // local search done / all-gather done / merge done (stage timing)
    float last_ms[3] = {0, 0, 0};        // local search, all-gather, merge of the most recent profiled call
    ~lgpu_comm()
    {
        try { if (comm) nccl_api().CommDestroy(comm); } catch (const Failure &) {}
        for (auto &e : ev) if (e) cudaEventDestroy(e);
    }
};

namespace {

struct WsLease {
    WorkspacePool &pool;
    Workspace *ws;
    cudaStream_t st;
    WsLease(WorkspacePool &p, cudaStream_t user, bool use_user) : pool(p), ws(p.take())
    {
        st = use_user ? user : ws->stream;
        // the workspace may still be in use by an earlier call on another stream
        if (cudaStreamWaitEvent(st, ws->done, 0) != cudaSuccess) cudaGetLastError();
    }
    ~WsLease()
    {
        // side-stream work of a call that failed half-way.  Only after an eager fork: an event whose last record sits
        // inside a captured graph cannot be waited on outside the capture (cudaErrorInvalidValue, which would then be
        // reported by the next cudaGetLastError() of an unrelated launch).
        if (ws->front_open) {
            if (cudaEventRecord(ws->ev_join, ws->front) != cudaSuccess || cudaStreamWaitEvent(st, ws->ev_join, 0) != cudaSuccess)
                cudaGetLastError();
            ws->front_open = false;
        }
        if (cudaEventRecord(ws->done, st) != cudaSuccess) cudaGetLastError();
        pool.give(ws);
    }
};

// Deadline of one call (QueryExecutionOptions::timeout -> TimeoutStream, rust/lancedb/src/utils/mod.rs:328-393,
// used at rust/lancedb/src/query.rs:1452-1457).  Kernels cannot be cancelled, so the deadline is enforced where
// the host waits: between sub-batches and before the results are copied back.  On expiry the call returns
// LGPU_TIMEOUT without touching the caller's output buffers; work already enqueued drains into the workspace,
// which stays fenced by its `done` event until then.
struct Deadline {
    bool armed = false;
    std::chrono::steady_clock::time_point at;
    explicit Deadline(uint32_t timeout_ms)
    {
        if (timeout_ms) { armed = true; at = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms); }
    }
    bool expired() const { return armed && std::chrono::steady_clock::now() >= at; }
    // wait for everything enqueued on `st` so far, or for the deadline
    void wait(cudaStream_t st, cudaEvent_t ev) const
    {
        if (!armed) return;
        LGPU_CUDA(cudaEventRecord(ev, st));
        for (;;) {
            cudaError_t e = cudaEventQuery(ev);
            if (e == cudaSuccess) return;
            if (e != cudaErrorNotReady) LGPU_CUDA(e);
            if (expired()) { set_error("Query timeout"); throw Failure{LGPU_TIMEOUT}; }
            std::this_thread::sleep_for(std::chrono::microseconds(50));
        }
    }
};

// prefilter: device bitmap over row ids (nullptr = no filter)
struct RowFilter {
    const uint32_t *bits = nullptr;
    uint64_t nbits = 0;
};

// LGPU_EXACT_SCAN=1 sends every query through the exact kernel (scan2.cu) instead of filter + verify
// (scan3.cu + tables.cu).  Results are bit-identical either way; the switch exists for A/B timing and tests.
static bool exact_scan_forced()
{
    const char *e = getenv("LGPU_EXACT_SCAN");
    return e && e[0] == '1';
}

// Mode switches of the IVF path, re-read on every call (tests flip them between calls; getenv is ~100 ns) and folded
// into the CUDA-graph key so a captured launch sequence is never replayed under a different mode.
struct ScanModes {
    bool exact, dense_forced, force_tc_coarse;
    uint32_t cand_kmax, cap_env, small_slots, coarse_list_min;
    uint64_t signature() const
    {
        return ((uint64_t)exact | (uint64_t)dense_forced << 1 | (uint64_t)force_tc_coarse << 2 | (uint64_t)cand_kmax << 8 |
                (uint64_t)cap_env << 20 | (uint64_t)small_slots << 36 | (uint64_t)(coarse_list_min & 0xffffu) << 48) *
               0x9e3779b97f4a7c15ull;
    }
};
static ScanModes scan_modes()
{
    auto num = [](const char *name, uint32_t dflt) { const char *e = getenv(name); return e ? (uint32_t)atoi(e) : dflt; };
    ScanModes m;
    m.exact = exact_scan_forced();
    m.dense_forced = getenv("LGPU_DENSE_FILTER") != nullptr;
    m.force_tc_coarse = getenv("LGPU_FORCE_TC_COARSE") != nullptr;   // the tensor-core coarse step at any B x nlist
    m.cand_kmax = std::min<uint32_t>(CAND_TOPK_MAX, num("LGPU_CAND_KMAX", CAND_TOPK_MAX));
    m.cap_env = num("LGPU_CAND_CAP", 0u);
    m.small_slots = num("LGPU_SMALL_SLOTS", 1024u);
    m.coarse_list_min = num("LGPU_COARSE_LIST_MIN", 8192u);     // nlist from which the coarse GEMM filters (0: never)
    return m;
}

static bool tc_enabled()
{
    static int v = -1;
    if (v < 0) { const char *e = getenv("LGPU_NO_TENSOR_CORE"); v = (e && e[0] == '1') ? 0 : 1; }
    return v == 1;
}

// bf16 copy + squared norms + max norm and max bf16 rounding error |bf16(x) - x| of a row-major f32 matrix (open time)
static void prepare_tc_operand(const float *X, uint64_t n, uint32_t d, DevBuf &Xb, DevBuf &n2, float &xmax, float &xerr,
                               cudaStream_t st)
{
    Xb.ensure(std::max<size_t>((size_t)n * d * 2, 16));
    n2.ensure(std::max<size_t>((size_t)n * 4, 16));
    DevBuf err;
    err.ensure(std::max<size_t>((size_t)n * 4, 16));
    launch_to_bf16(X, n, d, Xb.p, n2.as<float>(), st, err.as<float>());
    std::vector<float> h(n), he(n);
    LGPU_CUDA(cudaMemcpyAsync(h.data(), n2.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaMemcpyAsync(he.data(), err.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaStreamSynchronize(st));
    float m = 0.f, me = 0.f;
    for (float v : h) m = std::max(m, v);
    for (float v : he) me = std::max(me, v);
    xmax = std::sqrt(m) * 1.0001f;
    xerr = me;
}

// where a top-k goes: [B][k] ids and distances, [B] counts and, optionally, [B][k] storage positions
struct TopkOut {
    uint64_t *ids;
    float *dist;
    uint32_t *cnt;
    uint64_t *pos = nullptr;
    // the rows of queries q0, q0 + 1, ... of a [B][k] output
    TopkOut at(uint32_t q0, uint32_t k) const { return {ids + (size_t)q0 * k, dist + (size_t)q0 * k, cnt + q0}; }
};

// SelectArgs with the fields every mode needs; callers add the optional ones (only, gate, col_ids, range, allow, ...)
static SelectArgs select_args(int mode, uint32_t B, uint32_t k, TopkOut out)
{
    SelectArgs s{};
    s.mode = mode; s.B = B; s.k = k;
    s.out_ids = out.ids; s.out_dist = out.dist; s.out_count = out.cnt; s.out_pos = out.pos;
    return s;
}
// mode 1: the k best of the first ncols columns of every row of the dense block D [B][ld]
static SelectArgs select_rows(const float *D, uint64_t ncols, uint64_t ld, uint32_t B, uint32_t k, TopkOut out)
{
    SelectArgs s = select_args(1, B, k, out);
    s.dense = D; s.ncols = ncols; s.row_stride = ld;
    return s;
}
// mode 2: the k best of every query's n candidates, values and ids [B][n]
static SelectArgs select_cands(const float *vals, const uint64_t *ids, uint64_t n, uint32_t B, uint32_t k, TopkOut out)
{
    SelectArgs s = select_args(2, B, k, out);
    s.dense = vals; s.cand_ids = ids; s.ncols = n; s.inner = n; s.row_stride = n; s.outer_stride = 0;
    return s;
}
static void with_range(SelectArgs &s, const lgpu_search_params &sp)
{
    s.has_lower = sp.has_lower; s.has_upper = sp.has_upper; s.lower = sp.lower; s.upper = sp.upper;
}

// The tail of tc_topk_l2 and tc_topk_l2_filtered: exact re-score of the [B][cap] candidate slots (ws->t_pos, t_ids;
// one pair per slot, empty slots included), their top-k into the outputs, then the dense fix-up of the queries
// flagged in ws->flags (no-ops when none is).
static void tc_rescore_fixup(Workspace *ws, cudaStream_t st, const float *Q, uint32_t B, const float *X, uint64_t N,
                             uint32_t d, const uint64_t *col_ids, uint32_t k, uint32_t cap, TopkOut out, float *Dbuf,
                             uint64_t ld)
{
    launch_pair_distance(Q, X, ws->t_pos.as<uint64_t>(), B, cap, d, LGPU_L2, ws->t_exact.as<float>(), st);
    launch_select(select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), cap, B, k, out), st);
    launch_dist_matrix(Q, X, B, N, d, 0, nullptr, nullptr, Dbuf, ld, st, ws->flags.as<uint32_t>());
    SelectArgs sc = select_rows(Dbuf, N, ld, B, k, out);
    sc.col_ids = col_ids; sc.only = ws->flags.as<uint32_t>();
    launch_select(sc, st);
}

// Tensor-core shortlist + exact re-score (squared L2 only): the k best of the N rows of X for each
// of B queries by exact lance-order distance, ids from col_ids (or the row index), ascending by
// (distance, id).  Dbuf: [B][ld] f32 scratch.  Queries whose shortlist cannot be proven complete
// (band_check) are redone by the exact kernels in the same stream, without a host round trip.
static void tc_topk_l2(Workspace *ws, cudaStream_t st, int num_sms, const float *Q, uint32_t B, const float *X,
                       const void *Xb, const float *xnorm2, float xmax, float xerr, uint64_t N, uint32_t d,
                       const uint64_t *col_ids, uint32_t k, uint32_t kp, TopkOut out, float *Dbuf, uint64_t ld)
{
    ws->qb.ensure((size_t)B * d * 2); ws->qn2.ensure((size_t)B * 4); ws->qerr.ensure((size_t)B * 4);
    ws->flags.ensure((size_t)B * 4);
    ws->t_ids.ensure((size_t)B * kp * 8); ws->t_dist.ensure((size_t)B * kp * 4);
    ws->t_pos.ensure((size_t)B * kp * 8); ws->t_cnt.ensure((size_t)B * 4); ws->t_exact.ensure((size_t)B * kp * 4);
    launch_to_bf16(Q, B, d, ws->qb.p, ws->qn2.as<float>(), st, ws->qerr.as<float>());
    launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, N, d, Dbuf, ld, num_sms, st);
    SelectArgs sa = select_rows(Dbuf, N, ld, B, kp, {ws->t_ids.as<uint64_t>(), ws->t_dist.as<float>(),
                                                     ws->t_cnt.as<uint32_t>(), ws->t_pos.as<uint64_t>()});
    sa.col_ids = col_ids;
    launch_select(sa, st);
    if (kp >= N) LGPU_CUDA(cudaMemsetAsync(ws->flags.p, 0, (size_t)B * 4, st));   // every row is a candidate
    else launch_band_check(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->qn2.as<float>(), ws->qerr.as<float>(),
                           xmax, xerr, d, B, k, kp, ws->flags.as<uint32_t>(), st);
    tc_rescore_fixup(ws, st, Q, B, X, N, d, col_ids, k, kp, out, Dbuf, ld);
}

// Large-N variant of tc_topk_l2 (flat search): a tensor-core pass over a row sample fixes, per query, a
// score threshold that provably admits every true top-k row; the pass over all rows then runs with the
// filtering epilogue (no dense score matrix), the few admitted rows are re-scored exactly, and queries whose
// candidate list overflowed are redone by the exact kernels.
static void tc_topk_l2_filtered(Workspace *ws, cudaStream_t st, int num_sms, const float *Q, uint32_t B, const float *X,
                                const void *Xb, const float *xnorm2, float xmax, float xerr, uint64_t N, uint32_t d,
                                const uint64_t *col_ids, uint32_t k, TopkOut out, float *Dbuf, uint64_t ld,
                                uint64_t min_sample = 65536, uint32_t cap = 1024)
{
    const uint64_t Ns = std::min<uint64_t>(N, std::max<uint64_t>(min_sample, N / 8));
    const uint64_t lds = (Ns + 3) & ~3ull;               // Dbuf is [B][ld >= lds]
    ws->qb.ensure((size_t)B * d * 2); ws->qn2.ensure((size_t)B * 4); ws->qerr.ensure((size_t)B * 4);
    ws->flags.ensure((size_t)B * 4);
    ws->t_ids.ensure((size_t)B * cap * 8); ws->t_dist.ensure((size_t)B * std::max<uint32_t>(k, 32) * 4);
    ws->t_pos.ensure((size_t)B * cap * 8); ws->t_cnt.ensure((size_t)B * 4); ws->t_exact.ensure((size_t)B * cap * 4);
    ws->probe_A.ensure((size_t)B * 4);                   // thr[q]
    ws->amax.ensure((size_t)B * 4);                      // candidate counters
    ws->sbound.ensure((size_t)B * std::max<uint32_t>(k, 32) * 8);   // sample ids (unused)
    launch_to_bf16(Q, B, d, ws->qb.p, ws->qn2.as<float>(), st, ws->qerr.as<float>());
    // 1. sample pass: dense scores of the first Ns rows, k-th best per query -> threshold
    launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, Ns, d, Dbuf, lds, num_sms, st);
    launch_select(select_rows(Dbuf, Ns, lds, B, k, {ws->sbound.as<uint64_t>(), ws->t_dist.as<float>(),
                                                    ws->t_cnt.as<uint32_t>()}), st);
    launch_sample_threshold(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->qn2.as<float>(), ws->qerr.as<float>(),
                            xmax, xerr, d, B, k, ws->probe_A.as<float>(), st);
    // 2. full pass with the filtering epilogue
    LGPU_CUDA(cudaMemsetAsync(ws->amax.p, 0, (size_t)B * 4, st));
    LGPU_CUDA(cudaMemsetAsync(ws->t_pos.p, 0xff, (size_t)B * cap * 8, st));
    LGPU_CUDA(cudaMemsetAsync(ws->t_ids.p, 0xff, (size_t)B * cap * 8, st));
    GemmFilter flt{};
    flt.thr = ws->probe_A.as<float>(); flt.count = ws->amax.as<uint32_t>(); flt.cand_pos = ws->t_pos.as<uint64_t>();
    flt.cand_ids = ws->t_ids.as<uint64_t>(); flt.col_ids = col_ids; flt.cap = cap;
    if (Ns == N) launch_filter_dense(Dbuf, lds, B, N, flt, st);      // the sample pass already scored every row
    else launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, N, d, nullptr, 0, num_sms, st, &flt);
    launch_overflow_flags(ws->amax.as<uint32_t>(), cap, B, ws->flags.as<uint32_t>(), st);
    // 3. exact re-score of the admitted rows, final top-k; 4. fix-up of overflowed queries
    tc_rescore_fixup(ws, st, Q, B, X, N, d, col_ids, k, cap, out, Dbuf, ld);
}

// top-k by (distance, id) of the dense scores D [b][ld] over N columns, with the request's distance range and
// prefilter, into `out`
static void select_dense(const float *D, uint64_t N, uint64_t ld, const uint64_t *col_ids, uint32_t b,
                         const lgpu_search_params &sp, RowFilter rf, TopkOut out, cudaStream_t st)
{
    SelectArgs sa = select_rows(D, N, ld, b, sp.k, out);
    sa.col_ids = col_ids;
    with_range(sa, sp);
    sa.allow = rf.bits; sa.allow_bits = rf.nbits;
    launch_select(sa, st);
}

// the arguments every search call takes: the parameters, then the query and output buffers of a call with queries.
// refine: the kind selects k * refine_factor candidates (a kind whose distances are exact ignores refine_factor)
static void check_call(const lgpu_search_params *p, uint32_t B, const void *q, const void *ids, const void *dist,
                       const void *cnt, bool refine = true)
{
    LGPU_REQUIRE(p != nullptr, "search params are null");
    LGPU_REQUIRE(p->k >= 1, "limit must be greater than 0");
    LGPU_REQUIRE(p->k <= SELECT_KMAX, "limit+offset above 2048 is not supported on the GPU path");
    if (refine && p->refine_factor)
        LGPU_REQUIRE((uint64_t)p->k * p->refine_factor <= SELECT_KMAX, "limit*refine_factor above 2048 is not supported");
    LGPU_REQUIRE(B == 0 || (q && ids && dist && cnt), "null buffer");
}

// ---- IVF search (IVF_PQ, IVF_SQ and IVF_RQ).  One sub-batch runs [cosine: normalise] -> coarse step (probes) ->
// small scan | regroup -> filter scan + fix-up | exact scan + select -> [refine], on the paths ivf_plan picks before
// any launch ----
enum class Coarse { exact, tc_dense, tc_list };   // see ivf_coarse
enum class IvfScan { small, filter_cand, filter_dense, exact_pq, sq, rq, pq4, ham };

struct IvfPlan {
    uint32_t B, nprobes, slots;
    uint32_t np_eff;          // probes that can hold rows: min(nprobes, nlist)
    uint32_t k, kk;           // the request's k; the PQ top-kk (k, or k * refine_factor candidates for the re-rank)
    uint32_t lb_short;        // dense filter scan: the rows of the lb_short smallest lower bounds are re-scored
    bool refine;
    Coarse coarse;
    IvfScan scan;
    uint32_t cand_cap;        // candidate mode: candidates per query (power of two >= kk)
    bool filter() const { return scan == IvfScan::filter_cand || scan == IvfScan::filter_dense; }
    uint32_t rows_tile() const
    {
        if (filter()) return SCAN3_ROWS_TILE;
        if (scan == IvfScan::pq4) return PQ4_ROWS_TILE;
        if (scan == IvfScan::ham) return HAM_ROWS_TILE;
        return scan == IvfScan::sq ? SQ_ROWS_TILE : (scan == IvfScan::rq ? RQ_ROWS_TILE : SCAN_ROWS_TILE_MID);
    }
};

// prefilter: the request carries an allow bitmap; widening: the sub-batch redoes the queries flagged by the
// maximum_nprobes widening (exact kernels only)
static IvfPlan ivf_plan(const lgpu_index *ix, uint32_t B, uint32_t nprobes, const lgpu_search_params &sp, bool prefilter,
                        bool widening, const ScanModes &modes)
{
    IvfPlan p{};
    const uint32_t nlist = ix->nlist;
    p.B = B; p.nprobes = nprobes; p.slots = B * nprobes; p.np_eff = std::min(nprobes, nlist);
    p.k = sp.k; p.kk = sp.refine_factor ? sp.k * sp.refine_factor : sp.k; p.refine = sp.refine_factor != 0;
    p.lb_short = p.kk <= 16 ? 32u : std::min<uint32_t>(SELECT_KMAX, 2 * p.kk + 32);
    // the bf16 error band around the nprobes-th centroid has to fit in the tensor-core shortlist: 3x nprobes (>= 64)
    // candidates (dense variant) or admission by threshold (list variant).  The tensor-core shortlist wins at every
    // shape measured on 1 x H100 (400 W), down to 64 queries x 1024 lists (coarse step 0.052 vs 0.063 ms; 512 x 1024:
    // 0.082 vs 0.160 ms); smaller problems were not measured and keep the exact kernels.  Many lists (C5: 16384): a
    // dense [B][nlist] score matrix is 537 MB written and read back, so from coarse_list_min lists the list variant.
    const uint32_t coarse_short = std::min<uint32_t>(SELECT_KMAX, std::max<uint32_t>(64, 3 * nprobes));
    const bool big = (uint64_t)B * nlist >= ((uint64_t)1 << 16) || modes.force_tc_coarse;
    p.coarse = Coarse::exact;
    if (ix->has_tc && tc_enabled() && ix->metric != LGPU_DOT && B >= 8 && nlist >= 256 && coarse_short > nprobes && big)
        p.coarse = modes.coarse_list_min && nlist >= modes.coarse_list_min && ix->cent_ns >= 4 * nprobes && nprobes <= 64
                       ? Coarse::tc_list : Coarse::tc_dense;
    // tiny batches (a single query, a micro-batch): the small path, 4 launches instead of ~25; LGPU_SMALL_SLOTS = 0
    // disables it.  Otherwise filter + verify (scan3.cu) unless the request needs every exact distance.
    if (ix->is_pq4) {                  // 4-bit codes: one exact integer scan, never the small or the filter path
        p.scan = IvfScan::pq4;
        return p;
    }
    const bool small = !ix->is_sq && !ix->is_rq && !widening && p.slots <= modes.small_slots &&
                       small_scan_smem(ix->m, ix->dim) <= 200 * 1024 &&
                       (size_t)p.slots * ix->pad_prefix[1] * 4 <= workspace_budget();
    const bool filter = ix->has_tables && !modes.exact && !sp.has_lower && !sp.has_upper && p.lb_short > p.kk &&
                        ix->m <= 512 && !widening && !small;
    if (small) p.scan = IvfScan::small;
    else if (!filter) p.scan = ix->is_sq ? IvfScan::sq : (ix->is_rq ? IvfScan::rq : IvfScan::exact_pq);
    if (!filter) return p;
    // candidate mode (no prefilter, kk <= LGPU_CAND_KMAX): the scanners threshold the rows themselves, nothing dense is
    // written.  LGPU_CAND_CAP shrinks the capacity to exercise the overflow path.
    const uint32_t kk = p.kk, np_eff = p.np_eff;
    uint32_t cap = kk <= 32 ? 512 : (kk <= 64 ? 1024 : CAND_CAP_MAX);
    // long partitions put more rows inside the band around the k-th distance (clustered data: a query near a big blob
    // sees thousands of nearly equidistant rows): give them longer lists rather than the exact fix-up
    const uint64_t rows_probe = std::max<uint64_t>(1, ix->pad_prefix[np_eff] / np_eff);   // mean of the np largest
    if (rows_probe > 16384) cap = std::max<uint32_t>(cap, CAND_CAP_MAX);
    else if (rows_probe > 4096) cap = std::max<uint32_t>(cap, 1024);
    const uint32_t cap_env = modes.cap_env;
    const bool cap_forced = cap_env >= 32 && cap_env <= CAND_CAP_MAX && !(cap_env & (cap_env - 1)) && cap_env >= kk;
    if (cap_forced) cap = cap_env;
    // A tile whose query has no threshold yet appends about k rows.  With few queries fanned out over many tiles
    // (small B, many probes, long partitions) most of a query's tiles run at the same moment on the 2 x SMs CTAs,
    // before any of them has published a threshold, and the list overflows whatever the scanners tighten later:
    // estimate that concurrency from the averages and take the dense mode (cheap at such B) when it is too high.
    bool cand_fits = true;
    if (!cap_forced) {
        const uint64_t tiles_part = (rows_probe + SCAN3_ROWS_TILE - 1) / SCAN3_ROWS_TILE;
        const uint64_t parts = std::min<uint64_t>(nlist, p.slots);
        const uint64_t groups_part = std::max<uint64_t>(1, (p.slots / parts + SCAN_G - 1) / SCAN_G);
        const double total = (double)parts * groups_part * tiles_part;
        const double conc = (double)np_eff * tiles_part * std::min(1.0, 2.0 * ix->num_sms / total);
        cand_fits = conc * kk <= 2.0 * cap;
    }
    p.cand_cap = cap;
    p.scan = !prefilter && kk <= modes.cand_kmax && !modes.dense_forced && cand_fits ? IvfScan::filter_cand
                                                                                     : IvfScan::filter_dense;
    return p;
}

// Profiling (lgpu_last_stage_ms): ws->ev[s] is recorded where stage s ends (IVF_START: where the sub-batch starts).
// A stage the path does not run is read back as ending where the stage before it ended.
enum IvfStage { IVF_START, IVF_COARSE, IVF_PROBES, IVF_REGROUP, IVF_SCAN, IVF_TOPK, IVF_REFINE };
struct StageMarks {
    Workspace *ws;
    bool on;
    void operator()(IvfStage s, cudaStream_t stream) const
    {
        if (on) { cudaEventRecord(ws->ev[s], stream); ws->stages_marked = (s ? ws->stages_marked : 0u) | 1u << s; }
    }
};

// the queries the search runs on: a normalised copy for cosine
static const float *ivf_queries(lgpu_index *ix, Workspace *ws, cudaStream_t st, const float *d_q, uint32_t B)
{
    if (ix->metric != LGPU_COSINE) return d_q;
    ws->qn.ensure((size_t)B * ix->dim * 4);
    launch_normalize(d_q, B, ix->dim, ws->qn.as<float>(), st);
    return ws->qn.as<float>();
}

// The filter scan's per-query tables depend on the queries alone, so they are built on `st` while the coarse step and
// the regroup (a latency chain of small kernels) run on the high-priority side stream `front`, returned here.  The
// search stream joins it (ev_join) before the per-probe terms.
static cudaStream_t fork_front(lgpu_index *ix, Workspace *ws, cudaStream_t st, uint32_t B)
{
    ws->qt.ensure((size_t)B * ix->nch * 256 * 16); ws->qt_mm.ensure((size_t)B * ix->nch * 8 * 8);
    ws->qt_step.ensure((size_t)B * 4); ws->qt_base.ensure((size_t)B * 4); ws->qt_bad.ensure((size_t)B * 4);
    ws->sbound.ensure((size_t)B * 4);
    LGPU_CUDA(cudaEventRecord(ws->ev_fork, st));
    LGPU_CUDA(cudaStreamWaitEvent(ws->front, ws->ev_fork, 0));
    ws->front_open = !g_capturing;
    return ws->front;
}

static void query_tables(lgpu_index *ix, Workspace *ws, const float *qs, uint32_t B, cudaStream_t st)
{
    launch_query_tables_q16(qs, ix->cb_tiled.as<float>(), ix->cb_n2.as<float>(), B, ix->dim, ix->m, ix->nch, ix->dsub,
                            ix->metric, ws->qt_mm.as<float>(), ws->qt.as<uint4>(), ws->qt_step.as<float>(),
                            ws->qt_base.as<float>(), ws->sbound.as<float>(), ws->qt_bad.as<uint32_t>(), st);
}

// Coarse::tc_list up to the finishing kernel: (1) dense scores of a strided SAMPLE of the centroids; their nprobes-th
// smallest + 2 E_q bounds, per query, the scores of every true probe; (2) the full GEMM runs with the filtering epilogue
// and appends (column, score) of the few columns under that bound to the query's list; (3) the finishing kernel works
// on the list (second-level threshold from the list's own nprobes-th smallest, exact re-score, sort).
static void coarse_list(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, uint32_t *cgate,
                        cudaStream_t cs, cudaStream_t st)
{
    const uint32_t B = p.B, nprobes = p.nprobes, dim = ix->dim;
    const uint32_t ns = ix->cent_ns, lds = (ns + 3u) & ~3u, lcap = 1024;
    ws->t_dist.ensure((size_t)B * nprobes * 4); ws->t_ids.ensure((size_t)B * nprobes * 8);
    ws->t_cnt.ensure((size_t)B * 4); ws->probe_A.ensure((size_t)B * 4); ws->amax.ensure((size_t)B * 4);
    ws->t_pos.ensure((size_t)B * lcap * 8); ws->t_exact.ensure((size_t)B * lcap * 4);
    launch_gemm_dist(ws->qb.p, ix->cent_sb.p, ix->cent_sn2.as<float>(), B, ns, dim, ws->D.as<float>(), lds, ix->num_sms, cs);
    if (!launch_sample_kth_threshold(ws->D.as<float>(), lds, ns, ws->qn2.as<float>(), ws->qerr.as<float>(), ix->cent_max,
                                     ix->cent_err, dim, B, nprobes, ws->probe_A.as<float>(), cs)) {
        launch_select(select_rows(ws->D.as<float>(), ns, lds, B, nprobes, {ws->t_ids.as<uint64_t>(),
                                  ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>()}), cs);
        launch_sample_threshold(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->qn2.as<float>(),
                                ws->qerr.as<float>(), ix->cent_max, ix->cent_err, dim, B, nprobes, ws->probe_A.as<float>(),
                                cs);
    }
    LGPU_CUDA(cudaMemsetAsync(ws->amax.p, 0, (size_t)B * 4, cs));
    GemmFilter flt{};
    flt.thr = ws->probe_A.as<float>(); flt.count = ws->amax.as<uint32_t>(); flt.cand_pos = ws->t_pos.as<uint64_t>();
    flt.cand_ids = nullptr; flt.col_ids = nullptr; flt.cap = lcap; flt.cand_s = ws->t_exact.as<float>();
    launch_gemm_dist(ws->qb.p, ix->cent_b.p, ix->cent_n2.as<float>(), B, ix->nlist, dim, nullptr, 0, ix->num_sms, cs, &flt);
    if (p.filter()) query_tables(ix, ws, qs, B, st);
    launch_coarse_finish(ws->t_exact.as<float>(), lcap, B, lcap, qs, ix->centroids.as<float>(), ws->qn2.as<float>(),
                         ws->qerr.as<float>(), ix->cent_max, ix->cent_err, dim, nprobes, ws->probes.as<uint64_t>(),
                         ws->probe_dist.as<float>(), ws->probe_cnt.as<uint32_t>(), ws->flags.as<uint32_t>(), cgate, cs,
                         ws->t_pos.as<uint64_t>(), ws->amax.as<uint32_t>());
}

// The nprobes nearest partitions of every query into ws->probes / probe_dist / probe_cnt, on `cs`.  With the filter
// scan the query tables go on `st`: right after the coarse GEMM (tensor-core variants), so that the GEMM's CTAs (each
// needs most of an SM's shared memory) are not queued behind the table grids and, as SMs free up, the probe selection
// after it is dispatched ahead of the waiting table CTAs by the priority of `front` (making the tables wait for the GEMM
// to finish was measured slower: the tables are then the longer branch); after the probe select (exact variant).
static void ivf_coarse(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, cudaStream_t cs,
                       cudaStream_t st, const StageMarks &mark)
{
    const uint32_t B = p.B, nprobes = p.nprobes, nlist = ix->nlist, dim = ix->dim;
    ws->probes.ensure((size_t)p.slots * 8);
    ws->probe_dist.ensure((size_t)p.slots * 4);
    ws->probe_cnt.ensure((size_t)B * 4);
    const uint64_t ldc = (nlist + 3u) & ~3u;
    ws->D.ensure((size_t)B * ldc * 4);
    const TopkOut probes{ws->probes.as<uint64_t>(), ws->probe_dist.as<float>(), ws->probe_cnt.as<uint32_t>()};
    if (p.coarse == Coarse::exact) {
        launch_dist_matrix(qs, ix->centroids.as<float>(), B, nlist, dim, ix->metric == LGPU_DOT ? 1 : 0, nullptr, nullptr,
                           ws->D.as<float>(), ldc, cs);
        mark(IVF_COARSE, cs);
        launch_select(select_rows(ws->D.as<float>(), nlist, ldc, B, nprobes, probes), cs);
        if (p.filter()) query_tables(ix, ws, qs, B, st);
        return;
    }
    // tensor-core GEMM scores + one finishing kernel per query (threshold, exact re-score in lance order, top nprobes):
    // bit-identical probe sets; queries whose candidate band overflowed are redone exactly
    mark(IVF_COARSE, cs);
    ws->qb.ensure((size_t)B * dim * 2); ws->qn2.ensure((size_t)B * 4); ws->qerr.ensure((size_t)B * 4);
    ws->flags.ensure((size_t)B * 4);
    ws->c_wcnt.ensure(16);
    uint32_t *cgate = ws->c_wcnt.as<uint32_t>() + 2;    // 0 = no query overflowed: the exact fix-up returns at once
    launch_to_bf16(qs, B, dim, ws->qb.p, ws->qn2.as<float>(), cs, ws->qerr.as<float>());
    if (p.coarse == Coarse::tc_list) {
        coarse_list(ix, ws, p, qs, cgate, cs, st);
    } else {
        launch_gemm_dist(ws->qb.p, ix->cent_b.p, ix->cent_n2.as<float>(), B, nlist, dim, ws->D.as<float>(), ldc,
                         ix->num_sms, cs);
        if (p.filter()) query_tables(ix, ws, qs, B, st);
        launch_coarse_finish(ws->D.as<float>(), ldc, B, nlist, qs, ix->centroids.as<float>(), ws->qn2.as<float>(),
                             ws->qerr.as<float>(), ix->cent_max, ix->cent_err, dim, nprobes, ws->probes.as<uint64_t>(),
                             ws->probe_dist.as<float>(), ws->probe_cnt.as<uint32_t>(), ws->flags.as<uint32_t>(), cgate, cs);
    }
    launch_dist_matrix(qs, ix->centroids.as<float>(), B, nlist, dim, 0, nullptr, nullptr, ws->D.as<float>(), ldc, cs,
                       ws->flags.as<uint32_t>(), cgate);
    SelectArgs sc = select_rows(ws->D.as<float>(), nlist, ldc, B, nprobes, probes);
    sc.only = ws->flags.as<uint32_t>(); sc.gate = cgate;
    launch_select(sc, cs);
}

// mode 0: the k best rows of every query's probed segments of ws->dist_out, prefilter applied before the top-k
static SelectArgs select_segments(lgpu_index *ix, Workspace *ws, const IvfPlan &p, uint32_t k, TopkOut out, RowFilter rf)
{
    SelectArgs s = select_args(0, p.B, k, out);
    s.dist = ws->dist_out.as<float>(); s.seg_off = ws->seg_off.as<uint64_t>(); s.probes = ws->probes.as<uint64_t>();
    s.nprobes = p.nprobes; s.nlist = ix->nlist; s.part_n = ix->part_n.as<uint32_t>();
    s.part_off = ix->part_off.as<uint64_t>(); s.row_ids = ix->row_ids.as<uint64_t>();
    s.allow = rf.bits; s.allow_bits = rf.nbits;
    return s;
}

// where the PQ top-kk goes: straight to the caller, or to the refine stage's candidate lists
static TopkOut pq_out(Workspace *ws, const IvfPlan &p, TopkOut out)
{
    if (!p.refine) return out;
    const size_t n = (size_t)p.B * p.kk;
    ws->t_ids.ensure(n * 8); ws->t_dist.ensure(n * 4); ws->t_pos.ensure(n * 8); ws->t_cnt.ensure((size_t)p.B * 4);
    ws->t_exact.ensure(n * 4);
    return {ws->t_ids.as<uint64_t>(), ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->t_pos.as<uint64_t>()};
}

// IvfScan::small: small_scan into one segment per probe slot, then the PQ top-kk
static void ivf_small(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const lgpu_search_params &sp, const float *qs,
                      RowFilter rf, TopkOut out, cudaStream_t st, const StageMarks &mark)
{
    const uint64_t stride = std::max<uint64_t>(ix->pad_prefix[1], 4);
    ws->seg_off.ensure((size_t)p.slots * 8);
    ws->dist_out.ensure((size_t)p.slots * stride * 4);
    SmallScanArgs ss{};
    ss.centroids = ix->centroids.as<float>(); ss.cb_tiled = ix->cb_tiled.as<float>();
    ss.codes = ix->codes.as<unsigned char>(); ss.code_base = ix->code_base.as<uint64_t>();
    ss.part_n = ix->part_n.as<uint32_t>(); ss.part_npad = ix->part_npad.as<uint32_t>();
    ss.dim = ix->dim; ss.m = ix->m; ss.nch = ix->nch; ss.metric = (uint32_t)ix->metric; ss.nlist = ix->nlist;
    ss.nprobes = p.nprobes;
    ss.queries = qs; ss.probes = ws->probes.as<uint64_t>(); ss.seg_stride = stride;
    ss.seg_off = ws->seg_off.as<uint64_t>(); ss.dist_out = ws->dist_out.as<float>();
    launch_small_scan(ss, ix->dsub, p.slots, st);
    mark(IVF_SCAN, st);
    SelectArgs sa = select_segments(ix, ws, p, p.kk, pq_out(ws, p, out), rf);
    with_range(sa, sp);
    launch_select(sa, st);
    mark(IVF_TOPK, st);
}

// regroup the probe slots by partition into tiles of p.rows_tile() rows (group.cu) on `cs`, and size ws->dist_out for
// the distance segments.  only (device, [B]): just the flagged queries.
static GroupArgs ivf_regroup(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const uint32_t *only, cudaStream_t cs)
{
    const uint32_t B = p.B, slots = p.slots, nlist = ix->nlist;
    ws->part_cnt.ensure((size_t)nlist * 4);
    ws->slot_pos.ensure((size_t)slots * 4);
    ws->seg_local.ensure((size_t)slots * 8);
    ws->qtot.ensure((size_t)B * 8);
    ws->seg_off.ensure((size_t)slots * 8);
    ws->qlist_off.ensure((size_t)nlist * 4);
    ws->tile_off.ensure((size_t)(nlist + 1) * 4); ws->tile_off_b.ensure((size_t)(nlist + 1) * 4);
    ws->qlist.ensure((size_t)slots * 4);
    ws->scalars.ensure(64);
    GroupArgs ga{};
    ga.probes = ws->probes.as<uint64_t>(); ga.B = B; ga.nprobes = p.nprobes; ga.nlist = nlist;
    ga.part_n = ix->part_n.as<uint32_t>(); ga.part_cnt = ws->part_cnt.as<uint32_t>();
    ga.part_npad = ix->part_npad.as<uint32_t>(); ga.code_base = ix->code_base.as<uint64_t>(); ga.part_off = ix->part_off.as<uint64_t>();
    ga.slot_pos = ws->slot_pos.as<uint32_t>(); ga.seg_local = ws->seg_local.as<uint64_t>();
    ga.qtot = ws->qtot.as<uint64_t>(); ga.seg_off = ws->seg_off.as<uint64_t>();
    ga.qlist_off = ws->qlist_off.as<uint32_t>(); ga.tile_off = ws->tile_off.as<uint32_t>(); ga.tile_off_b = ws->tile_off_b.as<uint32_t>();
    ga.qlist = ws->qlist.as<uint32_t>();
    ga.total_tiles = ws->scalars.as<uint32_t>(); ga.tile_counter = ws->scalars.as<uint32_t>() + 1;
    ga.scanned_rows = reinterpret_cast<unsigned long long *>(ws->scalars.as<char>() + 16);
    // tile descriptors, sized by a host bound on the tile count (for 1536-row tiles; 3072-row tiles need fewer)
    // sum_p ceil(cnt_p / 8) * nrb_p <= (slots / 8 + #probed partitions) * max_p nrb_p
    const uint64_t max_tiles = ((uint64_t)slots / SCAN_G + std::min<uint64_t>(nlist, slots) + 1) * ix->max_nrb;
    LGPU_REQUIRE(max_tiles < (1ull << 31), "batch too large for one scan launch");
    ws->tile_desc.ensure((size_t)max_tiles * sizeof(TileDesc));
    ga.tile_desc = ws->tile_desc.as<TileDesc>(); ga.max_tiles = (uint32_t)max_tiles;
    ga.only = only;
    ga.rows_tile = p.rows_tile();
    launch_group(ga, cs);
    ws->dist_out.ensure(std::max<size_t>((size_t)B * ix->pad_prefix[p.np_eff], 4) * 4);
    return ga;
}

// the arguments scan2 and scan3 share: the regrouped tiles, the distance segments
static ScanArgs scan_args(lgpu_index *ix, Workspace *ws, const float *qs, const GroupArgs &ga)
{
    ScanArgs sc{};
    sc.centroids = ix->centroids.as<float>(); sc.cb_tiled = ix->cb_tiled.as<float>();
    sc.codes = ix->codes.as<unsigned char>(); sc.code_base = ix->code_base.as<uint64_t>();
    sc.part_n = ix->part_n.as<uint32_t>(); sc.part_npad = ix->part_npad.as<uint32_t>();
    sc.dim = ix->dim; sc.m = ix->m; sc.nch = ix->nch; sc.metric = (uint32_t)ix->metric; sc.nlist = ix->nlist;
    sc.rows_tile = ga.rows_tile; sc.fzero2 = 0ull;
    sc.queries = qs;
    sc.total_tiles = ga.total_tiles; sc.tile_counter = ga.tile_counter;
    sc.dist_out = ws->dist_out.as<float>();
    sc.tile_desc = ga.tile_desc;
    sc.part_off = ix->part_off.as<uint64_t>();
    return sc;
}

// IvfScan::pq4: the per-slot u8 tables of every probe slot (after the coarse step), then the scan's arguments
static void pq4_tables(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, cudaStream_t st)
{
    ws->pq4_tab.ensure((size_t)p.slots * ix->m * 16);
    ws->pq4_slots.ensure((size_t)p.slots * sizeof(Pq4Slot));
    launch_pq4_tables(qs, ix->centroids.as<float>(), ix->pq4_cb.as<float>(), ws->probes.as<uint64_t>(), p.slots,
                      p.nprobes, ix->nlist, ix->m, ix->dsub, ix->metric, ws->pq4_tab.as<uint8_t>(),
                      ws->pq4_slots.as<Pq4Slot>(), st);
}

static Pq4ScanArgs pq4_args(lgpu_index *ix, Workspace *ws, const GroupArgs &ga)
{
    Pq4ScanArgs a{};
    a.codes = ix->codes.as<uint32_t>(); a.tables = ws->pq4_tab.as<uint8_t>(); a.slots = ws->pq4_slots.as<Pq4Slot>();
    a.m = ix->m; a.metric = (uint32_t)ix->metric;
    a.total_tiles = ga.total_tiles; a.tile_counter = ga.tile_counter; a.tile_desc = ga.tile_desc;
    a.dist_out = ws->dist_out.as<float>();
    return a;
}

// The filter scan's prologue on `st`: its buffers, the join with `front` (probes and regroup), the per-probe terms and
// the 16-bit per-query tables in `sc`
static void filter_terms(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, ScanArgs &sc, cudaStream_t st)
{
    const uint32_t B = p.B, kp = p.lb_short;
    const bool dot = ix->metric == LGPU_DOT;
    ws->flags.ensure((size_t)B * 4); ws->c_wcnt.ensure(16); ws->c_surv.ensure((size_t)B * 4);
    ws->s_ids.ensure((size_t)B * kp * 8); ws->s_lb.ensure((size_t)B * kp * 4); ws->s_pos.ensure((size_t)B * kp * 8);
    ws->s_cnt.ensure((size_t)B * 4); ws->s_exact.ensure((size_t)B * kp * 4);
    LGPU_CUDA(cudaStreamWaitEvent(st, ws->ev_join, 0));
    ws->front_open = false;
    ws->qn2.ensure((size_t)B * 4);
    if (!dot) {
        ws->probe_A.ensure((size_t)p.slots * 4); ws->amax.ensure((size_t)B * 4);
        sc.probe_A = ws->probe_A.as<float>(); sc.row_R = ix->row_R.as<float>();
    }
    launch_probe_terms(ws->probe_dist.as<float>(), qs, B, p.nprobes, ix->dim, dot ? nullptr : ws->probe_A.as<float>(),
                       dot ? nullptr : ws->amax.as<float>(), ws->qn2.as<float>(), ws->qt_base.as<float>(),
                       ws->qt_bad.as<uint32_t>(), st);
    sc.qt = ws->qt.as<uint4>(); sc.qt_step = ws->qt_step.as<float>(); sc.qt_base = ws->qt_base.as<float>();
}

// IvfScan::filter_cand: scan3 appends the rows under each query's threshold to its candidate list, the finalize kernel
// re-scores them exactly into the PQ top-kk and flags the queries it cannot prove
static void filter_candidates(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, ScanArgs &sc,
                              TopkOut pq, bool prof, cudaStream_t st, const StageMarks &mark)
{
    const uint32_t B = p.B, cap = p.cand_cap;
    const bool dot = ix->metric == LGPU_DOT;
    const float mscale = ix->metric == LGPU_COSINE ? 0.5f : 1.0f;
    ws->c_thr.ensure((size_t)B * 4); ws->c_slack.ensure((size_t)B * 4); ws->c_cnt.ensure((size_t)B * 4);
    ws->c_rec.ensure((size_t)B * cap * sizeof(CandRec));
    ws->c_key.ensure((size_t)B * cap * 4); ws->c_last.ensure((size_t)B * 4);
    launch_cand_prepare(ws->qt_step.as<float>(), ws->sbound.as<float>(), dot ? nullptr : ws->amax.as<float>(),
                        dot ? nullptr : ix->rmax_bits.as<int>(), ws->qn2.as<float>(), ix->cb2, mscale, ix->m, dot, B,
                        ws->c_slack.as<float>(), ws->c_thr.as<uint32_t>(), ws->c_cnt.as<uint32_t>(),
                        ws->c_last.as<uint32_t>(), ws->c_key.as<uint32_t>(), cap, st);
    sc.cand_key = ws->c_key.as<uint32_t>(); sc.cand_last = ws->c_last.as<uint32_t>();
    sc.nprobes = p.nprobes; sc.topk = p.kk; sc.thr = ws->c_thr.as<uint32_t>(); sc.slack = ws->c_slack.as<float>();
    sc.cand_cnt = ws->c_cnt.as<uint32_t>(); sc.cand = ws->c_rec.as<CandRec>(); sc.cand_cap = cap;
    launch_scan3(sc, ix->num_sms, st);
    mark(IVF_SCAN, st);
    FinalizeArgs fa{};
    fa.Q = qs; fa.cand = sc.cand; fa.cand_cnt = sc.cand_cnt; fa.cand_cap = cap; fa.cand_key = sc.cand_key; fa.thr = sc.thr;
    fa.slack = sc.slack; fa.bad = ws->qt_bad.as<uint32_t>();
    fa.codes = ix->codes.as<unsigned char>(); fa.code_base = ix->code_base.as<uint64_t>();
    fa.part_npad = ix->part_npad.as<uint32_t>(); fa.part_off = ix->part_off.as<uint64_t>();
    fa.row_ids = ix->row_ids.as<uint64_t>(); fa.centroids = ix->centroids.as<float>();
    fa.cb_tiled = ix->cb_tiled.as<float>();
    fa.B = B; fa.dim = ix->dim; fa.m = ix->m; fa.dsub = ix->dsub; fa.k = p.kk; fa.metric = ix->metric;
    fa.out_ids = pq.ids; fa.out_dist = pq.dist; fa.out_count = pq.cnt; fa.out_pos = pq.pos;
    fa.flags = ws->flags.as<uint32_t>();
    ws->c_work.ensure((size_t)B * cap * 8); ws->c_wcnt.ensure(16); ws->c_surv.ensure((size_t)B * 4);
    ws->c_exd.ensure((size_t)B * cap * 4); ws->c_exi.ensure((size_t)B * cap * 8); ws->c_exp.ensure((size_t)B * cap * 8);
    fa.work = ws->c_work.as<uint2>(); fa.work_cnt = ws->c_wcnt.as<uint32_t>(); fa.surv_cnt = ws->c_surv.as<uint32_t>();
    fa.ex_dist = ws->c_exd.as<float>(); fa.ex_id = ws->c_exi.as<uint64_t>(); fa.ex_pos = ws->c_exp.as<uint64_t>();
    fa.num_sms = ix->num_sms;
    if (prof) {
        ws->c_stats.ensure(32);
        LGPU_CUDA(cudaMemsetAsync(ws->c_stats.p, 0, 32, st));
        fa.stats = ws->c_stats.as<unsigned long long>();
        ws->stats_mode = 1;
    }
    launch_cand_finalize(fa, st);
    sc.cand = nullptr;                      // (the fix-up pass is the exact kernel)
}

// IvfScan::filter_dense: scan3 writes a lower bound per row; the lb_short smallest are re-scored exactly (oracle
// arithmetic) into the PQ top-kk, and the queries the band check cannot prove are flagged
static void filter_dense(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *qs, const ScanArgs &sc,
                         RowFilter rf, TopkOut pq, cudaStream_t st, const StageMarks &mark)
{
    const uint32_t B = p.B, kp = p.lb_short;
    const bool dot = ix->metric == LGPU_DOT;
    const float mscale = ix->metric == LGPU_COSINE ? 0.5f : 1.0f;
    launch_scan3(sc, ix->num_sms, st);
    mark(IVF_SCAN, st);
    launch_select(select_segments(ix, ws, p, kp, {ws->s_ids.as<uint64_t>(), ws->s_lb.as<float>(),
                                  ws->s_cnt.as<uint32_t>(), ws->s_pos.as<uint64_t>()}, rf), st);
    ws->stats_mode = 2;
    launch_band_check3(ws->s_lb.as<float>(), ws->s_cnt.as<uint32_t>(), ws->qt_step.as<float>(), ws->sbound.as<float>(),
                       dot ? nullptr : ws->amax.as<float>(), dot ? nullptr : ix->rmax_bits.as<int>(),
                       ws->qt_bad.as<uint32_t>(), ws->qn2.as<float>(), ix->cb2, mscale, ix->m, dot, B, p.kk, kp,
                       ws->flags.as<uint32_t>(), ws->c_wcnt.as<uint32_t>() + 1, ws->c_surv.as<uint32_t>(), st);
    launch_pq_rescore(qs, ws->s_pos.as<uint64_t>(), B, kp, ix->codes.as<unsigned char>(), ix->code_base.as<uint64_t>(),
                      ix->part_npad.as<uint32_t>(), ix->part_off.as<uint64_t>(), ix->nlist, ix->centroids.as<float>(),
                      ix->cb_tiled.as<float>(), ix->dim, ix->m, ix->dsub, ix->metric, ws->c_surv.as<uint32_t>(),
                      ws->s_exact.as<float>(), st);
    SelectArgs sb = select_cands(ws->s_exact.as<float>(), ws->s_ids.as<uint64_t>(), kp, B, p.kk, pq);
    sb.cand_pos = ws->s_pos.as<uint64_t>(); sb.ncols_q = ws->c_surv.as<uint32_t>();
    launch_select(sb, st);
}

// fix-up of the queries the filter scan could not prove (ws->flags): regroup them alone, exact scan, exact top-kk over
// their segments.  Always issued: with nothing flagged the gate is 0 and every kernel returns at once.
static void filter_fixup(lgpu_index *ix, Workspace *ws, const IvfPlan &p, GroupArgs ga, ScanArgs sc, RowFilter rf,
                         TopkOut pq, cudaStream_t st)
{
    const uint32_t *gate = ws->c_wcnt.as<uint32_t>() + 1;
    ga.only = ws->flags.as<uint32_t>(); ga.gate = gate;
    ga.rows_tile = SCAN_ROWS_TILE_MID;
    launch_group(ga, st);
    sc.rows_tile = SCAN_ROWS_TILE_MID; sc.gate = gate;
    launch_scan2(sc, ix->dsub, ix->num_sms, st);
    SelectArgs sf = select_segments(ix, ws, p, p.kk, pq, rf);
    sf.only = ws->flags.as<uint32_t>(); sf.gate = gate;
    launch_select(sf, st);
}

// IvfScan::exact_pq / sq / rq: the exact scan of every regrouped tile, then the PQ top-kk
static void ivf_exact(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const lgpu_search_params &sp, const float *qs,
                      const GroupArgs &ga, RowFilter rf, const uint32_t *only, TopkOut pq, cudaStream_t st,
                      const StageMarks &mark)
{
    if (p.scan == IvfScan::sq) {
        SqScanArgs qa{};
        qa.codes = ix->codes.as<uint8_t>(); qa.xx = ix->sq_xx.as<uint32_t>();
        qa.qcodes = ws->sq_q.as<uint8_t>(); qa.qq = ws->sq_qq.as<uint32_t>(); qa.dim_pad = ix->dim_pad;
        qa.total_tiles = ga.total_tiles; qa.tile_counter = ga.tile_counter; qa.tile_desc = ga.tile_desc;
        qa.dist_out = ws->dist_out.as<float>();
        launch_sq_scan(qa, 2 * ix->num_sms, st);
    } else if (p.scan == IvfScan::rq) {
        RqScanArgs ra{};
        ra.codes = ix->codes.as<uint32_t>(); ra.add = ix->rq_add.as<float>(); ra.scale = ix->rq_scale.as<float>();
        ra.popc = ix->rq_popc.as<uint32_t>();
        ra.planes = ws->rq_planes.as<uint32_t>(); ra.slots = ws->rq_slots.as<RqSlot>();
        ra.dim = ix->dim; ra.wpr = ix->rq_wpr; ra.cosine = ix->metric == LGPU_COSINE;
        ra.total_tiles = ga.total_tiles; ra.tile_counter = ga.tile_counter; ra.tile_desc = ga.tile_desc;
        ra.dist_out = ws->dist_out.as<float>();
        launch_rq_scan(ra, 2 * ix->num_sms, st);
    } else if (p.scan == IvfScan::pq4) {
        launch_pq4_scan(pq4_args(ix, ws, ga), 2 * ix->num_sms, st);
    } else {
        launch_scan2(scan_args(ix, ws, qs, ga), ix->dsub, ix->num_sms, st);
    }
    mark(IVF_SCAN, st);
    SelectArgs sa = select_segments(ix, ws, p, p.kk, pq, rf);
    sa.only = only;
    with_range(sa, sp);
    launch_select(sa, st);
    mark(IVF_TOPK, st);
}

// refine (query.rs:1302-1332): exact distance of the k * refine_factor candidates (ws->t_*), re-sort into `out`
static void ivf_refine(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *d_q, TopkOut out,
                       const uint32_t *only, cudaStream_t st)
{
    launch_pair_distance(d_q, ix->vectors.as<float>(), ws->t_pos.as<uint64_t>(), p.B, p.kk, ix->dim, ix->metric,
                         ws->t_exact.as<float>(), st);
    SelectArgs sr = select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), p.kk, p.B, p.k, out);
    sr.only = only;
    launch_select(sr, st);
}

// one sub-batch of an IVF_PQ / IVF_SQ / IVF_RQ search, everything device-side on `st` (and `front`, joined).  only
// (device, [B]): redo just the flagged queries (maximum_nprobes widening) -- exact kernels, the other queries' outputs
// are left untouched.
void ivf_sub_batch(lgpu_index *ix, Workspace *ws, cudaStream_t st, const float *d_q, uint32_t B,
                   const lgpu_search_params &sp, uint32_t nprobes, TopkOut out, bool prof, RowFilter rf,
                   const uint32_t *only = nullptr)
{
    const IvfPlan p = ivf_plan(ix, B, nprobes, sp, rf.bits != nullptr, only != nullptr, scan_modes());
    const StageMarks mark{ws, prof};
    mark(IVF_START, st);
    ws->stats_mode = 0;
    const float *qs = ivf_queries(ix, ws, st, d_q, B);
    const cudaStream_t cs = p.filter() ? fork_front(ix, ws, st, B) : st;   // the coarse step's and the regroup's
    ivf_coarse(ix, ws, p, qs, cs, st, mark);
    if (p.scan == IvfScan::sq) {
        ws->sq_q.ensure((size_t)B * ix->dim_pad); ws->sq_qq.ensure((size_t)B * 4);
        launch_sq_encode(qs, B, ix->dim, ix->dim_pad, ix->sq_lo, ix->sq_hi, ws->sq_q.as<uint8_t>(),
                         ws->sq_qq.as<uint32_t>(), st);
    } else if (p.scan == IvfScan::rq) {        // rotate the queries, then each probe slot's 4-bit grid of q - c_p
        ws->rq_q.ensure((size_t)B * ix->dim * 4);
        ws->rq_planes.ensure((size_t)p.slots * 4 * ix->rq_wpr * 4);
        ws->rq_slots.ensure((size_t)p.slots * sizeof(RqSlot));
        launch_rq_rotate(ix->rq_rot.as<float>(), qs, B, ix->dim, ws->rq_q.as<float>(), st);
        launch_rq_planes(ws->rq_q.as<float>(), ix->rq_rc.as<float>(), ws->probes.as<uint64_t>(), p.slots, nprobes,
                         ix->nlist, ix->dim, ix->rq_wpr, ws->rq_planes.as<uint32_t>(), ws->rq_slots.as<RqSlot>(), st);
    } else if (p.scan == IvfScan::pq4) {
        pq4_tables(ix, ws, p, qs, st);
    }
    mark(IVF_PROBES, cs);
    if (p.scan == IvfScan::small) {
        ivf_small(ix, ws, p, sp, qs, rf, out, st, mark);
    } else {
        const GroupArgs ga = ivf_regroup(ix, ws, p, only, cs);
        mark(IVF_REGROUP, cs);
        const TopkOut pq = pq_out(ws, p, out);
        if (p.filter()) {
            LGPU_CUDA(cudaEventRecord(ws->ev_join, ws->front));
            ScanArgs sc = scan_args(ix, ws, qs, ga);
            filter_terms(ix, ws, p, qs, sc, st);
            if (p.scan == IvfScan::filter_cand) filter_candidates(ix, ws, p, qs, sc, pq, prof, st, mark);
            else filter_dense(ix, ws, p, qs, sc, rf, pq, st, mark);
            filter_fixup(ix, ws, p, ga, sc, rf, pq, st);
            mark(IVF_TOPK, st);
        } else {
            ivf_exact(ix, ws, p, sp, qs, ga, rf, only, pq, st, mark);
        }
    }
    if (!p.refine) return;
    ivf_refine(ix, ws, p, d_q, out, only, st);
    mark(IVF_REFINE, st);
}

uint32_t ivf_sub_batch_size(lgpu_index *ix, uint32_t B, uint32_t nprobes)
{
    uint32_t np_eff = std::min<uint32_t>(nprobes, ix->nlist);
    size_t per_q = std::max<size_t>(ix->pad_prefix[np_eff] * 4 + (size_t)ix->nlist * 4 + (size_t)ix->nch * 256 * 8 * 4, 4);
    if (ix->is_rq) per_q += (size_t)nprobes * (16 * ix->rq_wpr + sizeof(RqSlot)) + (size_t)ix->dim * 4;  // planes, rq
    if (ix->is_pq4) per_q += (size_t)nprobes * (16 * ix->m + sizeof(Pq4Slot));                        // u8 tables
    size_t bs = workspace_budget() / per_q;
    // tile descriptors address the distance segments with 32-bit float offsets
    bs = std::min<size_t>(bs, (size_t)0xffffffffull / std::max<size_t>(ix->pad_prefix[np_eff], 1));
    bs = std::max<size_t>(1, std::min<size_t>(bs, 65535));
    return (uint32_t)std::min<size_t>(bs, B);
}

// After a profiled IVF sub-batch: its stage times are added to g_stage_ms; returns the rows its regroup handed to the
// scan (the small path has no regroup and counts none).  Synchronises `st`.
static uint64_t add_stage_marks(Workspace *ws, cudaStream_t st)
{
    LGPU_CUDA(cudaStreamSynchronize(st));
    cudaEvent_t end[7];
    for (int i = 0; i < 7; i++) end[i] = i == 0 || (ws->stages_marked >> i & 1) ? ws->ev[i] : end[i - 1];
    for (int i = 0; i < 7; i++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, i < 6 ? end[i] : end[0], i < 6 ? end[i + 1] : end[6]);
        g_stage_ms[i] += ms;
    }
    unsigned long long rows = 0;
    if (ws->stages_marked >> IVF_REGROUP & 1)
        LGPU_CUDA(cudaMemcpy(&rows, ws->scalars.as<char>() + 16, 8, cudaMemcpyDeviceToHost));
    return rows;
}

// Profiling covers the whole call: every sub-batch's first pass is marked and read back here (a synchronisation per
// sub-batch, which profiling accepts), its stage times, scanned rows and filter counters added to the call's.  The
// maximum_nprobes widening pass is not part of any of them.  b: the sub-batch's queries (ws->flags holds b flags).
static uint64_t add_ivf_profile(Workspace *ws, cudaStream_t st, uint32_t b)
{
    const uint64_t rows = add_stage_marks(ws, st);
    if (ws->stats_mode == 1) {
        uint64_t s[4];
        LGPU_CUDA(cudaMemcpy(s, ws->c_stats.p, 32, cudaMemcpyDeviceToHost));
        for (int i = 0; i < 4; i++) g_filter_stats[i] += s[i];
    } else if (ws->stats_mode == 2) {                       // dense filter: queries the band check could not prove
        std::vector<uint32_t> fl(b);
        LGPU_CUDA(cudaMemcpy(fl.data(), ws->flags.p, (size_t)b * 4, cudaMemcpyDeviceToHost));
        for (uint32_t f : fl) g_filter_stats[2] += f ? 1 : 0;
        g_filter_stats[3] += b;
    }
    return rows;
}

void ivf_search_device(lgpu_index *ix, Workspace *ws, cudaStream_t st, const float *d_q, uint32_t B,
                       const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                       RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint32_t nprobes = std::min<uint32_t>(std::max<uint32_t>(sp.nprobes, 1), ix->nlist);
    const uint32_t np_widest = rf.bits ? std::max(nprobes, std::min<uint32_t>(sp.max_nprobes, ix->nlist)) : nprobes;
    const uint32_t bs = ivf_sub_batch_size(ix, B, np_widest);
    const bool prof = profiling_enabled();
    const uint32_t row_bytes = ix->is_sq ? ix->dim : ix->is_rq ? ix->rq_wpr * 4 : ix->is_pq4 ? ix->m / 2 : ix->m;
    if (prof) {
        memset(g_stage_ms, 0, sizeof(g_stage_ms));
        memset(g_filter_stats, 0, sizeof(g_filter_stats));
        g_scanned_bytes = 0;
    }
    const TopkOut out{d_ids, d_dist, d_cnt};
    for (uint32_t q0 = 0; q0 < B; q0 += bs) {
        uint32_t b = std::min(bs, B - q0);
        if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);      // the previous sub-batch, or LGPU_TIMEOUT
        const float *q = d_q + (size_t)q0 * ix->dim;
        ivf_sub_batch(ix, ws, st, q, b, sp, nprobes, out.at(q0, sp.k), prof, rf);
        if (prof) g_scanned_bytes += add_ivf_profile(ws, st, b) * row_bytes;
        // maximum_nprobes (query.rs:1250-1275): under a prefilter, the queries that found fewer than k rows in their
        // minimum_nprobes partitions are searched again over their maximum_nprobes nearest (no work if none is)
        const uint32_t np_max = std::min<uint32_t>(sp.max_nprobes, ix->nlist);
        if (rf.bits && np_max > nprobes) {
            LGPU_REQUIRE(np_max <= SELECT_KMAX || np_max >= ix->nlist, "maximum_nprobes above 2048 is not supported");
            ws->widen.ensure((size_t)b * 4);
            launch_count_below(out.at(q0, sp.k).cnt, b, sp.k, ws->widen.as<uint32_t>(), st);
            ivf_sub_batch(ix, ws, st, q, b, sp, np_max, out.at(q0, sp.k), false, rf, ws->widen.as<uint32_t>());
        }
    }
}

void flat_search_device(lgpu_flat *fl, Workspace *ws, cudaStream_t st, int metric, const float *d_q, uint32_t B,
                        const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                        RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint64_t N = fl->nrows;
    const uint64_t ld = (N + 3) & ~3ull;
    if (metric == LGPU_COSINE) {
        std::lock_guard<std::mutex> g(fl->mu);
        if (!fl->has_norms) {
            fl->ysqrt.ensure(std::max<size_t>(N, 1) * 4);
            launch_row_norms(fl->vectors.as<float>(), N, fl->dim, fl->ysqrt.as<float>(), st);
            LGPU_CUDA(cudaStreamSynchronize(st));
            fl->has_norms = true;
        }
    }
    size_t per_q = std::max<size_t>(ld * 4, 4);
    uint32_t bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(workspace_budget() / per_q, B));
    const TopkOut out{d_ids, d_dist, d_cnt};
    for (uint32_t q0 = 0; q0 < B; q0 += bs) {
        uint32_t b = std::min(bs, B - q0);
        if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);
        const float *q = d_q + (size_t)q0 * fl->dim;
        ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
        const float *xn = nullptr;
        if (metric == LGPU_COSINE) {
            ws->xnorm.ensure((size_t)b * 4);
            launch_row_norms(q, b, fl->dim, ws->xnorm.as<float>(), st);
            xn = ws->xnorm.as<float>();
        }
        const uint32_t kp = (uint32_t)std::min<uint64_t>(N, std::min<uint32_t>(SELECT_KMAX, std::max<uint32_t>(8 * sp.k, 256)));
        // (a prefilter goes through the exact kernels: the shortlist thresholds are fixed on unfiltered rows)
        if (fl->has_tc && tc_enabled() && metric == LGPU_L2 && !sp.has_lower && !sp.has_upper && b >= 8 && N >= 4096 &&
            !rf.bits) {
            if (N >= 262144 && !getenv("LGPU_FLAT_DENSE"))
                tc_topk_l2_filtered(ws, st, fl->num_sms, q, b, fl->vectors.as<float>(), fl->vec_b.p,
                                    fl->vec_n2.as<float>(), fl->vec_max, fl->vec_err, N, fl->dim,
                                    fl->has_ids ? fl->row_ids.as<uint64_t>() : nullptr, sp.k, out.at(q0, sp.k),
                                    ws->D.as<float>(), ld);
            else
                tc_topk_l2(ws, st, fl->num_sms, q, b, fl->vectors.as<float>(), fl->vec_b.p, fl->vec_n2.as<float>(),
                           fl->vec_max, fl->vec_err, N, fl->dim, fl->has_ids ? fl->row_ids.as<uint64_t>() : nullptr, sp.k, kp,
                           out.at(q0, sp.k), ws->D.as<float>(), ld);
            continue;
        }
        launch_dist_matrix(q, fl->vectors.as<float>(), b, N, fl->dim, metric == LGPU_L2 ? 0 : (metric == LGPU_DOT ? 1 : 2),
                           xn, fl->ysqrt.as<float>(), ws->D.as<float>(), ld, st);
        select_dense(ws->D.as<float>(), N, ld, fl->has_ids ? fl->row_ids.as<uint64_t>() : nullptr, b, sp, rf,
                     out.at(q0, sp.k), st);
    }
}

// ---- binary vectors (Hamming distance) ----
// Paths, chosen from shape and request (DESIGN.md section 6):
//   SIMT dense    ham_dense_kernel -> D[b][N] -> select mode 1.  N < HAM_TC_MIN_N, or fewer than HAM_TC_MIN_B queries
//                 with N <= HAM_SAMPLE, prefilter or distance_range, LGPU_NO_TENSOR_CORE=1.
//   wgmma dense   the b1 gemm_dist_kernel writes D[b][N] -> select mode 1 (N <= HAM_SAMPLE).
//   wgmma list    N > HAM_SAMPLE, any batch size: sample pass -> threshold -> filtering pass -> select mode 2 -> dense
//                 fix-up of the queries whose list overflowed (ham_topk_list).  On the H100 it beat the SIMT kernel at
//                 every batch size measured, one query included: a single query's select over a dense row of N
//                 columns runs on one SM.
// Every path computes exact integer distances, so all three return the same rows.
constexpr uint64_t HAM_SAMPLE = 65536;     // rows of the threshold sample
constexpr uint32_t HAM_TC_MIN_B = 128;     // dense tensor-core path from this many queries (measured: SIMT faster at
                                           // 64 queries x 60000 rows, wgmma at 256) ...
constexpr uint64_t HAM_TC_MIN_N = 4096;    // ... and this many rows (not measured)

// Candidate-list capacity of the list path.  Rows with d <= tau_q, tau_q the k-th smallest distance among the sample's
// rows, number about k N / ns (more under ties): 4x that, at least 1024, at most 16384.
static uint32_t ham_list_cap(uint32_t k, uint64_t N, uint64_t ns)
{
    const uint64_t want = 4 * (uint64_t)k * ((N + ns - 1) / ns);
    uint32_t cap = 1024;
    while (cap < want && cap < 16384) cap <<= 1;
    return cap;
}

// One sub-batch through the tensor-core list path (Q: padded queries [B][nbytes_pad], qpop [B]).  The dense fix-up of
// overflowed queries runs in chunks of `bf` queries over a [bf][N] matrix: one launch lists each chunk's flagged
// queries, and each chunk's two launches return at once when its list is empty.
static void ham_topk_list(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *Q, const uint32_t *qpop,
                          uint32_t B, uint32_t k, uint32_t cap, uint32_t bf, TopkOut out)
{
    const uint64_t N = bx->nrows, ns = bx->nsample, lds = (ns + 3) & ~3ull, ld = (N + 3) & ~3ull;
    const uint32_t nbp = bx->nbytes_pad;
    const uint64_t *col_ids = bx->has_ids ? bx->row_ids.as<uint64_t>() : nullptr;
    // 1. sample pass: exact distances to the sample rows, tau_q = the k-th smallest (an upper bound of the true k-th)
    launch_ham_gemm(Q, bx->sample.p, bx->sample_pop.as<uint32_t>(), qpop, B, ns, nbp, ws->h_sample.as<float>(), lds,
                    bx->num_sms, st);
    launch_select(select_rows(ws->h_sample.as<float>(), ns, lds, B, k, {ws->sbound.as<uint64_t>(), ws->t_dist.as<float>(),
                                                                        ws->t_cnt.as<uint32_t>()}), st);
    launch_ham_threshold(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), B, k, ws->probe_A.as<float>(), st);
    // 2. full pass: every row with d <= tau_q is appended as (position, id, distance); the distance is final
    LGPU_CUDA(cudaMemsetAsync(ws->amax.p, 0, (size_t)B * 4, st));
    GemmFilter flt{};
    flt.thr = ws->probe_A.as<float>(); flt.count = ws->amax.as<uint32_t>(); flt.cand_pos = ws->t_pos.as<uint64_t>();
    flt.cand_ids = ws->t_ids.as<uint64_t>(); flt.col_ids = col_ids; flt.cap = cap; flt.cand_s = ws->t_exact.as<float>();
    launch_ham_gemm(Q, bx->vectors.p, bx->pop.as<uint32_t>(), qpop, B, N, nbp, nullptr, 0, bx->num_sms, st, &flt);
    launch_overflow_flags(ws->amax.as<uint32_t>(), cap, B, ws->flags.as<uint32_t>(), st);
    // 3. top-k by (distance, id) of each list (an overflowed list is complete up to cap; its query is redone below)
    SelectArgs sb = select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), cap, B, k, out);
    sb.ncols_q = ws->amax.as<uint32_t>();
    launch_select(sb, st);
    // 4. dense fix-up of the overflowed queries only
    launch_ham_flag_list(ws->flags.as<uint32_t>(), B, bf, ws->h_list.as<uint32_t>(), ws->h_cnt.as<uint32_t>(), st);
    for (uint32_t q0 = 0, c = 0; q0 < B; q0 += bf, c++) {
        const uint32_t b = std::min(bf, B - q0);
        launch_ham_dense(Q + (size_t)q0 * nbp, bx->vectors.as<uint8_t>(), b, N, nbp, ws->D.as<float>(), ld, bx->num_sms, st,
                         ws->h_list.as<uint32_t>() + q0, ws->h_cnt.as<uint32_t>() + c);
        SelectArgs sc = select_rows(ws->D.as<float>(), N, ld, b, k, out.at(q0, k));
        sc.col_ids = col_ids; sc.only = ws->flags.as<uint32_t>() + q0; sc.gate = ws->h_cnt.as<uint32_t>() + c;
        launch_select(sc, st);
    }
}

// d_q: raw queries [B][nbytes] in device memory
void binary_search_device(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *d_q, uint32_t B,
                          const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                          RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint64_t N = bx->nrows, ld = (N + 3) & ~3ull;
    const uint32_t nbp = bx->nbytes_pad, k = sp.k;
    const uint64_t *col_ids = bx->has_ids ? bx->row_ids.as<uint64_t>() : nullptr;
    const TopkOut out{d_ids, d_dist, d_cnt};
    const bool prof = profiling_enabled();
    if (prof) memset(g_filter_stats, 0, sizeof(g_filter_stats));
    ws->hq.ensure((size_t)B * nbp); ws->hq_pop.ensure((size_t)B * 4);
    launch_ham_pack(d_q, bx->nbytes, bx->nbytes, B, ws->hq.as<uint8_t>(), nbp, ws->hq_pop.as<uint32_t>(), st);
    const uint8_t *Q = ws->hq.as<uint8_t>();
    const bool tc_ok = tc_enabled() && !rf.bits && !sp.has_lower && !sp.has_upper;
    const bool list = tc_ok && bx->nsample > 0;
    const bool tc = list || (tc_ok && B >= HAM_TC_MIN_B && N >= HAM_TC_MIN_N);
    const size_t budget = workspace_budget();
    if (list) {
        // Workspace, all inside LGPU_WS_BYTES: the fix-up matrix [bf][N] gets at most half the budget and 1 GiB (it is
        // rarely used); the rest is split into sub-batches of bs queries, each holding its sample scores [bs][ns] and
        // candidate lists [bs][cap] (at the default 8 GiB, 1024 queries x 10M rows run as one sub-batch).
        const uint64_t ns = bx->nsample, lds = (ns + 3) & ~3ull;
        const uint32_t cap = ham_list_cap(k, N, ns);
        const uint32_t bf = (uint32_t)std::max<size_t>(1, std::min<size_t>(std::min<size_t>(budget / 2, (size_t)1 << 30) / (ld * 4), B));
        const size_t per_q = lds * 4 + (size_t)cap * 20 + (size_t)k * 12 + 16;
        const size_t left = budget > (size_t)bf * ld * 4 ? budget - (size_t)bf * ld * 4 : 0;
        const uint32_t bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(left / per_q, B));
        ws->h_sample.ensure((size_t)bs * lds * 4);
        ws->t_dist.ensure((size_t)bs * k * 4); ws->sbound.ensure((size_t)bs * k * 8); ws->t_cnt.ensure((size_t)bs * 4);
        ws->probe_A.ensure((size_t)bs * 4); ws->amax.ensure((size_t)bs * 4); ws->flags.ensure((size_t)bs * 4);
        ws->t_pos.ensure((size_t)bs * cap * 8); ws->t_ids.ensure((size_t)bs * cap * 8);
        ws->t_exact.ensure((size_t)bs * cap * 4);
        ws->D.ensure((size_t)bf * ld * 4); ws->h_list.ensure((size_t)bs * 4);
        ws->h_cnt.ensure((size_t)((bs + bf - 1) / bf) * 4);
        for (uint32_t q0 = 0; q0 < B; q0 += bs) {
            const uint32_t b = std::min(bs, B - q0);
            if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);
            ham_topk_list(bx, ws, st, Q + (size_t)q0 * nbp, ws->hq_pop.as<uint32_t>() + q0, b, k, cap, bf, out.at(q0, k));
            if (prof) {             // [0] list appends, [2] queries redone densely (over every sub-batch)
                std::vector<uint32_t> cnt(b), fl(b);
                LGPU_CUDA(cudaMemcpyAsync(cnt.data(), ws->amax.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaMemcpyAsync(fl.data(), ws->flags.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaStreamSynchronize(st));
                for (uint32_t q = 0; q < b; q++) { g_filter_stats[0] += cnt[q]; g_filter_stats[2] += fl[q] ? 1 : 0; }
            }
        }
    } else {
        const uint32_t bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(budget / std::max<size_t>(ld * 4, 4), B));
        for (uint32_t q0 = 0; q0 < B; q0 += bs) {
            const uint32_t b = std::min(bs, B - q0);
            if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);
            ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
            if (tc)
                launch_ham_gemm(Q + (size_t)q0 * nbp, bx->vectors.p, bx->pop.as<uint32_t>(), ws->hq_pop.as<uint32_t>() + q0, b,
                                N, nbp, ws->D.as<float>(), ld, bx->num_sms, st);
            else
                launch_ham_dense(Q + (size_t)q0 * nbp, bx->vectors.as<uint8_t>(), b, N, nbp, ws->D.as<float>(), ld,
                                 bx->num_sms, st);
            select_dense(ws->D.as<float>(), N, ld, col_ids, b, sp, rf, out.at(q0, k), st);
        }
    }
    if (prof) {                     // [1] distances computed on the tensor cores, [3] queries
        LGPU_CUDA(cudaStreamSynchronize(st));
        g_filter_stats[1] = tc ? (uint64_t)B * (N + (list ? bx->nsample : 0)) : 0;
        g_filter_stats[3] = B;
    }
}

// ---- binary IVF_FLAT (lgpu_ivf_binary): Hamming coarse step -> regroup (group.cu) -> b1 MMA scan of the probed rows
// (ivf_ham_scan.cu) -> top-k over the distance segments (select mode 0), the IVF stages of lgpu_index ----

// One sub-batch, everything on `st`.  Q / qpop: the sub-batch's packed queries [B][nbytes_pad] and their popcounts.
// nprobes <= nlist.  only (device, [B]): redo just the flagged queries (maximum_nprobes widening).
static void ham_ivf_sub_batch(lgpu_ivf_binary *ix, Workspace *ws, cudaStream_t st, const uint8_t *Q, const uint32_t *qpop,
                              uint32_t B, const lgpu_search_params &sp, uint32_t nprobes, TopkOut out, bool prof,
                              RowFilter rf, const uint32_t *only = nullptr)
{
    IvfPlan p{};
    p.B = B; p.nprobes = nprobes; p.slots = B * nprobes; p.np_eff = nprobes;
    p.k = p.kk = sp.k; p.coarse = Coarse::exact; p.scan = IvfScan::ham;
    const uint32_t nlist = ix->nlist, nbp = ix->nbytes_pad;
    const StageMarks mark{ws, prof};
    mark(IVF_START, st);
    ws->stats_mode = 0;
    ws->probes.ensure((size_t)p.slots * 8);
    if (nprobes >= nlist) {                       // every partition: no coarse step, no top-nprobes select
        launch_ham_all_probes(ws->probes.as<uint64_t>(), B, nlist, st);
        mark(IVF_COARSE, st);
    } else {
        // Hamming distances to the packed centroids, then the nprobes nearest by (distance, partition id).  The b1
        // wgmma kernel from the flat path's crossover (HAM_TC_MIN_B x HAM_TC_MIN_N); for the coarse step's shapes the
        // crossover is not measured.
        const uint64_t ldc = (nlist + 3u) & ~3u;
        ws->probe_dist.ensure((size_t)p.slots * 4); ws->probe_cnt.ensure((size_t)B * 4);
        ws->D.ensure((size_t)B * ldc * 4);
        if (tc_enabled() && B >= HAM_TC_MIN_B && nlist >= HAM_TC_MIN_N)
            launch_ham_gemm(Q, ix->centroids.p, ix->cent_pop.as<uint32_t>(), qpop, B, nlist, nbp, ws->D.as<float>(), ldc,
                            ix->num_sms, st);
        else
            launch_ham_dense(Q, ix->centroids.as<uint8_t>(), B, nlist, nbp, ws->D.as<float>(), ldc, ix->num_sms, st);
        mark(IVF_COARSE, st);
        launch_select(select_rows(ws->D.as<float>(), nlist, ldc, B, nprobes, {ws->probes.as<uint64_t>(),
                                  ws->probe_dist.as<float>(), ws->probe_cnt.as<uint32_t>()}), st);
    }
    mark(IVF_PROBES, st);
    const GroupArgs ga = ivf_regroup(ix, ws, p, only, st);
    mark(IVF_REGROUP, st);
    HamScanArgs ha{};
    ha.rows = ix->codes.as<uint8_t>(); ha.row_pop = ix->row_pop.as<uint32_t>(); ha.queries = Q; ha.qpop = qpop;
    ha.nbytes_pad = nbp;
    ha.total_tiles = ga.total_tiles; ha.tile_counter = ga.tile_counter; ha.tile_desc = ga.tile_desc;
    ha.dist_out = ws->dist_out.as<float>();
    launch_ivf_ham_scan(ha, 2 * ix->num_sms, st);
    mark(IVF_SCAN, st);
    // distances are exact: refine_factor has nothing to re-rank, the top-k is taken directly
    SelectArgs sa = select_segments(ix, ws, p, sp.k, out, rf);
    sa.only = only;
    with_range(sa, sp);
    launch_select(sa, st);
    mark(IVF_TOPK, st);
}

static uint32_t ham_ivf_sub_batch_size(lgpu_ivf_binary *ix, uint32_t B, uint32_t nprobes)
{
    const uint32_t np_eff = std::min<uint32_t>(nprobes, ix->nlist);
    // distance segments, coarse scores, probe slots (ids, distances, regroup) and their tile descriptors
    const size_t per_q = ix->pad_prefix[np_eff] * 4 + (size_t)ix->nlist * 4 + (size_t)np_eff * 36 +
                         (size_t)np_eff * ix->max_nrb * (sizeof(TileDesc) / SCAN_G + 1) + 64;
    size_t bs = workspace_budget() / per_q;
    bs = std::min<size_t>(bs, (size_t)0xffffffffull / std::max<size_t>(ix->pad_prefix[np_eff], 1));
    bs = std::max<size_t>(1, std::min<size_t>(bs, 65535));
    return (uint32_t)std::min<size_t>(bs, B);
}

// d_q: raw queries [B][nbytes] in device memory
void ivf_binary_search_device(lgpu_ivf_binary *ix, Workspace *ws, cudaStream_t st, const uint8_t *d_q, uint32_t B,
                              const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                              RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint32_t nbp = ix->nbytes_pad;
    const uint32_t nprobes = std::min<uint32_t>(std::max<uint32_t>(sp.nprobes, 1), ix->nlist);
    const uint32_t np_max = std::min<uint32_t>(sp.max_nprobes, ix->nlist);
    const bool widen = rf.bits && np_max > nprobes;
    // maximum_nprobes is only read when it widens (under a prefilter), as on lgpu_index
    if (widen)
        LGPU_REQUIRE(np_max <= SELECT_KMAX || np_max >= ix->nlist,
                     "maximum_nprobes above 2048 is not supported unless it covers every partition");
    const uint32_t bs = ham_ivf_sub_batch_size(ix, B, widen ? np_max : nprobes);
    const bool prof = profiling_enabled();
    const TopkOut out{d_ids, d_dist, d_cnt};
    if (prof) {
        memset(g_stage_ms, 0, sizeof(g_stage_ms));
        memset(g_filter_stats, 0, sizeof(g_filter_stats));
        g_scanned_bytes = 0;
    }
    ws->hq.ensure((size_t)B * nbp); ws->hq_pop.ensure((size_t)B * 4);
    launch_ham_pack(d_q, ix->nbytes, ix->nbytes, B, ws->hq.as<uint8_t>(), nbp, ws->hq_pop.as<uint32_t>(), st);
    for (uint32_t q0 = 0; q0 < B; q0 += bs) {
        const uint32_t b = std::min(bs, B - q0);
        if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);      // the previous sub-batch, or LGPU_TIMEOUT
        const uint8_t *Q = ws->hq.as<uint8_t>() + (size_t)q0 * nbp;
        const uint32_t *qpop = ws->hq_pop.as<uint32_t>() + q0;
        ham_ivf_sub_batch(ix, ws, st, Q, qpop, b, sp, nprobes, out.at(q0, sp.k), prof, rf);
        if (prof) g_scanned_bytes += add_stage_marks(ws, st) * nbp;      // the whole call, as on lgpu_index
        // maximum_nprobes under a prefilter, as on lgpu_index: the queries that found fewer than k rows are searched
        // again over their np_max nearest partitions
        if (widen) {
            ws->widen.ensure((size_t)b * 4);
            launch_count_below(out.at(q0, sp.k).cnt, b, sp.k, ws->widen.as<uint32_t>(), st);
            ham_ivf_sub_batch(ix, ws, st, Q, qpop, b, sp, np_max, out.at(q0, sp.k), false, rf, ws->widen.as<uint32_t>());
        }
    }
}

// ---- multivector columns (late interaction: sum over the query's vectors of the min cosine distance) ----
// Limits of one call: a query holds 1..MV_MAX_NQ vectors, a row 0..MV_MAX_ROW, a vector at most MV_MAX_DIM components.
constexpr uint32_t MV_MAX_NQ = 4096;
constexpr uint64_t MV_MAX_ROW = (uint64_t)1 << 20;
constexpr uint32_t MV_MAX_DIM = 65536;

// Paths (multivec.cu, DESIGN.md section 6), chosen per call:
//   tensor cores  the F16MaxSim gemm_dist_kernel scores fp16 copies of the normalised vectors and keeps the largest
//                 similarity per (query vector, row); approximate distances -> the k-th smallest (select mode 1) -> every
//                 row within 2 E_q of it (mv_band) -> exact re-score of those rows (dist.cu) -> select mode 2; a query
//                 whose list overflowed or that holds a zero / non-finite vector is redone by the exact path below in
//                 the same stream (flags / gate: nothing runs when no query is flagged).  Taken when the column holds at
//                 least MV_TC_MIN_T vectors (all of them finite and non-zero), dim is a multiple of 8, there is no
//                 prefilter or distance_range, LGPU_NO_TENSOR_CORE is not set and one query's scores fit the workspace.
//   exact         for every sub-batch of queries, blocks of consecutive query vectors against chunks of whole rows --
//                 dist_matrix_kernel (cosine, lance order) -> per-row minimum -> in-order running sum into D[b][N] --
//                 then select mode 1 (distance_range, prefilter, (_distance, _rowid) order, NaN dropped).
// Workspace stays inside LGPU_WS_BYTES.
constexpr uint64_t MV_TC_MIN_T = 65536;   // stored vectors from which the tensor-core path runs (not measured)

// the exact distances of queries [qa, qb) into D[b - qa][N] (only / vflags / gate: the fix-up of flagged queries)
static void mv_exact_dense(lgpu_multivec *mv, Workspace *ws, cudaStream_t st, const float *d_q, const uint32_t *h_qoff,
                           uint32_t qa, uint32_t qb, float *D, uint64_t ld, const uint32_t *only = nullptr,
                           const uint32_t *vflags = nullptr, const uint32_t *gate = nullptr)
{
    const uint64_t N = mv->nrows;
    const uint32_t dim = mv->dim;
    const size_t budget = workspace_budget();
    // a chunk of rows costs (n_r + 1) floats per query vector in the block (P and M); every row fits in half a chunk
    const size_t pair_floats = std::max<size_t>(budget / 2 / 4, 1);
    const uint64_t row_cost = mv->max_row + 1;
    const uint32_t qv_max = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(pair_floats / (2 * row_cost), 65535ull * 16));
    const uint64_t *off = mv->h_offsets.data();
    uint32_t blo = qa;
    for (uint32_t i0 = h_qoff[qa]; i0 < h_qoff[qb]; i0 += qv_max) {
        const uint32_t i1 = std::min(h_qoff[qb], i0 + qv_max), nqv = i1 - i0;
        while (h_qoff[blo + 1] <= i0) blo++;                         // first query with a vector in [i0, i1)
        uint32_t bhi = blo;
        while (bhi < qb && h_qoff[bhi] < i1) bhi++;                  // one past the last
        const uint64_t cap = std::max<uint64_t>(pair_floats / nqv, 2 * row_cost);
        for (uint64_t r0 = 0; r0 < N;) {
            uint64_t r1 = r0 + 1;
            while (r1 < N && (off[r1 + 1] - off[r0]) + (r1 + 1 - r0) <= cap) r1++;
            const uint64_t span = off[r1] - off[r0], ldP = (span + 3) & ~3ull;
            const uint32_t nr = (uint32_t)(r1 - r0);
            ws->mv_P.ensure(std::max<size_t>((size_t)nqv * ldP, 4) * 4);
            ws->mv_M.ensure((size_t)nqv * nr * 4);
            if (span)
                launch_dist_matrix(d_q + (size_t)i0 * dim, mv->vectors.as<float>() + (size_t)off[r0] * dim, nqv, span,
                                   dim, 2, ws->xnorm.as<float>() + i0, mv->ysqrt.as<float>() + off[r0],
                                   ws->mv_P.as<float>(), ldP, st, vflags ? vflags + (i0 - h_qoff[qa]) : nullptr, gate);
            launch_mv_rowmin(ws->mv_P.as<float>(), ldP, nqv, mv->offsets.as<uint64_t>(), r0, nr, ws->mv_M.as<float>(),
                             nr, mv->num_sms, st, gate);
            launch_mv_rowsum(ws->mv_M.as<float>(), nr, ws->mv_qoff.as<uint32_t>(), blo, bhi, qa, i0, i1, nr, D, ld, r0,
                             mv->num_sms, st, only, gate);
            r0 = r1;
        }
    }
}

// h_qoff: HOST [B+1] offsets of each query's vectors in d_q (validated by the caller).
void multivec_search_device(lgpu_multivec *mv, Workspace *ws, cudaStream_t st, const float *d_q, const uint32_t *h_qoff,
                            uint32_t B, const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                            RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint64_t N = mv->nrows, ld = (N + 3) & ~3ull;
    const uint32_t dim = mv->dim, k = sp.k, Tq = h_qoff[B];
    const TopkOut out{d_ids, d_dist, d_cnt};
    const bool prof = profiling_enabled();
    if (prof) memset(g_filter_stats, 0, sizeof(g_filter_stats));
    ws->mv_qoff.ensure((size_t)(B + 1) * 4);
    LGPU_CUDA(cudaMemcpyAsync(ws->mv_qoff.p, h_qoff, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, st));
    ws->xnorm.ensure(std::max<size_t>(Tq, 1) * 4);
    launch_row_norms(d_q, Tq, dim, ws->xnorm.as<float>(), st);
    const size_t budget = workspace_budget();
    uint32_t max_nq = 0;
    for (uint32_t b = 0; b < B; b++) max_nq = std::max(max_nq, h_qoff[b + 1] - h_qoff[b]);
    const size_t quarter = budget / 4;
    const bool tc = mv->tc_ok && tc_enabled() && !rf.bits && !sp.has_lower && !sp.has_upper &&
                    (size_t)(max_nq + 1) * ld * 4 <= quarter;
    if (tc) {
        // fp16 normalised queries (and the queries holding a bad vector), then sub-batches of whole queries whose scores
        // M [vectors][ld] u32 and approximate distances A [queries][ld] f32 take a quarter of the budget each
        ws->mv_qh.ensure(std::max<size_t>((size_t)Tq * dim * 2, 16));
        ws->mv_qbad.ensure(std::max<size_t>(Tq, 1) * 4);
        launch_mv_normalize_f16(d_q, Tq, dim, ws->mv_qh.p, ws->mv_qbad.as<uint32_t>(), st);
        uint32_t cap = 1024;
        while (cap < 8 * k && cap < 16384) cap <<= 1;
        for (uint32_t qa = 0; qa < B;) {
            uint32_t qb = qa + 1;
            while (qb < B && (size_t)(h_qoff[qb + 1] - h_qoff[qa]) * ld * 4 <= quarter && (size_t)(qb + 1 - qa) * ld * 4 <= quarter)
                qb++;
            if (deadline && qa > 0) deadline->wait(st, ws->ev[7]);
            const uint32_t b = qb - qa, va = h_qoff[qa], nqv = h_qoff[qb] - va;
            ws->mv_Mk.ensure((size_t)nqv * ld * 4);
            ws->mv_A.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
            ws->mv_kd.ensure((size_t)b * k * 4); ws->mv_ki.ensure((size_t)b * k * 8); ws->mv_kc.ensure((size_t)b * 4);
            ws->mv_thr.ensure((size_t)b * 4); ws->mv_cnt.ensure((size_t)b * 4); ws->mv_cand.ensure((size_t)b * cap * 4);
            ws->mv_flags.ensure((size_t)b * 4); ws->mv_vflags.ensure((size_t)nqv * 4); ws->mv_gate.ensure(16);
            ws->mv_ex.ensure((size_t)b * cap * 4); ws->mv_exid.ensure((size_t)b * cap * 8);
            LGPU_CUDA(cudaMemsetAsync(ws->mv_Mk.p, 0, (size_t)nqv * ld * 4, st));
            MaxSimOut mo{};
            mo.col_row = mv->col_row.as<uint32_t>(); mo.M = ws->mv_Mk.as<uint32_t>(); mo.ldM = ld; mo.row_base = 0;
            mo.xdummy = mv->ysqrt.as<float>();
            launch_maxsim_gemm(ws->mv_qh.as<char>() + (size_t)va * dim * 2, mv->vec_h.p, nqv, mv->total, dim, mo,
                               mv->num_sms, st);
            launch_mv_approx_sum(ws->mv_Mk.as<uint32_t>(), ld, ws->mv_qoff.as<uint32_t>(), qa, qb, va, N,
                                 ws->mv_A.as<float>(), ld, mv->num_sms, st);
            // the k-th smallest approximate distance of each query
            launch_select(select_rows(ws->mv_A.as<float>(), N, ld, b, k, {ws->mv_ki.as<uint64_t>(), ws->mv_kd.as<float>(),
                                                                          ws->mv_kc.as<uint32_t>()}), st);
            launch_mv_threshold(ws->mv_kd.as<float>(), ws->mv_kc.as<uint32_t>(), ws->mv_qoff.as<uint32_t>(), qa, b, k, dim,
                                ws->mv_thr.as<float>(), st);
            LGPU_CUDA(cudaMemsetAsync(ws->mv_cnt.p, 0, (size_t)b * 4, st));
            launch_mv_admit(ws->mv_A.as<float>(), ld, b, N, ws->mv_thr.as<float>(), cap, ws->mv_cnt.as<uint32_t>(),
                            ws->mv_cand.as<uint32_t>(), st);
            launch_mv_flags(ws->mv_cnt.as<uint32_t>(), cap, ws->mv_qbad.as<uint32_t>(), ws->mv_qoff.as<uint32_t>(), qa, b,
                            ws->mv_flags.as<uint32_t>(), ws->mv_vflags.as<uint32_t>(), ws->mv_gate.as<uint32_t>(), st);
            launch_mv_rescore(d_q, ws->mv_qoff.as<uint32_t>(), qa, ws->xnorm.as<float>(), mv->vectors.as<float>(),
                              mv->ysqrt.as<float>(), mv->offsets.as<uint64_t>(),
                              mv->has_ids ? mv->row_ids.as<uint64_t>() : nullptr, dim, b, ws->mv_cand.as<uint32_t>(),
                              ws->mv_cnt.as<uint32_t>(), cap, ws->mv_ex.as<float>(), ws->mv_exid.as<uint64_t>(), st);
            launch_select(select_cands(ws->mv_ex.as<float>(), ws->mv_exid.as<uint64_t>(), cap, b, k, out.at(qa, k)), st);
            // exact fix-up of the flagged queries (A is free again: it holds their exact distances)
            mv_exact_dense(mv, ws, st, d_q, h_qoff, qa, qb, ws->mv_A.as<float>(), ld, ws->mv_flags.as<uint32_t>(),
                           ws->mv_vflags.as<uint32_t>(), ws->mv_gate.as<uint32_t>());
            SelectArgs sc = select_rows(ws->mv_A.as<float>(), N, ld, b, k, out.at(qa, k));
            sc.col_ids = mv->has_ids ? mv->row_ids.as<uint64_t>() : nullptr;
            sc.only = ws->mv_flags.as<uint32_t>(); sc.gate = ws->mv_gate.as<uint32_t>();
            launch_select(sc, st);
            if (prof) {             // [0] rows admitted, [1] rows re-scored exactly, [2] queries redone densely
                std::vector<uint32_t> cnt(b), fl(b);
                LGPU_CUDA(cudaMemcpyAsync(cnt.data(), ws->mv_cnt.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaMemcpyAsync(fl.data(), ws->mv_flags.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaStreamSynchronize(st));
                for (uint32_t q = 0; q < b; q++) {
                    g_filter_stats[0] += cnt[q]; g_filter_stats[1] += std::min(cnt[q], cap);
                    g_filter_stats[2] += fl[q] ? 1 : 0;
                }
            }
            qa = qb;
        }
    } else {
        const uint32_t bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(budget / 2 / std::max<size_t>(ld * 4, 4), B));
        for (uint32_t qa = 0; qa < B; qa += bs) {
            const uint32_t qb = std::min(B, qa + bs), b = qb - qa;
            if (deadline && qa > 0) deadline->wait(st, ws->ev[7]);
            ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
            mv_exact_dense(mv, ws, st, d_q, h_qoff, qa, qb, ws->D.as<float>(), ld);
            select_dense(ws->D.as<float>(), N, ld, mv->has_ids ? mv->row_ids.as<uint64_t>() : nullptr, b, sp, rf,
                         out.at(qa, k), st);
        }
    }
    if (prof) {                     // exact path: [1] rows scored exactly; both: [3] queries
        LGPU_CUDA(cudaStreamSynchronize(st));
        if (!tc) g_filter_stats[1] = (uint64_t)B * N;
        g_filter_stats[3] = B;
    }
}

// the query vector offsets of a multivector call: [B+1], starting at 0, every query holding 1..MV_MAX_NQ vectors
static void check_multivec_offsets(const uint32_t *q_off, uint32_t B)
{
    LGPU_REQUIRE(q_off != nullptr, "query offsets are null");
    LGPU_REQUIRE(q_off[0] == 0, "query offsets must start at 0");
    for (uint32_t b = 0; b < B; b++) {
        LGPU_REQUIRE(q_off[b + 1] > q_off[b], "every multivector query needs at least one vector (offsets must increase)");
        LGPU_REQUIRE(q_off[b + 1] - q_off[b] <= MV_MAX_NQ, "a multivector query holds at most 4096 vectors");
    }
}

template <class F> int guarded(F &&f)
{
    try { f(); return LGPU_OK; }
    catch (const Failure &e) { return e.status; }
    catch (const std::bad_alloc &) { set_error("host allocation failed"); return LGPU_OOM; }
    catch (const std::exception &e) { set_error(e.what()); return LGPU_RUNTIME; }
}

void require_device(int device)
{
    if (g_fork_poisoned.load()) {
        set_error("this process is a fork() of one that already used CUDA through lancedb_b200: the GPU context "
                  "does not survive fork; open the index in a spawned process instead");
        throw Failure{LGPU_RUNTIME};
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_error("no CUDA device available: lancedb_b200 has no CPU fallback");
        throw Failure{LGPU_RUNTIME};
    }
    LGPU_REQUIRE(device >= 0 && device < n, "invalid CUDA device ordinal");
    LGPU_CUDA(cudaSetDevice(device));
    g_cuda_touched.store(true);
}

// CUDA-graph replay of the host-buffer entry points is on by default; LGPU_NO_GRAPH=1 disables it.
static bool graphs_enabled()
{
    static int v = -1;
    if (v < 0) { const char *e = getenv("LGPU_NO_GRAPH"); v = (e && e[0] == '1') ? 0 : 1; }
    return v == 1;
}

// host-buffer wrapper: stage in, run, stage out, synchronise.  The queries are `q_elems` elements of T (f32 vectors,
// or the bytes of packed binary vectors).  `key` (nullptr: always eager) identifies the launch sequence
// (shapes + parameters): the second call with the same key is captured into a CUDA graph and later calls
// replay it, which removes ~15 launch latencies from the synchronous end-to-end path.  Any device
// (re)allocation anywhere in the process since the capture, profiling mode, or a failed capture falls back to
// eager launches.
template <class T, class Run>
void host_submit(WsLease &lease, const Deadline &deadline, const T *queries, size_t q_elems, uint32_t B, uint32_t k,
                 uint64_t *out_ids, float *out_dist, uint32_t *out_count, const uint64_t *key, Run &&run, bool sync)
{
    Workspace *ws = lease.ws;
    cudaStream_t st = lease.st;
    ws->q.ensure(std::max<size_t>(q_elems, 1) * sizeof(T));
    ws->out_ids.ensure(std::max<size_t>((size_t)B * k, 1) * 8);
    ws->out_dist.ensure(std::max<size_t>((size_t)B * k, 1) * 4);
    ws->out_count.ensure(std::max<size_t>(B, 1) * 4);
    LGPU_CUDA(cudaMemcpyAsync(ws->q.p, queries, q_elems * sizeof(T), cudaMemcpyHostToDevice, st));
    auto eager = [&] {
        run(ws, st, ws->q.as<T>(), ws->out_ids.as<uint64_t>(), ws->out_dist.as<float>(), ws->out_count.as<uint32_t>(),
            deadline);
    };
    if (!key || !graphs_enabled() || profiling_enabled() || ws->graph_state < 0 || deadline.armed) {
        eager();
    } else if (memcmp(key, ws->graph_key, sizeof(ws->graph_key)) != 0) {   // new shape: warm up (allocations), capture next time
        if (ws->graph) { cudaGraphExecDestroy(ws->graph); ws->graph = nullptr; }
        memcpy(ws->graph_key, key, sizeof(ws->graph_key));
        ws->graph_state = 0;
        eager();
        ws->graph_state = 1;
    } else if (ws->graph_state == 2 && g_alloc_epoch.load() == ws->graph_epoch) {
        LGPU_CUDA(cudaGraphLaunch(ws->graph, st));
        count_launches(ws->graph_kernels);
    } else if (ws->graph_state == 1) {
        bool ok = false;
        cudaGraph_t g = nullptr;
        const uint64_t epoch0 = g_alloc_epoch.load();
        if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            g_capturing = true; g_captured_launches = 0;
            try {
                eager();
                ok = cudaStreamEndCapture(st, &g) == cudaSuccess && g != nullptr && g_alloc_epoch.load() == epoch0;
            } catch (const Failure &) {
                cudaStreamEndCapture(st, &g);
                ok = false;
            }
            g_capturing = false;
        }
        if (ok && cudaGraphInstantiate(&ws->graph, g, 0) == cudaSuccess) {
            ws->graph_state = 2;
            ws->graph_epoch = epoch0;
            ws->graph_kernels = g_captured_launches;
            cudaGraphDestroy(g);
            LGPU_CUDA(cudaGraphLaunch(ws->graph, st));
            count_launches(ws->graph_kernels);
        } else if (g_alloc_epoch.load() != epoch0) {        // a buffer moved during the capture: try again next call
            if (g) cudaGraphDestroy(g);
            cudaGetLastError();
            ws->graph = nullptr;
            LGPU_CUDA(cudaMemcpyAsync(ws->q.p, queries, q_elems * sizeof(T), cudaMemcpyHostToDevice, st));
            eager();
        } else {                                            // never try again with this workspace
            if (g) cudaGraphDestroy(g);
            cudaGetLastError();
            ws->graph = nullptr;
            ws->graph_state = -1;
            LGPU_CUDA(cudaMemcpyAsync(ws->q.p, queries, q_elems * sizeof(T), cudaMemcpyHostToDevice, st));
            eager();
        }
    } else {                                                // captured, but a buffer moved since: capture again
        if (ws->graph) { cudaGraphExecDestroy(ws->graph); ws->graph = nullptr; }
        ws->graph_state = 1;
        eager();
    }
    if (sync) deadline.wait(st, ws->ev[7]);
    LGPU_CUDA(cudaMemcpyAsync(out_ids, ws->out_ids.p, (size_t)B * k * 8, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaMemcpyAsync(out_dist, ws->out_dist.p, (size_t)B * k * 4, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaMemcpyAsync(out_count, ws->out_count.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    if (sync) LGPU_CUDA(cudaStreamSynchronize(st));
}

template <class T, class Run>
void host_call(WorkspacePool &pool, const T *queries, size_t q_elems, uint32_t B, uint32_t k, uint64_t *out_ids,
               float *out_dist, uint32_t *out_count, const uint64_t *key, uint32_t timeout_ms, Run &&run)
{
    const Deadline deadline(timeout_ms);
    WsLease lease(pool, nullptr, false);
    host_submit(lease, deadline, queries, q_elems, B, k, out_ids, out_dist, out_count, key, run, true);
}

static inline void make_key(uint64_t (&key)[4], uint64_t tag, uint32_t B, const lgpu_search_params &p)
{
    uint32_t lo, hi;
    memcpy(&lo, &p.lower, 4); memcpy(&hi, &p.upper, 4);
    key[0] = tag ^ ((uint64_t)B << 32);
    key[1] = (uint64_t)p.k | ((uint64_t)p.nprobes << 32);
    key[2] = (uint64_t)p.refine_factor | ((uint64_t)(p.has_lower ? 1 : 0) << 32) | ((uint64_t)(p.has_upper ? 1 : 0) << 33) |
             ((uint64_t)(p.max_nprobes & 0x3fffffu) << 34);
    key[3] = ((uint64_t)lo | ((uint64_t)hi << 32)) ^ scan_modes().signature();
}

// the host bitmap over row ids of a filtered call, staged into the workspace on `st`
static RowFilter upload_allow(Workspace *ws, cudaStream_t st, const uint32_t *allow, uint64_t allow_bits)
{
    const size_t words = (size_t)((allow_bits + 31) / 32);
    ws->allow.ensure(std::max<size_t>(words, 1) * 4);
    if (words) LGPU_CUDA(cudaMemcpyAsync(ws->allow.p, allow, words * 4, cudaMemcpyHostToDevice, st));
    RowFilter rf; rf.bits = ws->allow.as<uint32_t>(); rf.nbits = allow_bits;
    return rf;
}

// where a search call's buffers live
struct Route {
    enum Via { HOST, FILTERED, DEVICE } via;
    uint64_t graph_tag;                 // HOST: tag of the CUDA-graph key (0: never captured)
    const uint32_t *allow;              // FILTERED: host bitmap over row ids
    uint64_t allow_bits;
    void *stream;                       // DEVICE: the caller's stream
};
static Route host_route(uint64_t graph_tag) { return {Route::HOST, graph_tag, nullptr, 0, nullptr}; }
static Route filtered_route(const uint32_t *allow, uint64_t allow_bits)
{
    return {Route::FILTERED, 0, allow, allow_bits, nullptr};
}
static Route device_route(void *stream) { return {Route::DEVICE, 0, nullptr, 0, stream}; }

// The sequence of every search entry point: resolve the handle; the kind's own checks, `check(h)`, which return how
// many query elements (T) the call reads; the bitmap of a filtered call; nothing more for B == 0; the device; then
// the kind's `search(h, ws, st, d_q, B, params, d_ids, d_dist, d_cnt, rf, deadline)` on a workspace leased for the
// caller's stream, or staged through host_submit.
template <class H, class T, class Check, class Search>
int search_call(H *hp, const char *what, const Route &r, const T *queries, uint32_t B, const lgpu_search_params *p,
                uint64_t *ids, float *dist, uint32_t *cnt, Check &&check, Search &&search)
{
    return guarded([&] {
        HandleRef<H> h(hp, what);
        const size_t q_elems = check(h.h);
        if (r.via == Route::FILTERED) LGPU_REQUIRE(r.allow != nullptr || r.allow_bits == 0, "allow bitmap is null");
        if (B == 0) return;
        require_device(h->device);
        if (r.via == Route::DEVICE) {
            WsLease lease(h->pool, (cudaStream_t)r.stream, true);
            search(h.h, lease.ws, lease.st, queries, B, *p, ids, dist, cnt, RowFilter(), nullptr);
            return;
        }
        uint64_t key[4];
        if (r.graph_tag) make_key(key, r.graph_tag, B, *p);
        host_call(h->pool, queries, q_elems, B, p->k, ids, dist, cnt, r.graph_tag ? key : nullptr, p->timeout_ms,
                  [&](Workspace *ws, cudaStream_t st, const T *dq, uint64_t *di, float *dd, uint32_t *dc,
                      const Deadline &dl) {
                      const RowFilter rf = r.via == Route::FILTERED ? upload_allow(ws, st, r.allow, r.allow_bits)
                                                                    : RowFilter();
                      search(h.h, ws, st, dq, B, *p, di, dd, dc, rf, &dl);
                  });
    });
}

// what the flat, binary and multivector opens share: the device's SM count and the optional row ids
template <class H> static void open_rows(H *h, const uint64_t *row_ids, uint64_t nrows)
{
    cudaDeviceProp prop;
    LGPU_CUDA(cudaGetDeviceProperties(&prop, h->device));
    h->num_sms = prop.multiProcessorCount;
    if (row_ids && nrows) {
        h->row_ids.ensure((size_t)nrows * 8);
        LGPU_CUDA(cudaMemcpy(h->row_ids.p, row_ids, (size_t)nrows * 8, cudaMemcpyHostToDevice));
        h->has_ids = true;
    }
}

// the partition layout every IVF index shares (lgpu_index_open, lgpu_ivf_sq_open): checked before any device work
static void check_ivf_layout(uint32_t dim, uint32_t nlist, int metric, uint64_t nrows, const void *centroids,
                             const uint64_t *part_offsets, const void *codes, const uint64_t *row_ids)
{
    LGPU_REQUIRE(dim > 0 && nlist > 0, "dim and nlist must be positive");
    LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE || metric == LGPU_DOT, "unknown distance type");
    LGPU_REQUIRE(centroids && part_offsets, "null index array");
    LGPU_REQUIRE(nrows == 0 || (codes && row_ids), "null codes / row_ids");
    LGPU_REQUIRE(nrows < (1ull << 32), "more than 2^32 rows in one GPU shard are not supported (shard the index)");
    LGPU_REQUIRE(part_offsets[0] == 0 && part_offsets[nlist] == nrows, "part_offsets must start at 0 and end at nrows");
    for (uint32_t p = 0; p < nlist; p++) {
        LGPU_REQUIRE(part_offsets[p + 1] >= part_offsets[p], "part_offsets must be non-decreasing");
        LGPU_REQUIRE(part_offsets[p + 1] - part_offsets[p] < (1ull << 31), "partition too large");
    }
}

// The arrays every IVF index holds in HBM, uploaded on the legacy stream: centroids (and their bf16 copy for the
// tensor-core coarse step), partition sizes and offsets, row ids, optional raw vectors.  `rows_tile` is the scan's
// tile height, which bounds the tile count of a search (max_nrb).
static void open_ivf_partitions(lgpu_index *ix, int device, uint32_t nlist, uint64_t nrows,
                                const uint64_t *part_offsets, const uint64_t *row_ids, uint32_t rows_tile);

static void open_ivf_common(lgpu_index *ix, int device, uint32_t dim, uint32_t nlist, int metric, uint64_t nrows,
                            const float *centroids, const uint64_t *part_offsets, const uint64_t *row_ids,
                            const float *vectors, uint32_t rows_tile)
{
    ix->dim = dim; ix->metric = metric;
    cudaStream_t st = nullptr;
    auto up = [&](DevBuf &b, const void *src, size_t bytes) {
        b.ensure(std::max<size_t>(bytes, 16));
        if (bytes) LGPU_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, st));
        ix->device_bytes += b.bytes;
    };
    up(ix->centroids, centroids, (size_t)nlist * dim * 4);
    open_ivf_partitions(ix, device, nlist, nrows, part_offsets, row_ids, rows_tile);
    if (vectors) { up(ix->vectors, vectors, (size_t)nrows * dim * 4); ix->has_vectors = true; }
    if (gemm_shape_supported(dim) && metric != LGPU_DOT) {
        LGPU_CUDA(cudaStreamSynchronize(st));
        prepare_tc_operand(ix->centroids.as<float>(), nlist, dim, ix->cent_b, ix->cent_n2, ix->cent_max, ix->cent_err, st);
        ix->device_bytes += ix->cent_b.bytes + ix->cent_n2.bytes;
        if (nlist >= 1024) {
            // every 8th centroid, for the sampled threshold of the coarse step (strided: whatever order the
            // trainer left the lists in -- hierarchical k-means groups neighbours -- the sample spans all of them)
            constexpr uint32_t COARSE_SAMPLE_STRIDE = 8;
            const uint32_t ns = nlist / COARSE_SAMPLE_STRIDE;
            ix->cent_sb.ensure((size_t)ns * dim * 2); ix->cent_sn2.ensure((size_t)ns * 4);
            LGPU_CUDA(cudaMemcpy2DAsync(ix->cent_sb.p, (size_t)dim * 2, ix->cent_b.p, (size_t)COARSE_SAMPLE_STRIDE * dim * 2,
                                        (size_t)dim * 2, ns, cudaMemcpyDeviceToDevice, st));
            LGPU_CUDA(cudaMemcpy2DAsync(ix->cent_sn2.p, 4, ix->cent_n2.p, (size_t)COARSE_SAMPLE_STRIDE * 4, 4, ns,
                                        cudaMemcpyDeviceToDevice, st));
            LGPU_CUDA(cudaStreamSynchronize(st));
            ix->cent_ns = ns;
            ix->device_bytes += ix->cent_sb.bytes + ix->cent_sn2.bytes;
        }
        ix->has_tc = true;
    }
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// The partition arrays every IVF index holds (part_n, part_npad, part_off, row_ids, the host-side tile bound max_nrb and
// pad_prefix), uploaded on the legacy stream; `rows_tile` is the scan's tile height
static void open_ivf_partitions(lgpu_index *ix, int device, uint32_t nlist, uint64_t nrows,
                                const uint64_t *part_offsets, const uint64_t *row_ids, uint32_t rows_tile)
{
    ix->device = device;
    cudaDeviceProp prop;
    LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
    ix->num_sms = prop.multiProcessorCount;
    ix->nlist = nlist; ix->nrows = nrows;
    std::vector<uint32_t> part_n(nlist), part_npad(nlist);
    std::vector<uint64_t> pads(nlist);
    for (uint32_t p = 0; p < nlist; p++) {
        const uint32_t n = (uint32_t)(part_offsets[p + 1] - part_offsets[p]);
        part_n[p] = n; part_npad[p] = (n + 31u) & ~31u;
        pads[p] = (n + 3ull) & ~3ull;
        ix->max_nrb = std::max(ix->max_nrb, scan_nrb(n, rows_tile));
    }
    ix->h_part_n = part_n;
    std::sort(pads.begin(), pads.end(), std::greater<uint64_t>());
    ix->pad_prefix.assign(nlist + 1, 0);
    for (uint32_t p = 0; p < nlist; p++) ix->pad_prefix[p + 1] = ix->pad_prefix[p] + pads[p];

    cudaStream_t st = nullptr;
    auto up = [&](DevBuf &b, const void *src, size_t bytes) {
        b.ensure(std::max<size_t>(bytes, 16));
        if (bytes) LGPU_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, st));
        ix->device_bytes += b.bytes;
    };
    up(ix->part_n, part_n.data(), (size_t)nlist * 4);
    up(ix->part_npad, part_npad.data(), (size_t)nlist * 4);
    up(ix->part_off, part_offsets, (size_t)(nlist + 1) * 8);
    up(ix->row_ids, row_ids, (size_t)nrows * 8);
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// IVF_SQ stored rows: dim zero-padded to the scan's K step
static uint32_t sq_dim_pad(uint32_t dim) { return (uint32_t)round_up64(dim, SQ_K_CHUNK); }

// codes [n][dim] (host) -> dst [n][dim_pad] (device, zero padding) and xx[r] = sum of row r's squared codes
static void upload_sq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, DevBuf &dst, DevBuf &xx)
{
    const uint32_t dim_pad = sq_dim_pad(dim);
    dst.ensure(std::max<size_t>((size_t)n * dim_pad, 16));
    xx.ensure(std::max<size_t>((size_t)n * 4, 16));
    cudaStream_t st = nullptr;
    LGPU_CUDA(cudaMemsetAsync(dst.p, 0, dst.bytes, st));
    if (n) {
        LGPU_CUDA(cudaMemcpy2DAsync(dst.p, dim_pad, codes, dim, dim, n, cudaMemcpyHostToDevice, st));
        launch_sq_row_norms(dst.as<uint8_t>(), n, dim_pad, xx.as<uint32_t>(), st);
    }
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// IVF_RQ stored rows: dim zero-padded to the scan's K step, in 32-bit words
static uint32_t rq_wpr(uint32_t dim) { return (uint32_t)round_up64(dim, RQ_K_BITS) / 32; }

// codes [n][ceil(dim / 8)] (host) -> dst [n][wpr] u32 (device, zero padding, bits past dim cleared) and popc[r]
static void upload_rq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, DevBuf &dst, DevBuf &popc)
{
    const uint32_t wpr = rq_wpr(dim), nb = (dim + 7) / 8;
    dst.ensure(std::max<size_t>((size_t)n * wpr * 4, 16));
    popc.ensure(std::max<size_t>((size_t)n * 4, 16));
    cudaStream_t st = nullptr;
    LGPU_CUDA(cudaMemsetAsync(dst.p, 0, dst.bytes, st));
    if (n) {
        LGPU_CUDA(cudaMemcpy2DAsync(dst.p, (size_t)wpr * 4, codes, nb, nb, n, cudaMemcpyHostToDevice, st));
        launch_rq_row_prep(dst.as<uint32_t>(), n, dim, wpr, popc.as<uint32_t>(), st);
    }
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// 4-bit IVF_PQ codes: per partition [m/2][npad] bytes (zero padding rows) at code_base[p] = m/2 x the npad of the
// partitions before it.  Returns the total bytes.
static uint64_t pq4_code_base(const uint64_t *part_offsets, uint32_t nlist, uint32_t m, std::vector<uint64_t> &code_base)
{
    code_base.resize(nlist);
    uint64_t cb = 0;
    for (uint32_t p = 0; p < nlist; p++) {
        code_base[p] = cb;
        cb += (uint64_t)(m / 2) * (((part_offsets[p + 1] - part_offsets[p]) + 31u) & ~31ull);
        LGPU_REQUIRE((cb >> 3) < (1ull << 32), "index too large for one GPU shard (re-laid-out codes above 32 GiB)");
    }
    return cb;
}

// host codes (m/2 bytes per row, `layout`) -> dst laid out for the 4-bit scan, on the legacy stream
static void upload_pq4_codes(const uint8_t *codes, int layout, uint64_t nrows, uint32_t m, uint32_t nlist,
                             const uint64_t *d_part_off, const uint64_t *d_code_base, const uint32_t *d_part_npad,
                             uint64_t total, DevBuf &dst)
{
    cudaStream_t st = nullptr;
    dst.ensure(std::max<uint64_t>(total, 16));
    LGPU_CUDA(cudaMemsetAsync(dst.p, 0, dst.bytes, st));
    if (nrows) {
        DevBuf tmp;
        const size_t bytes = (size_t)nrows * (m / 2);
        tmp.ensure(bytes);
        LGPU_CUDA(cudaMemcpyAsync(tmp.p, codes, bytes, cudaMemcpyHostToDevice, st));
        launch_pq4_relayout(tmp.as<uint8_t>(), layout, d_part_off, nlist, nrows, m, d_code_base, d_part_npad,
                            dst.as<uint8_t>(), st);
        LGPU_CUDA(cudaStreamSynchronize(st));
    }
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// lgpu_index_open with nbits = 4 (the desc's common fields are checked): the IVF arrays, the codebook and the codes
// re-laid out for pq4_tables / pq4_scan.  No filter tables: the scan is exact.
static void open_pq4(const lgpu_index_desc *d, lgpu_index *&ix)
{
    LGPU_REQUIRE(d->m % 2 == 0, "num_sub_vectors must be even for 4-bit PQ codes");
    LGPU_REQUIRE(d->m <= LGPU_PQ4_MAX_M, "4-bit PQ codes support num_sub_vectors up to 256");
    std::vector<uint64_t> code_base;
    const uint64_t total = pq4_code_base(d->part_offsets, d->nlist, d->m, code_base);
    require_device(d->device);
    ix = new lgpu_index();
    ix->is_pq4 = true;
    ix->m = d->m; ix->dsub = d->dim / d->m; ix->nch = (d->m + 7) / 8;
    open_ivf_common(ix, d->device, d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->row_ids,
                    d->vectors, PQ4_ROWS_TILE);
    ix->code_base.ensure((size_t)d->nlist * 8);
    LGPU_CUDA(cudaMemcpy(ix->code_base.p, code_base.data(), (size_t)d->nlist * 8, cudaMemcpyHostToDevice));
    // codebook [m][16][dsub] -> [m][dsub][16], the layout the table kernel reads
    const uint32_t m = d->m, dsub = ix->dsub;
    std::vector<float> cbt((size_t)m * 16 * dsub);
    for (uint32_t i = 0; i < m; i++)
        for (uint32_t j = 0; j < 16; j++)
            for (uint32_t t = 0; t < dsub; t++)
                cbt[((size_t)i * dsub + t) * 16 + j] = d->codebook[((size_t)i * 16 + j) * dsub + t];
    ix->pq4_cb.ensure(cbt.size() * 4);
    LGPU_CUDA(cudaMemcpy(ix->pq4_cb.p, cbt.data(), cbt.size() * 4, cudaMemcpyHostToDevice));
    upload_pq4_codes(d->codes, d->codes_layout, d->nrows, d->m, d->nlist, ix->part_off.as<uint64_t>(),
                     ix->code_base.as<uint64_t>(), ix->part_npad.as<uint32_t>(), total, ix->codes);
    ix->device_bytes += ix->code_base.bytes + ix->pq4_cb.bytes + ix->codes.bytes;
}

}  // namespace

extern "C" {

const char *lgpu_last_error(void) { return g_err.c_str(); }
uint32_t lgpu_abi_version(void) { return LGPU_ABI_VERSION; }

int lgpu_device_count(int *count)
{
    return guarded([&] {
        LGPU_REQUIRE(count != nullptr, "count is null");
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
        *count = n;
    });
}

int lgpu_index_open(const lgpu_index_desc *d, lgpu_index **out)
{
    lgpu_index *ix = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(d != nullptr && out != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->dim > 0 && d->nlist > 0 && d->m > 0, "dim, nlist and m must be positive");
        LGPU_REQUIRE(d->dim % d->m == 0, "num_sub_vectors must divide the vector dimension");
        LGPU_REQUIRE(d->nbits == 8 || d->nbits == 4, "num_bits must be 4 or 8");
        LGPU_REQUIRE(d->codes_layout == LGPU_CODES_ROW_MAJOR || d->codes_layout == LGPU_CODES_PARTITION_TRANSPOSED,
                     "unknown codes layout");
        LGPU_REQUIRE(scan_dsub_supported(d->dim / d->m),
                     "unsupported PQ sub-vector length (dim/num_sub_vectors must be 1,2,4,8,16 or 32)");
        LGPU_REQUIRE(d->codebook, "null index array");
        check_ivf_layout(d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->codes, d->row_ids);
        if (d->nbits == 4) {
            open_pq4(d, ix);
            register_handle(ix);
            *out = ix;
            return;
        }
        const uint32_t nlist = d->nlist, nch = (d->m + 7) / 8;
        std::vector<uint64_t> code_base(nlist);
        uint64_t cb = 0;
        for (uint32_t p = 0; p < nlist; p++) {
            code_base[p] = cb;
            cb += (uint64_t)(nch + 1) * (((d->part_offsets[p + 1] - d->part_offsets[p]) + 31u) & ~31ull) * 8;
            LGPU_REQUIRE((cb >> 3) < (1ull << 32), "index too large for one GPU shard (re-laid-out codes above 32 GiB)");
        }
        require_device(d->device);
        ix = new lgpu_index();
        ix->m = d->m; ix->dsub = d->dim / d->m; ix->nch = nch;
        open_ivf_common(ix, d->device, d->dim, nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->row_ids,
                        d->vectors, SCAN_ROWS_TILE_MID);
        cudaStream_t st = nullptr;
        auto up = [&](DevBuf &b, const void *src, size_t bytes) {
            b.ensure(std::max<size_t>(bytes, 16));
            if (bytes) LGPU_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, st));
            ix->device_bytes += b.bytes;
        };
        up(ix->code_base, code_base.data(), (size_t)nlist * 8);
        // codebook -> [nch][256][8][dsub]
        {
            DevBuf tmp;
            size_t bytes = (size_t)d->m * 256 * ix->dsub * 4;
            tmp.ensure(bytes);
            LGPU_CUDA(cudaMemcpyAsync(tmp.p, d->codebook, bytes, cudaMemcpyHostToDevice, st));
            ix->cb_tiled.ensure((size_t)ix->nch * 256 * 8 * ix->dsub * 4);
            ix->device_bytes += ix->cb_tiled.bytes;
            launch_retile_codebook(tmp.as<float>(), d->m, ix->dsub, ix->nch, ix->cb_tiled.as<float>(), st);
            LGPU_CUDA(cudaStreamSynchronize(st));
        }
        // codes -> skewed streams
        {
            ix->codes.ensure(std::max<uint64_t>(cb, 16));
            ix->device_bytes += ix->codes.bytes;
            LGPU_CUDA(cudaMemsetAsync(ix->codes.p, 0, ix->codes.bytes, st));
            DevBuf tmp;
            size_t bytes = (size_t)d->nrows * d->m;
            if (bytes) {
                tmp.ensure(bytes);
                LGPU_CUDA(cudaMemcpyAsync(tmp.p, d->codes, bytes, cudaMemcpyHostToDevice, st));
                launch_retile_codes(tmp.as<unsigned char>(), d->codes_layout, ix->part_off.as<uint64_t>(), nlist,
                                    d->nrows, d->m, ix->nch, ix->code_base.as<uint64_t>(),
                                    ix->part_npad.as<uint32_t>(), ix->codes.as<unsigned char>(), st);
            }
            LGPU_CUDA(cudaStreamSynchronize(st));
        }
        {   // |b|^2 of the tiled codebook entries and CB2 = sum_i max_c |b|^2 (filter scan, tables.cu)
            const size_t ne = (size_t)ix->nch * 256 * 8;
            ix->cb_n2.ensure(ne * 4);
            ix->device_bytes += ix->cb_n2.bytes;
            launch_cb_norms(ix->cb_tiled.as<float>(), ix->nch, ix->dsub, ix->cb_n2.as<float>(), st);
            double cb2 = 0.0;
            for (uint32_t i = 0; i < d->m; i++) {
                double mx = 0.0;
                for (uint32_t c = 0; c < 256; c++) {
                    double n2 = 0.0;
                    const float *e = d->codebook + ((size_t)i * 256 + c) * ix->dsub;
                    for (uint32_t t = 0; t < ix->dsub; t++) n2 += (double)e[t] * e[t];
                    mx = std::max(mx, n2);
                }
                cb2 += mx;
            }
            ix->cb2 = (float)(cb2 * 1.000001);
        }
        if (d->metric != LGPU_DOT) {   // per-row constants of the filter scan (tables.cu)
            ix->row_R.ensure(std::max<size_t>((size_t)d->nrows * 4, 16));
            ix->rmax_bits.ensure(16);
            ix->device_bytes += ix->row_R.bytes;
            launch_row_const(ix->codes.as<unsigned char>(), ix->code_base.as<uint64_t>(), ix->part_npad.as<uint32_t>(),
                             ix->part_off.as<uint64_t>(), nlist, d->nrows, ix->centroids.as<float>(),
                             ix->cb_tiled.as<float>(), d->dim, d->m, ix->dsub, ix->row_R.as<float>(),
                             ix->rmax_bits.as<int>(), st);
            LGPU_CUDA(cudaStreamSynchronize(st));
        }
        ix->has_tables = true;
        register_handle(ix);
        *out = ix;
    });
    if (rc != LGPU_OK && ix) delete ix;
    return rc;
}

int lgpu_ivf_sq_open(const lgpu_ivf_sq_desc *d, lgpu_index **out)
{
    lgpu_index *ix = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(d != nullptr && out != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->metric != LGPU_DOT, "IVF_SQ supports the l2 and cosine distance types, not dot");
        LGPU_REQUIRE(d->dim <= LGPU_SQ_MAX_DIM, "IVF_SQ supports dimensions up to 65536");
        LGPU_REQUIRE(std::isfinite(d->lo) && std::isfinite(d->hi) && d->lo <= d->hi,
                     "IVF_SQ bounds must be finite with lo <= hi");
        check_ivf_layout(d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->codes, d->row_ids);
        require_device(d->device);
        ix = new lgpu_index();
        ix->is_sq = true;
        ix->dim_pad = sq_dim_pad(d->dim);
        ix->sq_lo = d->lo; ix->sq_hi = d->hi;
        open_ivf_common(ix, d->device, d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->row_ids,
                        d->vectors, SQ_ROWS_TILE);
        // byte offset of each partition's codes (the tile descriptors carry it; the SQ scan addresses rows by part_off)
        std::vector<uint64_t> code_base(d->nlist);
        for (uint32_t p = 0; p < d->nlist; p++) code_base[p] = d->part_offsets[p] * ix->dim_pad;
        ix->code_base.ensure((size_t)d->nlist * 8);
        LGPU_CUDA(cudaMemcpy(ix->code_base.p, code_base.data(), (size_t)d->nlist * 8, cudaMemcpyHostToDevice));
        upload_sq_rows(d->codes, d->nrows, d->dim, ix->codes, ix->sq_xx);
        ix->device_bytes += ix->code_base.bytes + ix->codes.bytes + ix->sq_xx.bytes;
        register_handle(ix);
        *out = ix;
    });
    if (rc != LGPU_OK && ix) delete ix;
    return rc;
}

int lgpu_debug_sq_distances(const uint8_t *q_codes, uint32_t B, const uint8_t *x_codes, uint64_t N, uint32_t dim,
                            int device, uint32_t *out)
{
    return guarded([&] {
        LGPU_REQUIRE(dim >= 1 && dim <= LGPU_SQ_MAX_DIM, "dim must be in [1, 65536]");
        LGPU_REQUIRE(B == 0 || N == 0 || (q_codes && x_codes && out), "null buffer");
        LGPU_REQUIRE(N < (1ull << 31) && (uint64_t)B * N < (1ull << 32), "B x N must stay below 2^32");
        if (B == 0 || N == 0) return;
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        DevBuf X, xx, Q, qq, D, tiles, ctr;
        upload_sq_rows(x_codes, N, dim, X, xx);
        upload_sq_rows(q_codes, B, dim, Q, qq);
        // one partition of N rows that every query probes: tiles of SQ_ROWS_TILE rows x 8 queries, query b's
        // distances at out + b N
        std::vector<TileDesc> h;
        for (uint32_t q0 = 0; q0 < B; q0 += SCAN_G)
            for (uint64_t r0 = 0; r0 < N; r0 += SQ_ROWS_TILE) {
                TileDesc t{};
                t.row0 = (uint32_t)r0; t.nrows = (uint32_t)std::min<uint64_t>(SQ_ROWS_TILE, N - r0);
                t.ng = std::min<uint32_t>(SCAN_G, B - q0); t.n_p = (uint32_t)N;
                for (uint32_t g = 0; g < t.ng; g++) { t.q[g] = q0 + g; t.out[g] = (uint32_t)((q0 + g) * N); }
                h.push_back(t);
            }
        const uint32_t total = (uint32_t)h.size(), zero[2] = {total, 0u};
        tiles.ensure(h.size() * sizeof(TileDesc));
        ctr.ensure(8);
        D.ensure((size_t)B * N * 4);
        LGPU_CUDA(cudaMemcpy(tiles.p, h.data(), h.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(ctr.p, zero, 8, cudaMemcpyHostToDevice));
        SqScanArgs a{};
        a.codes = X.as<uint8_t>(); a.xx = xx.as<uint32_t>(); a.qcodes = Q.as<uint8_t>(); a.qq = qq.as<uint32_t>();
        a.dim_pad = sq_dim_pad(dim); a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1;
        a.tile_desc = tiles.as<TileDesc>(); a.dist_out = D.as<float>(); a.out_u32 = 1;
        launch_sq_scan(a, 2 * prop.multiProcessorCount, nullptr);
        LGPU_CUDA(cudaMemcpy(out, D.p, (size_t)B * N * 4, cudaMemcpyDeviceToHost));
    });
}

int lgpu_debug_pq4_sums(const uint8_t *tables, uint32_t B, const uint8_t *codes, uint64_t N, uint32_t m, int device,
                        uint32_t *out)
{
    return guarded([&] {
        LGPU_REQUIRE(m >= 2 && m % 2 == 0 && m <= LGPU_PQ4_MAX_M, "m must be even and in [2, 256]");
        LGPU_REQUIRE(B == 0 || N == 0 || (tables && codes && out), "null buffer");
        LGPU_REQUIRE(N < (1ull << 31) && (uint64_t)B * ((N + 3) & ~3ull) < (1ull << 32), "B x N must stay below 2^32");
        if (B == 0 || N == 0) return;
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        // one partition of N rows that every query probes as its own slot: tiles of PQ4_ROWS_TILE rows x 8 slots,
        // query b's sums at b * ld (segments padded to 4, as in a search)
        const uint64_t off[2] = {0, N}, ld = (N + 3) & ~3ull;
        const uint32_t npad = (uint32_t)((N + 31) & ~31ull);
        std::vector<uint64_t> code_base;
        const uint64_t total_bytes = pq4_code_base(off, 1, m, code_base);
        DevBuf d_off, d_cb, d_npad, X, tab, sl, D, tiles, ctr;
        d_off.ensure(16); d_cb.ensure(8); d_npad.ensure(4);
        LGPU_CUDA(cudaMemcpy(d_off.p, off, 16, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(d_cb.p, code_base.data(), 8, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(d_npad.p, &npad, 4, cudaMemcpyHostToDevice));
        upload_pq4_codes(codes, LGPU_CODES_ROW_MAJOR, N, m, 1, d_off.as<uint64_t>(), d_cb.as<uint64_t>(),
                         d_npad.as<uint32_t>(), total_bytes, X);
        tab.ensure((size_t)B * m * 16); sl.ensure((size_t)B * sizeof(Pq4Slot));
        LGPU_CUDA(cudaMemcpy(tab.p, tables, (size_t)B * m * 16, cudaMemcpyHostToDevice));
        std::vector<TileDesc> h;
        const uint32_t nrb = scan_nrb((uint32_t)N, PQ4_ROWS_TILE), rbr = scan_rb_rows((uint32_t)N, nrb);
        for (uint32_t q0 = 0; q0 < B; q0 += SCAN_G)
            for (uint32_t rb = 0; rb < nrb; rb++) {
                TileDesc t{};
                t.row0 = rb * rbr; t.nrows = std::min<uint32_t>(rbr, (uint32_t)N - t.row0);
                t.ng = std::min<uint32_t>(SCAN_G, B - q0); t.n_p = (uint32_t)N; t.npad = npad;
                for (uint32_t g = 0; g < t.ng; g++) { t.slot[g] = q0 + g; t.q[g] = q0 + g; t.out[g] = (uint32_t)((q0 + g) * ld); }
                h.push_back(t);
            }
        const uint32_t total = (uint32_t)h.size(), zero[2] = {total, 0u};
        tiles.ensure(h.size() * sizeof(TileDesc));
        ctr.ensure(8);
        D.ensure((size_t)B * ld * 4);
        LGPU_CUDA(cudaMemcpy(tiles.p, h.data(), h.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(ctr.p, zero, 8, cudaMemcpyHostToDevice));
        Pq4ScanArgs a{};
        a.codes = X.as<uint32_t>(); a.tables = tab.as<uint8_t>(); a.slots = sl.as<Pq4Slot>(); a.m = m; a.metric = LGPU_L2;
        a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1; a.tile_desc = tiles.as<TileDesc>();
        a.dist_out = D.as<float>(); a.out_u32 = 1;
        launch_pq4_scan(a, 2 * prop.multiProcessorCount, nullptr);
        LGPU_CUDA(cudaMemcpy2D(out, (size_t)N * 4, D.p, (size_t)ld * 4, (size_t)N * 4, B, cudaMemcpyDeviceToHost));
    });
}

int lgpu_ivf_rq_open(const lgpu_ivf_rq_desc *d, lgpu_index **out)
{
    lgpu_index *ix = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(d != nullptr && out != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->metric != LGPU_DOT, "IVF_RQ supports the l2 and cosine distance types, not dot");
        LGPU_REQUIRE(d->num_bits == 1, "IVF_RQ supports num_bits = 1 only");
        LGPU_REQUIRE(d->dim <= LGPU_RQ_MAX_DIM, "IVF_RQ supports dimensions up to 4096");
        LGPU_REQUIRE(d->rotation != nullptr, "null index array");
        LGPU_REQUIRE(d->nrows == 0 || (d->add_factors && d->scale_factors), "null index array");
        check_ivf_layout(d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->codes, d->row_ids);
        require_device(d->device);
        ix = new lgpu_index();
        ix->is_rq = true;
        ix->rq_wpr = rq_wpr(d->dim);
        open_ivf_common(ix, d->device, d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->row_ids,
                        d->vectors, RQ_ROWS_TILE);
        // byte offset of each partition's codes (the tile descriptors carry it; the RQ scan addresses rows by part_off)
        std::vector<uint64_t> code_base(d->nlist);
        for (uint32_t p = 0; p < d->nlist; p++) code_base[p] = d->part_offsets[p] * ix->rq_wpr * 4;
        ix->code_base.ensure((size_t)d->nlist * 8);
        LGPU_CUDA(cudaMemcpy(ix->code_base.p, code_base.data(), (size_t)d->nlist * 8, cudaMemcpyHostToDevice));
        upload_rq_rows(d->codes, d->nrows, d->dim, ix->codes, ix->rq_popc);
        const size_t rows = std::max<size_t>((size_t)d->nrows * 4, 16), rot = (size_t)d->dim * d->dim * 4;
        ix->rq_add.ensure(rows); ix->rq_scale.ensure(rows); ix->rq_rot.ensure(rot);
        ix->rq_rc.ensure((size_t)d->nlist * d->dim * 4);
        if (d->nrows) {
            LGPU_CUDA(cudaMemcpy(ix->rq_add.p, d->add_factors, (size_t)d->nrows * 4, cudaMemcpyHostToDevice));
            LGPU_CUDA(cudaMemcpy(ix->rq_scale.p, d->scale_factors, (size_t)d->nrows * 4, cudaMemcpyHostToDevice));
        }
        LGPU_CUDA(cudaMemcpy(ix->rq_rot.p, d->rotation, rot, cudaMemcpyHostToDevice));
        // rc_p = P c_p, once: each probe slot's residual is then one subtraction per dimension
        launch_rq_rotate(ix->rq_rot.as<float>(), ix->centroids.as<float>(), d->nlist, d->dim, ix->rq_rc.as<float>(),
                         nullptr);
        LGPU_CUDA(cudaStreamSynchronize(nullptr));
        ix->device_bytes += ix->code_base.bytes + ix->codes.bytes + ix->rq_popc.bytes + ix->rq_add.bytes +
                            ix->rq_scale.bytes + ix->rq_rot.bytes + ix->rq_rc.bytes;
        register_handle(ix);
        *out = ix;
    });
    if (rc != LGPU_OK && ix) delete ix;
    return rc;
}

int lgpu_debug_rq_distances(const float *q_res, uint32_t B, const uint8_t *codes, const float *add_factors,
                            const float *scale_factors, uint64_t N, uint32_t dim, int metric, int device,
                            float *out_est, uint32_t *out_ip)
{
    return guarded([&] {
        LGPU_REQUIRE(dim >= 1 && dim <= LGPU_RQ_MAX_DIM, "dim must be in [1, 4096]");
        LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE, "IVF_RQ supports the l2 and cosine distance types");
        LGPU_REQUIRE(B == 0 || N == 0 || (q_res && codes && add_factors && scale_factors && (out_est || out_ip)),
                     "null buffer");
        LGPU_REQUIRE(N < (1ull << 31) && (uint64_t)B * N < (1ull << 32), "B x N must stay below 2^32");
        if (B == 0 || N == 0) return;
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        const uint32_t wpr = rq_wpr(dim);
        DevBuf X, popc, add, scale, Q, zero, probes, planes, slots, D, tiles, ctr;
        upload_rq_rows(codes, N, dim, X, popc);
        add.ensure((size_t)N * 4); scale.ensure((size_t)N * 4);
        Q.ensure((size_t)B * dim * 4); zero.ensure((size_t)dim * 4); probes.ensure((size_t)B * 8);
        planes.ensure((size_t)B * 4 * wpr * 4); slots.ensure((size_t)B * sizeof(RqSlot));
        LGPU_CUDA(cudaMemcpy(add.p, add_factors, (size_t)N * 4, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(scale.p, scale_factors, (size_t)N * 4, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(Q.p, q_res, (size_t)B * dim * 4, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemset(zero.p, 0, (size_t)dim * 4));
        LGPU_CUDA(cudaMemset(probes.p, 0, (size_t)B * 8));
        // query b is one probe slot of partition 0 whose rotated centroid is 0: q' = the given residual
        launch_rq_planes(Q.as<float>(), zero.as<float>(), probes.as<uint64_t>(), B, 1, 1, dim, wpr,
                         planes.as<uint32_t>(), slots.as<RqSlot>(), nullptr);
        // one partition of N rows that every slot probes: tiles of RQ_ROWS_TILE rows x 8 slots, slot b's row r at
        // out + b N + r
        std::vector<TileDesc> h;
        for (uint32_t q0 = 0; q0 < B; q0 += SCAN_G)
            for (uint64_t r0 = 0; r0 < N; r0 += RQ_ROWS_TILE) {
                TileDesc t{};
                t.row0 = (uint32_t)r0; t.nrows = (uint32_t)std::min<uint64_t>(RQ_ROWS_TILE, N - r0);
                t.ng = std::min<uint32_t>(SCAN_G, B - q0); t.n_p = (uint32_t)N;
                for (uint32_t g = 0; g < t.ng; g++) {
                    t.q[g] = q0 + g; t.slot[g] = q0 + g; t.out[g] = (uint32_t)((q0 + g) * N);
                }
                h.push_back(t);
            }
        tiles.ensure(h.size() * sizeof(TileDesc));
        ctr.ensure(8);
        D.ensure((size_t)B * N * 4);
        LGPU_CUDA(cudaMemcpy(tiles.p, h.data(), h.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        RqScanArgs a{};
        a.codes = X.as<uint32_t>(); a.add = add.as<float>(); a.scale = scale.as<float>(); a.popc = popc.as<uint32_t>();
        a.planes = planes.as<uint32_t>(); a.slots = slots.as<RqSlot>(); a.dim = dim; a.wpr = wpr;
        a.cosine = metric == LGPU_COSINE;
        a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1;
        a.tile_desc = tiles.as<TileDesc>(); a.dist_out = D.as<float>();
        const uint32_t total = (uint32_t)h.size(), zero2[2] = {total, 0u};
        for (int mode = 0; mode < 2; mode++) {
            void *dst = mode ? (void *)out_ip : (void *)out_est;
            if (!dst) continue;
            LGPU_CUDA(cudaMemcpy(ctr.p, zero2, 8, cudaMemcpyHostToDevice));
            a.out_ip = mode;
            launch_rq_scan(a, 2 * prop.multiProcessorCount, nullptr);
            LGPU_CUDA(cudaMemcpy(dst, D.p, (size_t)B * N * 4, cudaMemcpyDeviceToHost));
        }
    });
}

void lgpu_index_close(lgpu_index *ix) { close_handle(ix); }

int lgpu_index_device_bytes(const lgpu_index *ixh, uint64_t *bytes)
{
    return guarded([&] {
        LGPU_REQUIRE(bytes, "null argument");
        HandleRef<lgpu_index> ix(const_cast<lgpu_index *>(ixh), "index");
        *bytes = ix->device_bytes;
    });
}

int lgpu_last_scanned_code_bytes(uint64_t *bytes)
{
    return guarded([&] { LGPU_REQUIRE(bytes, "null argument"); *bytes = g_scanned_bytes; });
}

int lgpu_kernel_launch_count(uint64_t *count)
{
    return guarded([&] { LGPU_REQUIRE(count, "null argument"); *count = g_kernel_launches.load(); });
}

int lgpu_last_filter_stats(uint64_t *stats)
{
    return guarded([&] { LGPU_REQUIRE(stats, "null argument"); memcpy(stats, g_filter_stats, sizeof(g_filter_stats)); });
}

int lgpu_set_profiling(int enabled)
{
    g_profiling.store(enabled ? 1 : 0);
    return LGPU_OK;
}

int lgpu_last_stage_ms(float *times)
{
    return guarded([&] { LGPU_REQUIRE(times, "null argument"); memcpy(times, g_stage_ms, sizeof(g_stage_ms)); });
}

int lgpu_debug_sub_batch_size(lgpu_index *ixh, uint32_t B, uint32_t nprobes, uint32_t *out)
{
    return guarded([&] {
        LGPU_REQUIRE(out && B > 0 && nprobes > 0, "bad argument");
        HandleRef<lgpu_index> ix(ixh, "index");
        *out = ivf_sub_batch_size(ix.h, B, nprobes);
    });
}

static void check_ivf_call(lgpu_index *ix, const void *q, uint32_t B, const lgpu_search_params *p,
                           const void *a, const void *b, const void *c)
{
    check_call(p, B, q, a, b, c);
    LGPU_REQUIRE(p->nprobes >= 1, "minimum_nprobes must be greater than 0");
    LGPU_REQUIRE(p->nprobes <= SELECT_KMAX || p->nprobes >= ix->nlist, "nprobes above 2048 is not supported");
    LGPU_REQUIRE(p->refine_factor == 0 || ix->has_vectors,
                 "refine_factor needs the raw vectors: open the index with desc.vectors");
}

static int ivf_call(lgpu_index *ixh, const Route &r, const float *q, uint32_t B, const lgpu_search_params *p,
                    uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(ixh, "index", r, q, B, p, ids, dist, cnt,
                       [&](lgpu_index *ix) { check_ivf_call(ix, q, B, p, ids, dist, cnt); return (size_t)B * ix->dim; },
                       ivf_search_device);
}

int lgpu_search(lgpu_index *ixh, const float *queries, uint32_t B, const lgpu_search_params *params,
                uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return ivf_call(ixh, host_route(0x1f5ull), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_search_filtered(lgpu_index *ixh, const float *queries, uint32_t B, const lgpu_search_params *params,
                         const uint32_t *allow, uint64_t allow_bits, uint64_t *out_ids, float *out_dist,
                         uint32_t *out_count)
{
    return ivf_call(ixh, filtered_route(allow, allow_bits), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_search_coalesced(lgpu_index *ixh, const float *query, const lgpu_search_params *params, uint64_t *out_ids,
                          float *out_dist, uint32_t *out_count)
{
    static const uint32_t window_us = getenv("LGPU_COALESCE_US") ? (uint32_t)atoi(getenv("LGPU_COALESCE_US")) : 50u;
    constexpr size_t MAX_BATCH = 256;
    PendingQuery me{query, out_ids, out_dist, out_count};
    std::vector<PendingQuery *> batch;
    lgpu_search_params p{};
    int rc = guarded([&] {
        HandleRef<lgpu_index> ix(ixh, "index");
        check_ivf_call(ix.h, query, 1, params, out_ids, out_dist, out_count);
        p = *params;
        Coalescer &co = ix->coalescer;
        std::unique_lock<std::mutex> lk(co.mu);
        Coalescer::Lane *lane = nullptr;
        for (auto *l : co.lanes) if (memcmp(&l->params, &p, sizeof(p)) == 0) { lane = l; break; }
        if (!lane) { lane = new Coalescer::Lane(); lane->params = p; co.lanes.push_back(lane); }
        lane->queue.push_back(&me);
        if (lane->leader) {                               // follower: the lane's leader will fill our row in
            if (lane->queue.size() >= MAX_BATCH) co.cv.notify_all();
            co.cv.wait(lk, [&] { return me.done; });
            return;
        }
        lane->leader = true;                              // leader: collect for one window, then search the batch
        co.cv.wait_for(lk, std::chrono::microseconds(window_us), [&] { return lane->queue.size() >= MAX_BATCH; });
        batch.swap(lane->queue);
        lane->leader = false;
        lk.unlock();
        const uint32_t B = (uint32_t)batch.size();
        const uint32_t dim = ix->dim, k = p.k;
        std::vector<float> q((size_t)B * dim);
        std::vector<uint64_t> ids((size_t)B * k);
        std::vector<float> dist((size_t)B * k);
        std::vector<uint32_t> cnt(B);
        for (uint32_t i = 0; i < B; i++) memcpy(q.data() + (size_t)i * dim, batch[i]->q, (size_t)dim * 4);
        const int brc = lgpu_search(ix.h, q.data(), B, &p, ids.data(), dist.data(), cnt.data());
        const std::string berr = brc == LGPU_OK ? std::string() : std::string(lgpu_last_error());
        lk.lock();
        for (uint32_t i = 0; i < B; i++) {
            PendingQuery *pq = batch[i];
            pq->status = brc; pq->err = berr;
            if (brc == LGPU_OK) {
                memcpy(pq->ids, ids.data() + (size_t)i * k, (size_t)k * 8);
                memcpy(pq->dist, dist.data() + (size_t)i * k, (size_t)k * 4);
                *pq->cnt = cnt[i];
            }
            pq->done = true;
        }
        lk.unlock();
        co.cv.notify_all();
    });
    if (rc != LGPU_OK) return rc;
    if (me.status != LGPU_OK) { set_error(me.err); return me.status; }
    return LGPU_OK;
}

int lgpu_search_device(lgpu_index *ixh, const float *d_queries, uint32_t B, const lgpu_search_params *params,
                       uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count, void *cuda_stream)
{
    return ivf_call(ixh, device_route(cuda_stream), d_queries, B, params, d_out_ids, d_out_dist, d_out_count);
}

// ---- asynchronous completion (SURVEY.md 8b "Threading": a tokio worker must not be blocked for the length of a
// search -- python/src/runtime.rs:113-119 uses spawn_blocking for that today).  lgpu_search_async stages the
// queries, enqueues the search and the copy-back on a private stream and returns; lgpu_ticket_wait blocks until
// the results are in the caller's buffers.  Two tickets in flight use two workspaces/streams, so batch i+1's
// H2D overlaps batch i's kernels. ----
struct lgpu_ticket {
    HandleRef<lgpu_index> ix;
    WsLease lease;
    Deadline deadline;
    cudaEvent_t done = nullptr;
    lgpu_ticket(lgpu_index *h, uint32_t timeout_ms)
        : ix(h, "index"), lease(ix->pool, nullptr, false), deadline(timeout_ms) {}
    ~lgpu_ticket() { if (done) cudaEventDestroy(done); }
};

int lgpu_search_async(lgpu_index *ixh, const float *queries, uint32_t B, const lgpu_search_params *params,
                      uint64_t *out_ids, float *out_dist, uint32_t *out_count, lgpu_ticket **ticket)
{
    lgpu_ticket *t = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(ticket != nullptr, "ticket is null");
        LGPU_REQUIRE(params != nullptr, "search params are null");
        {   // validate before taking a workspace
            HandleRef<lgpu_index> ix(ixh, "index");
            check_ivf_call(ix.h, queries, B, params, out_ids, out_dist, out_count);
            require_device(ix->device);
        }
        t = new lgpu_ticket(ixh, params->timeout_ms);
        LGPU_CUDA(cudaEventCreateWithFlags(&t->done, cudaEventDisableTiming));
        if (B > 0) {
            uint64_t key[4];
            make_key(key, 0x1f5ull, B, *params);
            lgpu_index *ix = t->ix.h;
            const lgpu_search_params sp = *params;
            host_submit(t->lease, t->deadline, queries, (size_t)B * ix->dim, B, sp.k, out_ids, out_dist, out_count, key,
                        [&](Workspace *ws, cudaStream_t st, const float *dq, uint64_t *di, float *dd, uint32_t *dc,
                            const Deadline &) { ivf_search_device(ix, ws, st, dq, B, sp, di, dd, dc); },
                        false);
        }
        LGPU_CUDA(cudaEventRecord(t->done, t->lease.st));
        *ticket = t;
    });
    if (rc != LGPU_OK && t) { cudaStreamSynchronize(t->lease.st); delete t; }
    return rc;
}

int lgpu_ticket_poll(lgpu_ticket *t, int *done)
{
    return guarded([&] {
        LGPU_REQUIRE(t && done, "null argument");
        cudaError_t e = cudaEventQuery(t->done);
        if (e != cudaSuccess && e != cudaErrorNotReady) LGPU_CUDA(e);
        *done = e == cudaSuccess ? 1 : 0;
    });
}

/* blocks until the call's results are in the caller's buffers, then frees the ticket.  With a timeout armed the
 * status is LGPU_TIMEOUT when the deadline passed first -- the wait still runs to completion, because a DMA into
 * the caller's buffers may not be left in flight. */
int lgpu_ticket_wait(lgpu_ticket *t)
{
    if (!t) { set_error("ticket is null"); return LGPU_INVALID_INPUT; }
    int rc = guarded([&] {
        bool late = false;
        if (t->deadline.armed) {
            for (;;) {
                cudaError_t e = cudaEventQuery(t->done);
                if (e == cudaSuccess) break;
                if (e != cudaErrorNotReady) LGPU_CUDA(e);
                if (t->deadline.expired()) { late = true; break; }
                std::this_thread::sleep_for(std::chrono::microseconds(50));
            }
        }
        LGPU_CUDA(cudaEventSynchronize(t->done));
        if (late) { set_error("Query timeout"); throw Failure{LGPU_TIMEOUT}; }
    });
    delete t;
    return rc;
}

int lgpu_merge_topk_device(int device, uint32_t nlists, uint32_t B, uint32_t k, const uint64_t *d_ids,
                           const float *d_dist, uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count,
                           void *cuda_stream)
{
    return guarded([&] {
        LGPU_REQUIRE(nlists >= 1 && k >= 1 && k <= SELECT_KMAX, "bad merge shape");
        LGPU_REQUIRE(B == 0 || (d_ids && d_dist && d_out_ids && d_out_dist && d_out_count), "null buffer");
        if (B == 0) return;
        require_device(device);
        // list l of query q at l * B * k + q * k
        SelectArgs sb = select_cands(d_dist, d_ids, k, B, k, {d_out_ids, d_out_dist, d_out_count});
        sb.ncols = (uint64_t)nlists * k; sb.outer_stride = (uint64_t)B * k;
        launch_select(sb, (cudaStream_t)cuda_stream);
    });
}

int lgpu_flat_open(const float *vectors, uint64_t nrows, uint32_t dim, const uint64_t *row_ids, int device,
                   lgpu_flat **out)
{
    lgpu_flat *fl = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr && dim > 0, "null argument / zero dimension");
        LGPU_REQUIRE(nrows == 0 || vectors != nullptr, "null vectors");
        require_device(device);
        fl = new lgpu_flat();
        fl->device = device; fl->nrows = nrows; fl->dim = dim;
        fl->vectors.ensure(std::max<size_t>((size_t)nrows * dim * 4, 16));
        if (nrows) LGPU_CUDA(cudaMemcpy(fl->vectors.p, vectors, (size_t)nrows * dim * 4, cudaMemcpyHostToDevice));
        if (gemm_shape_supported(dim) && nrows >= 4096) {
            prepare_tc_operand(fl->vectors.as<float>(), nrows, dim, fl->vec_b, fl->vec_n2, fl->vec_max, fl->vec_err, nullptr);
            fl->has_tc = true;
        }
        open_rows(fl, row_ids, nrows);
        register_handle(fl);
        *out = fl;
    });
    if (rc != LGPU_OK && fl) delete fl;
    return rc;
}

void lgpu_flat_close(lgpu_flat *fl) { close_handle(fl); }

static int flat_call(lgpu_flat *flh, int metric, const Route &r, const float *q, uint32_t B,
                     const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(flh, "flat", r, q, B, p, ids, dist, cnt,
                       [&](lgpu_flat *fl) {
                           LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE || metric == LGPU_DOT,
                                        "unknown distance type");
                           check_call(p, B, q, ids, dist, cnt);
                           return (size_t)B * fl->dim;
                       },
                       [&](lgpu_flat *fl, Workspace *ws, cudaStream_t st, auto &&...a) {
                           flat_search_device(fl, ws, st, metric, a...);
                       });
}

int lgpu_flat_search(lgpu_flat *flh, int metric, const float *queries, uint32_t B, const lgpu_search_params *params,
                     uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return flat_call(flh, metric, host_route(0xf1a7ull + (uint64_t)metric), queries, B, params, out_ids, out_dist,
                     out_count);
}

int lgpu_flat_search_filtered(lgpu_flat *flh, int metric, const float *queries, uint32_t B,
                              const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                              uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return flat_call(flh, metric, filtered_route(allow, allow_bits), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_flat_search_device(lgpu_flat *flh, int metric, const float *d_queries, uint32_t B,
                            const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                            uint32_t *d_out_count, void *cuda_stream)
{
    return flat_call(flh, metric, device_route(cuda_stream), d_queries, B, params, d_out_ids, d_out_dist,
                     d_out_count);
}

int lgpu_binary_open(const uint8_t *vectors, uint64_t nrows, uint32_t nbytes, const uint64_t *row_ids, int device,
                     lgpu_binary **out)
{
    lgpu_binary *bx = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr && nbytes > 0, "null argument / zero bytes per vector");
        LGPU_REQUIRE((uint64_t)nbytes * 8 <= ((uint64_t)1 << 24), "binary vectors above 2^24 bits are not supported");
        LGPU_REQUIRE(nrows == 0 || vectors != nullptr, "null vectors");
        require_device(device);
        bx = new lgpu_binary();
        bx->device = device; bx->nrows = nrows; bx->nbytes = nbytes; bx->nbytes_pad = (nbytes + 31) & ~31u;
        const uint32_t nbp = bx->nbytes_pad;
        bx->vectors.ensure(std::max<size_t>((size_t)nrows * nbp, 16));
        bx->pop.ensure(std::max<size_t>((size_t)nrows * 4, 16));
        if (nrows) {
            DevBuf raw;
            raw.ensure((size_t)nrows * nbytes);
            LGPU_CUDA(cudaMemcpy(raw.p, vectors, (size_t)nrows * nbytes, cudaMemcpyHostToDevice));
            launch_ham_pack(raw.as<uint8_t>(), nbytes, nbytes, nrows, bx->vectors.as<uint8_t>(), nbp, bx->pop.as<uint32_t>(),
                            nullptr);
        }
        if (nrows > HAM_SAMPLE) {
            const uint64_t stride = nrows / HAM_SAMPLE;
            bx->nsample = HAM_SAMPLE;
            bx->sample.ensure((size_t)HAM_SAMPLE * nbp);
            bx->sample_pop.ensure((size_t)HAM_SAMPLE * 4);
            launch_ham_pack(bx->vectors.as<uint8_t>(), stride * nbp, nbp, HAM_SAMPLE, bx->sample.as<uint8_t>(), nbp,
                            bx->sample_pop.as<uint32_t>(), nullptr);
        }
        LGPU_CUDA(cudaDeviceSynchronize());
        open_rows(bx, row_ids, nrows);
        register_handle(bx);
        *out = bx;
    });
    if (rc != LGPU_OK && bx) delete bx;
    return rc;
}

void lgpu_binary_close(lgpu_binary *bx) { close_handle(bx); }

static int binary_call(lgpu_binary *bxh, const Route &r, const uint8_t *q, uint32_t B, const lgpu_search_params *p,
                       uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(bxh, "binary", r, q, B, p, ids, dist, cnt,
                       [&](lgpu_binary *bx) { check_call(p, B, q, ids, dist, cnt); return (size_t)B * bx->nbytes; },
                       binary_search_device);
}

int lgpu_binary_search(lgpu_binary *bxh, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                       uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return binary_call(bxh, host_route(0xb1a7ull), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_binary_search_filtered(lgpu_binary *bxh, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                                const uint32_t *allow, uint64_t allow_bits, uint64_t *out_ids, float *out_dist,
                                uint32_t *out_count)
{
    return binary_call(bxh, filtered_route(allow, allow_bits), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_binary_search_device(lgpu_binary *bxh, const uint8_t *d_queries, uint32_t B, const lgpu_search_params *params,
                              uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count, void *cuda_stream)
{
    return binary_call(bxh, device_route(cuda_stream), d_queries, B, params, d_out_ids, d_out_dist, d_out_count);
}

int lgpu_ivf_binary_open(const lgpu_ivf_binary_desc *d, lgpu_ivf_binary **out)
{
    lgpu_ivf_binary *ix = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(d != nullptr && out != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->nbytes > 0, "zero bytes per vector");
        LGPU_REQUIRE((uint64_t)d->nbytes * 8 <= ((uint64_t)1 << 24), "binary vectors above 2^24 bits are not supported");
        check_ivf_layout(d->nbytes, d->nlist, LGPU_L2, d->nrows, d->centroids, d->part_offsets, d->vectors, d->row_ids);
        require_device(d->device);
        ix = new lgpu_ivf_binary();
        ix->nbytes = d->nbytes; ix->nbytes_pad = (d->nbytes + 31) & ~31u;
        ix->dim = d->nbytes;
        open_ivf_partitions(ix, d->device, d->nlist, d->nrows, d->part_offsets, d->row_ids, HAM_ROWS_TILE);
        // centroids and rows zero-padded to nbytes_pad, with their popcounts (ham_pack)
        const uint32_t nb = d->nbytes, nbp = ix->nbytes_pad;
        auto pack = [&](const uint8_t *src, uint64_t n, DevBuf &dst, DevBuf &pop) {
            dst.ensure(std::max<size_t>((size_t)n * nbp, 16));
            pop.ensure(std::max<size_t>((size_t)n * 4, 16));
            if (n) {
                DevBuf raw;
                raw.ensure((size_t)n * nb);
                LGPU_CUDA(cudaMemcpy(raw.p, src, (size_t)n * nb, cudaMemcpyHostToDevice));
                launch_ham_pack(raw.as<uint8_t>(), nb, nb, n, dst.as<uint8_t>(), nbp, pop.as<uint32_t>(), nullptr);
                LGPU_CUDA(cudaStreamSynchronize(nullptr));
            }
            ix->device_bytes += dst.bytes + pop.bytes;
        };
        pack(d->centroids, d->nlist, ix->centroids, ix->cent_pop);
        pack(d->vectors, d->nrows, ix->codes, ix->row_pop);
        // the tile descriptors' code offset is unused (the scan addresses rows by part_off)
        ix->code_base.ensure((size_t)d->nlist * 8);
        LGPU_CUDA(cudaMemset(ix->code_base.p, 0, (size_t)d->nlist * 8));
        ix->device_bytes += ix->code_base.bytes;
        register_handle(ix);
        *out = ix;
    });
    if (rc != LGPU_OK && ix) delete ix;
    return rc;
}

void lgpu_ivf_binary_close(lgpu_ivf_binary *ix) { close_handle(ix); }

static int ivf_binary_call(lgpu_ivf_binary *ixh, const Route &r, const uint8_t *q, uint32_t B,
                           const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(ixh, "binary IVF index", r, q, B, p, ids, dist, cnt,
                       [&](lgpu_ivf_binary *ix) {
                           check_call(p, B, q, ids, dist, cnt, false);   // refine_factor: exact distances
                           LGPU_REQUIRE(p->nprobes >= 1, "minimum_nprobes must be greater than 0");
                           LGPU_REQUIRE(p->nprobes <= SELECT_KMAX || p->nprobes >= ix->nlist,
                                        "nprobes above 2048 is not supported unless it covers every partition");
                           return (size_t)B * ix->nbytes;
                       },
                       ivf_binary_search_device);
}

int lgpu_ivf_binary_search(lgpu_ivf_binary *ixh, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                           uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return ivf_binary_call(ixh, host_route(0x1fb1ull), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_ivf_binary_search_filtered(lgpu_ivf_binary *ixh, const uint8_t *queries, uint32_t B,
                                    const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                    uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return ivf_binary_call(ixh, filtered_route(allow, allow_bits), queries, B, params, out_ids, out_dist, out_count);
}

int lgpu_ivf_binary_search_device(lgpu_ivf_binary *ixh, const uint8_t *d_queries, uint32_t B,
                                  const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                                  uint32_t *d_out_count, void *cuda_stream)
{
    return ivf_binary_call(ixh, device_route(cuda_stream), d_queries, B, params, d_out_ids, d_out_dist, d_out_count);
}

int lgpu_debug_ivf_hamming_scan(const uint8_t *queries, uint32_t B, const uint8_t *vectors, uint64_t N, uint32_t nbytes,
                                int device, uint32_t *out)
{
    return guarded([&] {
        LGPU_REQUIRE(nbytes > 0 && (uint64_t)nbytes * 8 <= ((uint64_t)1 << 24), "bytes per vector out of range");
        LGPU_REQUIRE(B == 0 || N == 0 || (queries && vectors && out), "null buffer");
        LGPU_REQUIRE(N < (1ull << 31) && (uint64_t)B * N < (1ull << 32), "B x N must stay below 2^32");
        if (B == 0 || N == 0) return;
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        const uint32_t nbp = (nbytes + 31) & ~31u;
        DevBuf rq, rx, q, x, qp, xp, D, tiles, ctr;
        rq.ensure((size_t)B * nbytes); rx.ensure((size_t)N * nbytes);
        q.ensure((size_t)B * nbp); x.ensure((size_t)N * nbp); qp.ensure((size_t)B * 4); xp.ensure((size_t)N * 4);
        LGPU_CUDA(cudaMemcpy(rq.p, queries, (size_t)B * nbytes, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(rx.p, vectors, (size_t)N * nbytes, cudaMemcpyHostToDevice));
        launch_ham_pack(rq.as<uint8_t>(), nbytes, nbytes, B, q.as<uint8_t>(), nbp, qp.as<uint32_t>(), nullptr);
        launch_ham_pack(rx.as<uint8_t>(), nbytes, nbytes, N, x.as<uint8_t>(), nbp, xp.as<uint32_t>(), nullptr);
        // one partition of N rows that every query probes: tiles of HAM_ROWS_TILE rows x 8 queries, query b's row r at
        // out + b N + r
        std::vector<TileDesc> h;
        for (uint32_t q0 = 0; q0 < B; q0 += SCAN_G)
            for (uint64_t r0 = 0; r0 < N; r0 += HAM_ROWS_TILE) {
                TileDesc t{};
                t.row0 = (uint32_t)r0; t.nrows = (uint32_t)std::min<uint64_t>(HAM_ROWS_TILE, N - r0);
                t.ng = std::min<uint32_t>(SCAN_G, B - q0); t.n_p = (uint32_t)N;
                for (uint32_t g = 0; g < t.ng; g++) {
                    t.q[g] = q0 + g; t.slot[g] = q0 + g; t.out[g] = (uint32_t)((q0 + g) * N);
                }
                h.push_back(t);
            }
        tiles.ensure(h.size() * sizeof(TileDesc));
        ctr.ensure(8);
        D.ensure((size_t)B * N * 4);
        LGPU_CUDA(cudaMemcpy(tiles.p, h.data(), h.size() * sizeof(TileDesc), cudaMemcpyHostToDevice));
        const uint32_t zero2[2] = {(uint32_t)h.size(), 0u};
        LGPU_CUDA(cudaMemcpy(ctr.p, zero2, 8, cudaMemcpyHostToDevice));
        HamScanArgs a{};
        a.rows = x.as<uint8_t>(); a.row_pop = xp.as<uint32_t>(); a.queries = q.as<uint8_t>(); a.qpop = qp.as<uint32_t>();
        a.nbytes_pad = nbp;
        a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1;
        a.tile_desc = tiles.as<TileDesc>(); a.dist_out = D.as<float>(); a.out_u32 = 1;
        launch_ivf_ham_scan(a, 2 * prop.multiProcessorCount, nullptr);
        LGPU_CUDA(cudaMemcpy(out, D.p, (size_t)B * N * 4, cudaMemcpyDeviceToHost));
    });
}

int lgpu_multivec_open(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                       const uint64_t *row_ids, int device, lgpu_multivec **out)
{
    lgpu_multivec *mv = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr && offsets != nullptr, "null argument");
        LGPU_REQUIRE(dim >= 1 && dim <= MV_MAX_DIM, "multivector dimension must be in [1, 65536]");
        LGPU_REQUIRE(offsets[0] == 0, "row offsets must start at 0");
        uint64_t max_row = 0;
        for (uint64_t r = 0; r < nrows; r++) {
            LGPU_REQUIRE(offsets[r + 1] >= offsets[r], "row offsets must not decrease");
            LGPU_REQUIRE(offsets[r + 1] - offsets[r] <= MV_MAX_ROW, "a multivector row holds at most 2^20 vectors");
            max_row = std::max<uint64_t>(max_row, offsets[r + 1] - offsets[r]);
        }
        const uint64_t T = offsets[nrows];
        LGPU_REQUIRE(T <= ((uint64_t)1 << 40), "a multivector column holds at most 2^40 vectors");
        LGPU_REQUIRE(T == 0 || values != nullptr, "null vectors");
        require_device(device);
        mv = new lgpu_multivec();
        mv->device = device; mv->nrows = nrows; mv->total = T; mv->dim = dim; mv->max_row = max_row;
        mv->h_offsets.assign(offsets, offsets + nrows + 1);
        mv->vectors.ensure(std::max<size_t>((size_t)T * dim * 4, 16));
        mv->ysqrt.ensure(std::max<size_t>((size_t)T * 4, 16));
        mv->offsets.ensure((size_t)(nrows + 1) * 8);
        LGPU_CUDA(cudaMemcpy(mv->offsets.p, offsets, (size_t)(nrows + 1) * 8, cudaMemcpyHostToDevice));
        if (T) {
            LGPU_CUDA(cudaMemcpy(mv->vectors.p, values, (size_t)T * dim * 4, cudaMemcpyHostToDevice));
            launch_row_norms(mv->vectors.as<float>(), T, dim, mv->ysqrt.as<float>(), nullptr);
        }
        // the tensor-core operand: only when every stored vector normalises (a zero or non-finite vector has NaN pairs,
        // which the approximate score cannot skip as the exact min does) and the shape suits the GEMM
        if (T >= MV_TC_MIN_T && T < ((uint64_t)1 << 31) && nrows < 0xffffffffull && gemm_shape_supported(dim)) {
            mv->vec_h.ensure((size_t)T * dim * 2);
            DevBuf bad;
            bad.ensure((size_t)T * 4);
            launch_mv_normalize_f16(mv->vectors.as<float>(), T, dim, mv->vec_h.p, bad.as<uint32_t>(), nullptr);
            std::vector<uint32_t> hb(T), cr(T);
            LGPU_CUDA(cudaMemcpy(hb.data(), bad.p, (size_t)T * 4, cudaMemcpyDeviceToHost));
            bool ok = true;
            for (uint64_t i = 0; i < T; i++) ok = ok && !hb[i];
            for (uint64_t r = 0; r < nrows; r++)
                for (uint64_t j = offsets[r]; j < offsets[r + 1]; j++) cr[j] = (uint32_t)r;
            mv->col_row.ensure((size_t)T * 4);
            LGPU_CUDA(cudaMemcpy(mv->col_row.p, cr.data(), (size_t)T * 4, cudaMemcpyHostToDevice));
            mv->tc_ok = ok;
        }
        LGPU_CUDA(cudaDeviceSynchronize());
        open_rows(mv, row_ids, nrows);
        register_handle(mv);
        *out = mv;
    });
    if (rc != LGPU_OK && mv) delete mv;
    return rc;
}

void lgpu_multivec_close(lgpu_multivec *mv) { close_handle(mv); }

// Host calls are never captured into a CUDA graph: the launch sequence depends on every query's vector count, not
// only on B.
static int multivec_call(lgpu_multivec *mvh, const Route &r, const float *q, const uint32_t *q_off, uint32_t B,
                         const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(mvh, "multivector", r, q, B, p, ids, dist, cnt,
                       [&](lgpu_multivec *mv) {
                           check_call(p, B, q, ids, dist, cnt);
                           if (B == 0) return (size_t)0;
                           check_multivec_offsets(q_off, B);
                           return (size_t)q_off[B] * mv->dim;
                       },
                       [&](lgpu_multivec *mv, Workspace *ws, cudaStream_t st, const float *dq, auto &&...a) {
                           multivec_search_device(mv, ws, st, dq, q_off, a...);
                       });
}

int lgpu_multivec_search(lgpu_multivec *mvh, const float *queries, const uint32_t *q_offsets, uint32_t B,
                         const lgpu_search_params *params, uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return multivec_call(mvh, host_route(0), queries, q_offsets, B, params, out_ids, out_dist, out_count);
}

int lgpu_multivec_search_filtered(lgpu_multivec *mvh, const float *queries, const uint32_t *q_offsets, uint32_t B,
                                  const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                  uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return multivec_call(mvh, filtered_route(allow, allow_bits), queries, q_offsets, B, params, out_ids, out_dist,
                         out_count);
}

int lgpu_multivec_search_device(lgpu_multivec *mvh, const float *d_queries, const uint32_t *q_offsets, uint32_t B,
                                const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                                uint32_t *d_out_count, void *cuda_stream)
{
    return multivec_call(mvh, device_route(cuda_stream), d_queries, q_offsets, B, params, d_out_ids, d_out_dist,
                         d_out_count);
}

int lgpu_debug_maxsim_gemm(const float *queries, uint32_t nqv, const float *values, const uint64_t *offsets,
                           uint64_t nrows, uint32_t dim, int device, float *out)
{
    return guarded([&] {
        LGPU_REQUIRE(offsets != nullptr && (nqv == 0 || (queries && out)), "null buffer");
        LGPU_REQUIRE(gemm_shape_supported(dim), "the tensor-core MaxSim score needs a dimension that is a multiple of 8");
        LGPU_REQUIRE(offsets[0] == 0, "row offsets must start at 0");
        for (uint64_t r = 0; r < nrows; r++) LGPU_REQUIRE(offsets[r + 1] >= offsets[r], "row offsets must not decrease");
        const uint64_t T = offsets[nrows];
        LGPU_REQUIRE(T < ((uint64_t)1 << 31) && (T == 0 || values), "bad stored vectors");
        require_device(device);
        if (nqv == 0 || nrows == 0) return;
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        DevBuf q, x, qh, xh, bad, cr, M;
        q.ensure((size_t)nqv * dim * 4); x.ensure(std::max<size_t>((size_t)T * dim * 4, 16));
        qh.ensure((size_t)nqv * dim * 2); xh.ensure(std::max<size_t>((size_t)T * dim * 2, 16));
        bad.ensure(std::max<size_t>(std::max<uint64_t>(T, nqv), 1) * 4); cr.ensure(std::max<size_t>(T, 1) * 4);
        M.ensure((size_t)nqv * nrows * 4);
        std::vector<uint32_t> hcr(T);
        for (uint64_t r = 0; r < nrows; r++)
            for (uint64_t j = offsets[r]; j < offsets[r + 1]; j++) hcr[j] = (uint32_t)r;
        LGPU_CUDA(cudaMemcpy(q.p, queries, (size_t)nqv * dim * 4, cudaMemcpyHostToDevice));
        if (T) {
            LGPU_CUDA(cudaMemcpy(x.p, values, (size_t)T * dim * 4, cudaMemcpyHostToDevice));
            LGPU_CUDA(cudaMemcpy(cr.p, hcr.data(), (size_t)T * 4, cudaMemcpyHostToDevice));
        }
        LGPU_CUDA(cudaMemset(M.p, 0, (size_t)nqv * nrows * 4));
        launch_mv_normalize_f16(q.as<float>(), nqv, dim, qh.p, bad.as<uint32_t>(), nullptr);
        launch_mv_normalize_f16(x.as<float>(), T, dim, xh.p, bad.as<uint32_t>(), nullptr);
        MaxSimOut mo{};
        mo.col_row = cr.as<uint32_t>(); mo.M = M.as<uint32_t>(); mo.ldM = nrows; mo.row_base = 0; mo.xdummy = x.as<float>();
        launch_maxsim_gemm(qh.p, xh.p, nqv, T, dim, mo, prop.multiProcessorCount, nullptr);
        std::vector<uint32_t> keys((size_t)nqv * nrows);
        LGPU_CUDA(cudaMemcpy(keys.data(), M.p, keys.size() * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < keys.size(); i++) out[i] = keys[i] ? key_f32(keys[i]) : NAN;
    });
}

int lgpu_debug_hamming_gemm(const uint8_t *queries, const uint8_t *vectors, uint32_t B, uint64_t N, uint32_t nbytes,
                            int device, uint32_t *out)
{
    return guarded([&] {
        LGPU_REQUIRE(nbytes > 0 && (uint64_t)nbytes * 8 <= ((uint64_t)1 << 24), "bytes per vector out of range");
        LGPU_REQUIRE((B == 0 || N == 0) || (queries && vectors && out), "null buffer");
        require_device(device);
        if (B == 0 || N == 0) return;
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        const uint32_t nbp = (nbytes + 31) & ~31u;
        DevBuf rq, rx, q, x, qp, xp, d;
        rq.ensure((size_t)B * nbytes); rx.ensure((size_t)N * nbytes);
        q.ensure((size_t)B * nbp); x.ensure((size_t)N * nbp); qp.ensure((size_t)B * 4); xp.ensure((size_t)N * 4);
        d.ensure((size_t)B * N * 4);
        LGPU_CUDA(cudaMemcpy(rq.p, queries, (size_t)B * nbytes, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(rx.p, vectors, (size_t)N * nbytes, cudaMemcpyHostToDevice));
        launch_ham_pack(rq.as<uint8_t>(), nbytes, nbytes, B, q.as<uint8_t>(), nbp, qp.as<uint32_t>(), nullptr);
        launch_ham_pack(rx.as<uint8_t>(), nbytes, nbytes, N, x.as<uint8_t>(), nbp, xp.as<uint32_t>(), nullptr);
        launch_ham_gemm(q.p, x.p, xp.as<uint32_t>(), qp.as<uint32_t>(), B, N, nbp, d.as<float>(), N, prop.multiProcessorCount,
                        nullptr);
        std::vector<float> h((size_t)B * N);
        LGPU_CUDA(cudaMemcpy(h.data(), d.p, (size_t)B * N * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < h.size(); i++) out[i] = (uint32_t)h[i];
    });
}

// ---- partition-sharded multi-GPU search (SURVEY.md 8e): one process per GPU, one ncclAllGather per batch ----
int lgpu_comm_unique_id(void *id_out, size_t id_bytes)
{
    return guarded([&] {
        LGPU_REQUIRE(id_out && id_bytes >= LGPU_COMM_ID_BYTES, "id buffer must hold LGPU_COMM_ID_BYTES bytes");
        static_assert(LGPU_COMM_ID_BYTES == sizeof(ncclUniqueId), "unique id size");
        ncclUniqueId id;
        LGPU_NCCL(nccl_api().GetUniqueId(&id));
        memcpy(id_out, &id, sizeof(id));
    });
}

int lgpu_comm_init(const void *unique_id, size_t id_bytes, int rank, int world, int device, lgpu_comm **out)
{
    lgpu_comm *c = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(unique_id && out && id_bytes >= LGPU_COMM_ID_BYTES, "null argument / short unique id");
        LGPU_REQUIRE(world >= 1 && rank >= 0 && rank < world, "rank must be in [0, world)");
        require_device(device);
        NcclApi &api = nccl_api();
        c = new lgpu_comm();
        c->device = device; c->rank = rank; c->world = world;
        ncclUniqueId id;
        memcpy(&id, unique_id, sizeof(id));
        LGPU_NCCL(api.CommInitRank(&c->comm, world, id, rank));
        for (auto &e : c->ev) LGPU_CUDA(cudaEventCreate(&e));
        register_handle(c);
        *out = c;
    });
    if (rc != LGPU_OK && c) delete c;
    return rc;
}

void lgpu_comm_destroy(lgpu_comm *c) { close_handle(c); }

// local top-k on this rank's shard -> pack -> ONE all-gather of [B][k] 16-byte records -> merge, all on `st`
static void sharded_search_device(lgpu_index *ix, lgpu_comm *c, Workspace *ws, cudaStream_t st, const float *d_q,
                                  uint32_t B, const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist,
                                  uint32_t *d_cnt, const Deadline *deadline)
{
    LGPU_REQUIRE(c->device == ix->device, "communicator and index live on different devices");
    LGPU_REQUIRE(sp.refine_factor == 0, "refine_factor is not supported on the sharded path (raw vectors are not sharded)");
    std::lock_guard<std::mutex> g(c->mu);
    const size_t n = (size_t)B * sp.k;
    c->l_ids.ensure(n * 8); c->l_dist.ensure(n * 4); c->l_cnt.ensure((size_t)B * 4);
    c->send.ensure(n * sizeof(TopkRecord)); c->recv.ensure(n * sizeof(TopkRecord) * c->world);
    const bool prof = profiling_enabled();
    ivf_search_device(ix, ws, st, d_q, B, sp, c->l_ids.as<uint64_t>(), c->l_dist.as<float>(), c->l_cnt.as<uint32_t>(),
                      RowFilter(), deadline);
    launch_pack_records(c->l_ids.as<uint64_t>(), c->l_dist.as<float>(), n, c->send.as<TopkRecord>(), st);
    if (prof) cudaEventRecord(c->ev[0], st);
    LGPU_NCCL(nccl_api().AllGather(c->send.p, c->recv.p, n * sizeof(TopkRecord), ncclUint8, c->comm, st));
    if (prof) cudaEventRecord(c->ev[1], st);
    // rank r's list of query q at r * B * k + q * k
    SelectArgs sb = select_cands(nullptr, nullptr, sp.k, B, sp.k, {d_ids, d_dist, d_cnt});
    sb.cand_rec = c->recv.as<TopkRecord>(); sb.ncols = (uint64_t)c->world * sp.k; sb.outer_stride = (uint64_t)B * sp.k;
    launch_select(sb, st);
    if (prof) {
        cudaEventRecord(c->ev[2], st);
        LGPU_CUDA(cudaStreamSynchronize(st));
        c->last_ms[0] = g_stage_ms[6];
        cudaEventElapsedTime(&c->last_ms[1], c->ev[0], c->ev[1]);
        cudaEventElapsedTime(&c->last_ms[2], c->ev[1], c->ev[2]);
    }
}

int lgpu_search_sharded(lgpu_index *ixh, lgpu_comm *ch, const float *queries, uint32_t B,
                        const lgpu_search_params *params, uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return guarded([&] {
        HandleRef<lgpu_index> ix(ixh, "index");
        HandleRef<lgpu_comm> c(ch, "communicator");
        LGPU_REQUIRE(!ix->is_sq && !ix->is_rq && !ix->is_pq4, "sharded search serves 8-bit IVF_PQ indexes only");
        check_ivf_call(ix.h, queries, B, params, out_ids, out_dist, out_count);
        if (B == 0) return;
        require_device(ix->device);
        host_call(ix->pool, queries, (size_t)B * ix->dim, B, params->k, out_ids, out_dist, out_count, nullptr,
                  params->timeout_ms,
                  [&](Workspace *ws, cudaStream_t st, const float *dq, uint64_t *di, float *dd, uint32_t *dc,
                      const Deadline &dl) { sharded_search_device(ix.h, c.h, ws, st, dq, B, *params, di, dd, dc, &dl); });
    });
}

int lgpu_search_sharded_device(lgpu_index *ixh, lgpu_comm *ch, const float *d_queries, uint32_t B,
                               const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                               uint32_t *d_out_count, void *cuda_stream)
{
    return guarded([&] {
        HandleRef<lgpu_index> ix(ixh, "index");
        HandleRef<lgpu_comm> c(ch, "communicator");
        LGPU_REQUIRE(!ix->is_sq && !ix->is_rq && !ix->is_pq4, "sharded search serves 8-bit IVF_PQ indexes only");
        check_ivf_call(ix.h, d_queries, B, params, d_out_ids, d_out_dist, d_out_count);
        if (B == 0) return;
        require_device(ix->device);
        WsLease lease(ix->pool, (cudaStream_t)cuda_stream, true);
        sharded_search_device(ix.h, c.h, lease.ws, lease.st, d_queries, B, *params, d_out_ids, d_out_dist, d_out_count,
                              nullptr);
    });
}

int lgpu_comm_last_stage_ms(lgpu_comm *ch, float *times)
{
    return guarded([&] {
        LGPU_REQUIRE(times, "null argument");
        HandleRef<lgpu_comm> c(ch, "communicator");
        memcpy(times, c->last_ms, sizeof(c->last_ms));
    });
}

int lgpu_debug_coarse(lgpu_index *ixh, const float *queries, uint32_t B, uint32_t nprobes, uint32_t *out_parts,
                      float *out_dists)
{
    return guarded([&] {
        LGPU_REQUIRE(queries && out_parts && out_dists && B > 0 && nprobes > 0, "bad argument");
        HandleRef<lgpu_index> ix(ixh, "index");
        require_device(ix->device);
        nprobes = std::min(nprobes, ix->nlist);
        WsLease lease(ix->pool, nullptr, false);
        Workspace *ws = lease.ws; cudaStream_t st = lease.st;
        ws->q.ensure((size_t)B * ix->dim * 4);
        LGPU_CUDA(cudaMemcpyAsync(ws->q.p, queries, (size_t)B * ix->dim * 4, cudaMemcpyHostToDevice, st));
        lgpu_search_params sp{};
        sp.k = 1; sp.nprobes = nprobes;
        ScanModes modes = scan_modes();
        modes.exact = true;                               // (no filter scan: no query tables)
        IvfPlan p = ivf_plan(ix.h, B, nprobes, sp, false, false, modes);
        p.coarse = Coarse::exact;                         // the exact kernels' probes and distances
        ivf_coarse(ix.h, ws, p, ivf_queries(ix.h, ws, st, ws->q.as<float>(), B), st, st, StageMarks{ws, false});
        std::vector<uint64_t> tmp((size_t)B * nprobes);
        LGPU_CUDA(cudaMemcpyAsync(tmp.data(), ws->probes.p, tmp.size() * 8, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaMemcpyAsync(out_dists, ws->probe_dist.p, tmp.size() * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
        for (size_t i = 0; i < tmp.size(); i++) out_parts[i] = (uint32_t)tmp[i];
    });
}

int lgpu_debug_gemm(const float *Q, const float *X, uint32_t B, uint64_t N, uint32_t d, int device, float *out)
{
    return guarded([&] {
        LGPU_REQUIRE(Q && X && out && B > 0 && N > 0, "bad argument");
        LGPU_REQUIRE(gemm_shape_supported(d), "dimension must be a multiple of 8");
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        DevBuf q, x, qb, xb, xn2, o;
        const uint64_t ld = (N + 3) & ~3ull;
        q.ensure((size_t)B * d * 4); x.ensure((size_t)N * d * 4); qb.ensure((size_t)B * d * 2); xb.ensure((size_t)N * d * 2);
        xn2.ensure((size_t)N * 4); o.ensure((size_t)B * ld * 4);
        LGPU_CUDA(cudaMemcpy(q.p, Q, (size_t)B * d * 4, cudaMemcpyHostToDevice));
        LGPU_CUDA(cudaMemcpy(x.p, X, (size_t)N * d * 4, cudaMemcpyHostToDevice));
        launch_to_bf16(q.as<float>(), B, d, qb.p, nullptr, nullptr);
        launch_to_bf16(x.as<float>(), N, d, xb.p, xn2.as<float>(), nullptr);
        launch_gemm_dist(qb.p, xb.p, xn2.as<float>(), B, N, d, o.as<float>(), ld, prop.multiProcessorCount, nullptr);
        LGPU_CUDA(cudaDeviceSynchronize());
        LGPU_CUDA(cudaMemcpy2D(out, (size_t)N * 4, o.p, (size_t)ld * 4, (size_t)N * 4, B, cudaMemcpyDeviceToHost));
    });
}

int lgpu_debug_partition_distances(lgpu_index *ixh, const float *query, uint32_t part, float *out)
{
    return guarded([&] {
        LGPU_REQUIRE(query && out, "null argument");
        HandleRef<lgpu_index> ix(ixh, "index");
        LGPU_REQUIRE(!ix->is_sq && !ix->is_rq, "lgpu_debug_partition_distances serves IVF_PQ indexes only");
        LGPU_REQUIRE(part < ix->nlist, "partition out of range");
        require_device(ix->device);
        WsLease lease(ix->pool, nullptr, false);
        Workspace *ws = lease.ws; cudaStream_t st = lease.st;
        ws->q.ensure((size_t)ix->dim * 4);
        LGPU_CUDA(cudaMemcpyAsync(ws->q.p, query, (size_t)ix->dim * 4, cudaMemcpyHostToDevice, st));
        // the one probe slot is `part`, regrouped for the exact scan (scan2.cu, or pq4_scan.cu for 4-bit codes)
        lgpu_search_params sp{};
        sp.k = 1; sp.nprobes = 1;
        ScanModes modes = scan_modes();
        modes.exact = true; modes.small_slots = 0;
        const IvfPlan p = ivf_plan(ix.h, 1, 1, sp, false, false, modes);
        const float *qs = ivf_queries(ix.h, ws, st, ws->q.as<float>(), 1);
        const uint64_t forced = part;
        ws->probes.ensure(8);
        LGPU_CUDA(cudaMemcpyAsync(ws->probes.p, &forced, 8, cudaMemcpyHostToDevice, st));
        if (p.scan == IvfScan::pq4) pq4_tables(ix.h, ws, p, qs, st);
        const GroupArgs ga = ivf_regroup(ix.h, ws, p, nullptr, st);
        if (p.scan == IvfScan::pq4) launch_pq4_scan(pq4_args(ix.h, ws, ga), 2 * ix->num_sms, st);
        else launch_scan2(scan_args(ix.h, ws, qs, ga), ix->dsub, ix->num_sms, st);
        uint32_t n = ix->h_part_n[part];
        if (n) LGPU_CUDA(cudaMemcpyAsync(out, ws->dist_out.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
    });
}

int lgpu_debug_filter_bounds(lgpu_index *ixh, const float *queries, uint32_t B, uint32_t nprobes, uint64_t ld,
                             uint32_t *out_parts, float *out_L, float *out_W, float *out_E, uint32_t *out_bad)
{
    return guarded([&] {
        LGPU_REQUIRE(queries && out_parts && out_L && out_W && out_E && out_bad && B > 0 && nprobes > 0, "bad argument");
        HandleRef<lgpu_index> ix(ixh, "index");
        LGPU_REQUIRE(!ix->is_sq && !ix->is_rq && !ix->is_pq4, "lgpu_debug_filter_bounds serves 8-bit IVF_PQ indexes only");
        require_device(ix->device);
        nprobes = std::min(nprobes, ix->nlist);
        LGPU_REQUIRE(ivf_sub_batch_size(ix.h, B, nprobes) == B, "batch too large for one filter-scan launch");
        WsLease lease(ix->pool, nullptr, false);
        Workspace *ws = lease.ws; cudaStream_t st = lease.st;
        ws->q.ensure((size_t)B * ix->dim * 4);
        LGPU_CUDA(cudaMemcpyAsync(ws->q.p, queries, (size_t)B * ix->dim * 4, cudaMemcpyHostToDevice, st));
        lgpu_search_params sp{};
        sp.k = 10; sp.nprobes = nprobes;
        ScanModes modes = scan_modes();
        modes.small_slots = 0;
        const IvfPlan p = ivf_plan(ix.h, B, nprobes, sp, false, false, modes);
        LGPU_REQUIRE(p.filter(), "this index or configuration does not use the filter scan");
        // the search's front, then the dense mode's scan: one lower bound L per row
        const float *qs = ivf_queries(ix.h, ws, st, ws->q.as<float>(), B);
        const cudaStream_t cs = fork_front(ix.h, ws, st, B);
        ivf_coarse(ix.h, ws, p, qs, cs, st, StageMarks{ws, false});
        const GroupArgs ga = ivf_regroup(ix.h, ws, p, nullptr, cs);
        LGPU_CUDA(cudaEventRecord(ws->ev_join, ws->front));
        ScanArgs sc = scan_args(ix.h, ws, qs, ga);
        filter_terms(ix.h, ws, p, qs, sc, st);
        launch_scan3(sc, ix->num_sms, st);
        // W, E of every query (the band the consumers use) and the scan's own L, per probe slot
        const bool dot = ix->metric == LGPU_DOT;
        const uint32_t slots = p.slots, nlist = ix->nlist;
        const size_t nL = (size_t)B * ix->pad_prefix[p.np_eff];
        ws->s_exact.ensure((size_t)B * 8);
        float *dW = ws->s_exact.as<float>(), *dE = dW + B;
        launch_scan_band(ws->qt_step.as<float>(), ws->sbound.as<float>(), dot ? nullptr : ws->amax.as<float>(),
                         dot ? nullptr : ix->rmax_bits.as<int>(), ws->qn2.as<float>(), ix->cb2, ix->m, dot, B, dW, dE, st);
        std::vector<uint64_t> probes(slots), seg(slots);
        std::vector<float> L(nL);
        LGPU_CUDA(cudaMemcpyAsync(probes.data(), ws->probes.p, (size_t)slots * 8, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaMemcpyAsync(seg.data(), ga.seg_off, (size_t)slots * 8, cudaMemcpyDeviceToHost, st));
        if (nL) LGPU_CUDA(cudaMemcpyAsync(L.data(), ws->dist_out.p, nL * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaMemcpyAsync(out_W, dW, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaMemcpyAsync(out_E, dE, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaMemcpyAsync(out_bad, ws->qt_bad.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
        for (uint32_t sl = 0; sl < slots; sl++) {
            const uint64_t pr = probes[sl];
            out_parts[sl] = pr < nlist ? (uint32_t)pr : UINT32_MAX;
            const uint64_t n = pr < nlist ? std::min<uint64_t>(ix->h_part_n[pr], ld) : 0;
            if (n) memcpy(out_L + (size_t)sl * ld, L.data() + seg[sl], n * 4);
        }
    });
}

// ---- index build passes (build.cu): host buffers in, host buffers out, chunked over rows ----
int lgpu_ivf_assign(const float *centroids, uint32_t nlist, uint32_t dim, int metric, const float *vectors,
                    uint64_t n, int device, uint32_t *out_parts)
{
    return guarded([&] {
        LGPU_REQUIRE(centroids && nlist > 0 && dim > 0, "null centroids / empty shape");
        LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE || metric == LGPU_DOT, "unknown distance type");
        LGPU_REQUIRE(n == 0 || (vectors && out_parts), "null vectors / output");
        if (n == 0) return;
        require_device(device);
        cudaStream_t st = nullptr;
        const uint64_t ld = (nlist + 3ull) & ~3ull;
        const uint64_t CH = std::max<uint64_t>(256, std::min<uint64_t>(65536, ((uint64_t)1 << 28) / (ld * 4)));
        DevBuf cent, x, xn, D, ids, dist, cnt;
        cent.ensure((size_t)nlist * dim * 4);
        LGPU_CUDA(cudaMemcpyAsync(cent.p, centroids, (size_t)nlist * dim * 4, cudaMemcpyHostToDevice, st));
        x.ensure((size_t)CH * dim * 4); D.ensure((size_t)CH * ld * 4);
        ids.ensure((size_t)CH * 8); dist.ensure((size_t)CH * 4); cnt.ensure((size_t)CH * 4);
        if (metric == LGPU_COSINE) xn.ensure((size_t)CH * dim * 4);
        std::vector<uint64_t> h_ids(CH);
        for (uint64_t r0 = 0; r0 < n; r0 += CH) {
            const uint32_t b = (uint32_t)std::min<uint64_t>(CH, n - r0);
            LGPU_CUDA(cudaMemcpyAsync(x.p, vectors + r0 * dim, (size_t)b * dim * 4, cudaMemcpyHostToDevice, st));
            const float *q = x.as<float>();
            if (metric == LGPU_COSINE) { launch_normalize(q, b, dim, xn.as<float>(), st); q = xn.as<float>(); }
            // the search path's own coarse step (find_partitions with nprobes = 1)
            launch_dist_matrix(q, cent.as<float>(), b, nlist, dim, metric == LGPU_DOT ? 1 : 0, nullptr, nullptr,
                               D.as<float>(), ld, st);
            launch_select(select_rows(D.as<float>(), nlist, ld, b, 1, {ids.as<uint64_t>(), dist.as<float>(),
                                      cnt.as<uint32_t>()}), st);
            LGPU_CUDA(cudaMemcpyAsync(h_ids.data(), ids.p, (size_t)b * 8, cudaMemcpyDeviceToHost, st));
            LGPU_CUDA(cudaStreamSynchronize(st));
            for (uint32_t i = 0; i < b; i++) {
                LGPU_REQUIRE(h_ids[i] < nlist, "a vector has no finite centroid distance (NaN input?)");
                out_parts[r0 + i] = (uint32_t)h_ids[i];
            }
        }
    });
}

// nearest centre of every row (device buffers): the search's coarse step with nprobes = 1 -- tensor-core GEMM scores +
// coarse_finish_kernel (exact re-score, lance arithmetic) where the shape allows it, the exact kernels otherwise
static void assign_nearest(const float *d_x, uint64_t n, uint32_t dim, const float *d_cent, uint32_t k, int num_sms,
                           uint64_t *d_ids, float *d_dist, cudaStream_t st)
{
    const uint64_t ld = (k + 3ull) & ~3ull;
    const uint64_t CH = std::max<uint64_t>(256, std::min<uint64_t>(65536, ((uint64_t)1 << 28) / (ld * 4)));
    DevBuf D, cnt, flags, gate, xb, xn2, xerr, cb, cn2;
    D.ensure((size_t)CH * ld * 4); cnt.ensure((size_t)CH * 4);
    const bool tc = gemm_shape_supported(dim) && k >= 256 && tc_enabled();
    float cmax = 0.f, cerr = 0.f;
    if (tc) {
        flags.ensure((size_t)CH * 4); gate.ensure(16);
        xb.ensure((size_t)CH * dim * 2); xn2.ensure((size_t)CH * 4); xerr.ensure((size_t)CH * 4);
        prepare_tc_operand(d_cent, k, dim, cb, cn2, cmax, cerr, st);
    }
    for (uint64_t r0 = 0; r0 < n; r0 += CH) {
        const uint32_t b = (uint32_t)std::min<uint64_t>(CH, n - r0);
        const float *q = d_x + r0 * dim;
        SelectArgs sa = select_rows(D.as<float>(), k, ld, b, 1, {d_ids + r0, d_dist + r0, cnt.as<uint32_t>()});
        if (tc) {
            launch_to_bf16(q, b, dim, xb.p, xn2.as<float>(), st, xerr.as<float>());
            launch_gemm_dist(xb.p, cb.p, cn2.as<float>(), b, k, dim, D.as<float>(), ld, num_sms, st);
            launch_coarse_finish(D.as<float>(), ld, b, k, q, d_cent, xn2.as<float>(), xerr.as<float>(), cmax, cerr, dim, 1,
                                 d_ids + r0, d_dist + r0,
                                 cnt.as<uint32_t>(), flags.as<uint32_t>(), gate.as<uint32_t>(), st);
            launch_dist_matrix(q, d_cent, b, k, dim, 0, nullptr, nullptr, D.as<float>(), ld, st, flags.as<uint32_t>(),
                               gate.as<uint32_t>());
            sa.only = flags.as<uint32_t>(); sa.gate = gate.as<uint32_t>();
            launch_select(sa, st);
        } else {
            launch_dist_matrix(q, d_cent, b, k, dim, 0, nullptr, nullptr, D.as<float>(), ld, st);
            launch_select(sa, st);
        }
    }
    LGPU_CUDA(cudaStreamSynchronize(st));                            // the scratch buffers die with this scope
}

int lgpu_kmeans_train(const float *x, uint64_t n, uint32_t dim, float *centroids, uint32_t k, uint32_t iters, int device,
                      double *inertia_out)
{
    return guarded([&] {
        LGPU_REQUIRE(x && centroids && n > 0 && dim > 0 && k > 0, "null argument / empty shape");
        LGPU_REQUIRE(n < (1ull << 32), "too many training rows (sample them: sample_rate * num_partitions)");
        require_device(device);
        cudaDeviceProp prop;
        LGPU_CUDA(cudaGetDeviceProperties(&prop, device));
        cudaStream_t st = nullptr;
        DevBuf dx, dc, ids, dist, counts, offsets, cursor, rows, inert;
        dx.ensure((size_t)n * dim * 4); dc.ensure((size_t)k * dim * 4);
        ids.ensure((size_t)n * 8); dist.ensure((size_t)n * 4);
        counts.ensure((size_t)k * 4); offsets.ensure((size_t)(k + 1) * 4); cursor.ensure((size_t)k * 4);
        rows.ensure((size_t)n * 4); inert.ensure(16);
        LGPU_CUDA(cudaMemcpyAsync(dx.p, x, (size_t)n * dim * 4, cudaMemcpyHostToDevice, st));
        LGPU_CUDA(cudaMemcpyAsync(dc.p, centroids, (size_t)k * dim * 4, cudaMemcpyHostToDevice, st));
        for (uint32_t it = 0; it < std::max<uint32_t>(iters, 1); it++) {
            assign_nearest(dx.as<float>(), n, dim, dc.as<float>(), k, prop.multiProcessorCount, ids.as<uint64_t>(),
                           dist.as<float>(), st);
            launch_kmeans_update(ids.as<uint64_t>(), dx.as<float>(), n, dim, k, counts.as<uint32_t>(), offsets.as<uint32_t>(),
                                 cursor.as<uint32_t>(), rows.as<uint32_t>(), dc.as<float>(), st);
        }
        if (inertia_out) {                                           // of the trained centres
            assign_nearest(dx.as<float>(), n, dim, dc.as<float>(), k, prop.multiProcessorCount, ids.as<uint64_t>(),
                           dist.as<float>(), st);
            launch_kmeans_inertia(dist.as<float>(), n, inert.as<double>(), st);
            LGPU_CUDA(cudaMemcpyAsync(inertia_out, inert.p, 8, cudaMemcpyDeviceToHost, st));
        }
        LGPU_CUDA(cudaMemcpyAsync(centroids, dc.p, (size_t)k * dim * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
    });
}

int lgpu_pq_train(const float *x, uint64_t n, uint32_t dim, uint32_t m, float *codebook, uint32_t iters, int device)
{
    return guarded([&] {
        LGPU_REQUIRE(x && codebook && n > 0 && dim > 0 && m > 0, "null argument / empty shape");
        LGPU_REQUIRE(dim % m == 0 && scan_dsub_supported(dim / m),
                     "unsupported PQ sub-vector length (dim/num_sub_vectors must be 1,2,4,8,16 or 32)");
        require_device(device);
        cudaStream_t st = nullptr;
        const uint32_t dsub = dim / m;
        DevBuf dx, cb, zero, parts, codes, sums, counts;
        dx.ensure((size_t)n * dim * 4); cb.ensure((size_t)m * 256 * dsub * 4); zero.ensure((size_t)dim * 4);
        parts.ensure((size_t)n * 4); codes.ensure((size_t)n * m); sums.ensure((size_t)m * 256 * dsub * 8);
        counts.ensure((size_t)m * 256 * 4);
        LGPU_CUDA(cudaMemcpyAsync(dx.p, x, (size_t)n * dim * 4, cudaMemcpyHostToDevice, st));
        LGPU_CUDA(cudaMemcpyAsync(cb.p, codebook, (size_t)m * 256 * dsub * 4, cudaMemcpyHostToDevice, st));
        LGPU_CUDA(cudaMemsetAsync(zero.p, 0, (size_t)dim * 4, st));          // one all-zero "centroid": residual = row
        LGPU_CUDA(cudaMemsetAsync(parts.p, 0, (size_t)n * 4, st));
        for (uint32_t it = 0; it < std::max<uint32_t>(iters, 1); it++) {
            launch_pq_encode(dx.as<float>(), parts.as<uint32_t>(), zero.as<float>(), cb.as<float>(), n, dim, m, LGPU_L2,
                             codes.as<unsigned char>(), st);
            launch_pq_update(dx.as<float>(), codes.as<unsigned char>(), n, dim, m, sums.as<double>(), counts.as<uint32_t>(),
                             cb.as<float>(), st);
        }
        LGPU_CUDA(cudaMemcpyAsync(codebook, cb.p, (size_t)m * 256 * dsub * 4, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
    });
}

int lgpu_pq_encode(const float *centroids, const float *codebook, uint32_t nlist, uint32_t dim, uint32_t m,
                   int metric, const float *vectors, const uint32_t *parts, uint64_t n, int device,
                   unsigned char *out_codes)
{
    return guarded([&] {
        LGPU_REQUIRE(centroids && codebook && nlist > 0 && dim > 0 && m > 0, "null index array / empty shape");
        LGPU_REQUIRE(dim % m == 0 && scan_dsub_supported(dim / m),
                     "unsupported PQ sub-vector length (dim/num_sub_vectors must be 1,2,4,8,16 or 32)");
        LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE || metric == LGPU_DOT, "unknown distance type");
        LGPU_REQUIRE(n == 0 || (vectors && parts && out_codes), "null vectors / partitions / output");
        if (n == 0) return;
        for (uint64_t r = 0; r < n; r++) LGPU_REQUIRE(parts[r] < nlist, "partition id out of range");
        require_device(device);
        cudaStream_t st = nullptr;
        const uint64_t CH = 65536;
        DevBuf cent, cb, x, xn, p, codes;
        cent.ensure((size_t)nlist * dim * 4); cb.ensure((size_t)m * 256 * (dim / m) * 4);
        LGPU_CUDA(cudaMemcpyAsync(cent.p, centroids, (size_t)nlist * dim * 4, cudaMemcpyHostToDevice, st));
        LGPU_CUDA(cudaMemcpyAsync(cb.p, codebook, (size_t)m * 256 * (dim / m) * 4, cudaMemcpyHostToDevice, st));
        x.ensure((size_t)CH * dim * 4); p.ensure((size_t)CH * 4); codes.ensure((size_t)CH * m);
        if (metric == LGPU_COSINE) xn.ensure((size_t)CH * dim * 4);
        for (uint64_t r0 = 0; r0 < n; r0 += CH) {
            const uint32_t b = (uint32_t)std::min<uint64_t>(CH, n - r0);
            LGPU_CUDA(cudaMemcpyAsync(x.p, vectors + r0 * dim, (size_t)b * dim * 4, cudaMemcpyHostToDevice, st));
            LGPU_CUDA(cudaMemcpyAsync(p.p, parts + r0, (size_t)b * 4, cudaMemcpyHostToDevice, st));
            const float *q = x.as<float>();
            if (metric == LGPU_COSINE) { launch_normalize(q, b, dim, xn.as<float>(), st); q = xn.as<float>(); }
            launch_pq_encode(q, p.as<uint32_t>(), cent.as<float>(), cb.as<float>(), b, dim, m, metric,
                             codes.as<unsigned char>(), st);
            LGPU_CUDA(cudaMemcpyAsync(out_codes + r0 * m, codes.p, (size_t)b * m, cudaMemcpyDeviceToHost, st));
            LGPU_CUDA(cudaStreamSynchronize(st));
        }
    });
}

}  // extern "C"
