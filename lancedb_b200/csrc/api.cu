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
#include <functional>
#include <mutex>
#include <thread>
#include <type_traits>
#include <unordered_map>
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
static thread_local uint64_t g_streamed_bytes = 0;   // profiling: the host-resident codes the last IVF call copied
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
// bytes of the calling thread's current call held in a workspace outside its sub-batches: the AND of the call's bitmap
// with a handle's live rows (with_live), charged to LGPU_WS_BYTES once per call and released when the call ends
// (WsCharge).  The sub-batches share what is left, at least the 1 MiB floor.
static thread_local size_t g_ws_charged = 0;
struct WsCharge {
    ~WsCharge() { g_ws_charged = 0; }
};
static size_t workspace_budget()
{
    static size_t v = 0;
    constexpr size_t floor = (size_t)1 << 20;
    if (!v) {
        const char *e = getenv("LGPU_WS_BYTES");
        v = e ? (size_t)strtoull(e, nullptr, 10) : ((size_t)8 << 30);
        if (v < floor) v = floor;
    }
    return v > g_ws_charged + floor ? v - g_ws_charged : floor;
}

// bumped by every device (re)allocation in the process.  A captured CUDA graph bakes workspace pointers in, so a
// graph is only replayed while the epoch still equals the one recorded at capture (Workspace::graph_epoch): any
// entry point, on any thread, that grows a buffer invalidates every captured graph (they re-capture on next use).
static std::atomic<uint64_t> g_alloc_epoch{0};

struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    // exact: no headroom (per-row storage of a handle, whose growth goes through grow_keep)
    void ensure(size_t n, bool exact = false)
    {
        if (n <= bytes) return;
        g_alloc_epoch++;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        size_t want = exact ? n : n + n / 8;
        LGPU_CUDA(cudaMalloc(&p, want));
        bytes = want;
    }
    template <class T> T *as() { return reinterpret_cast<T *>(p); }
    void reset() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    ~DevBuf() { reset(); }
};

// pinned host memory mapped into the device's address space (cudaHostAllocMapped): `dev` is the alias kernels read
// over PCIe
struct PinnedBuf {
    void *p = nullptr, *dev = nullptr;
    size_t bytes = 0;
    void alloc(size_t n)
    {
        reset();
        LGPU_CUDA(cudaHostAlloc(&p, std::max<size_t>(n, 16), cudaHostAllocMapped));
        bytes = n;
        LGPU_CUDA(cudaHostGetDevicePointer(&dev, p, 0));
    }
    void reset() { if (p) cudaFreeHost(p); p = dev = nullptr; bytes = 0; }
    ~PinnedBuf() { reset(); }
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

struct Workspace;

// Rows streamed from pinned host memory through HBM (RowStore::walk).  Between open and close, chunk s of `steps` is
// copied into buf[s & 1] by copier(s, buf, front) on the workspace's side stream (`front`, forked from the call's
// stream and joined back to it), chunk s + 1 while chunk s is used on the call's stream: take(s) hands over chunk s
// once the copy of chunk s + 1 is issued, release(s) marks every use of it enqueued.  copied[i]: buf[i] holds its chunk
// (side stream); freed[i]: the uses of its chunk are enqueued (call's stream), so the copy two steps later may
// overwrite it.  timeout_ms is checked between chunks.
struct Staging {
    using Copier = std::function<void(uint64_t, void *, cudaStream_t)>;        // chunk s into a buffer, on a stream
    DevBuf buf[2];
    cudaEvent_t copied[2] = {}, freed[2] = {};
    Staging()
    {
        for (int i = 0; i < 2; i++) {
            LGPU_CUDA(cudaEventCreateWithFlags(&copied[i], cudaEventDisableTiming));
            LGPU_CUDA(cudaEventCreateWithFlags(&freed[i], cudaEventDisableTiming));
        }
    }
    ~Staging()
    {
        for (int i = 0; i < 2; i++) {
            if (copied[i]) cudaEventDestroy(copied[i]);
            if (freed[i]) cudaEventDestroy(freed[i]);
        }
    }
    void open(Workspace *ws, cudaStream_t st, uint64_t steps, const Deadline *deadline, Copier copier);
    void *take(uint64_t s);
    void release(uint64_t s) { LGPU_CUDA(cudaEventRecord(freed[s & 1], st)); }
    void close();
    void copy(uint64_t s);
    // the open run
    Workspace *ws = nullptr;
    cudaStream_t st = nullptr;
    uint64_t steps = 0;
    const Deadline *deadline = nullptr;
    Copier copier;
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
    DevBuf hn_ids, hn_dist, hn_pos, hn_ctr;   // IVF_HNSW_SQ search: each probe slot's R [slots][kk], the slot counter
    DevBuf rq_q, rq_planes, rq_slots;   // IVF_RQ search: rotated queries [B][dim], per-slot bit-planes and grids
    DevBuf pq4_tab, pq4_slots;          // 4-bit IVF_PQ search: per-slot u8 tables [slots][m][16] and quantisers
    DevBuf sel_large;                   // the large select's scratch (k > SELECT_KMAX, select_large.cu)
    DevBuf u_ids, u_dist, u_cnt;        // union search: the index's and the tail's top-k, [2][B][k] and [2][B]
    DevBuf live_and;                    // a filtered call on a handle with deleted rows: its bitmap AND the live rows
    Staging stage;                      // a handle whose rows are in pinned host memory: the rows staged through HBM
    // a flat handle whose rows are in pinned host memory (flat_search): the staged chunk's tensor-core
    // operand, |x|^2 and |x|, and the running top-k, [2 buffers][2 lists][P][k] / [..][P]
    DevBuf chunk_xb, chunk_n2, chunk_ysqrt, run_ids, run_dist, run_cnt;
    DevBuf chunk_pop;                   // ... of a binary handle (binary_search_device): popc of each staged row
    DevBuf code_ctr;                    // an IVF index with codes on the host: each chunk's tile counter, the bytes copied
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

void Staging::open(Workspace *w, cudaStream_t s, uint64_t n, const Deadline *dl, Copier cp)
{
    ws = w; st = s; steps = n; deadline = dl; copier = std::move(cp);
    LGPU_CUDA(cudaEventRecord(ws->ev_fork, st));
    LGPU_CUDA(cudaStreamWaitEvent(ws->front, ws->ev_fork, 0));
    ws->front_open = true;
    if (steps) copy(0);
}

// chunk s into buf[s & 1], once the uses of the chunk it held two steps earlier are enqueued
void Staging::copy(uint64_t s)
{
    const int i = (int)(s & 1);
    if (s >= 2) LGPU_CUDA(cudaStreamWaitEvent(ws->front, freed[i], 0));
    copier(s, buf[i].p, ws->front);
    LGPU_CUDA(cudaEventRecord(copied[i], ws->front));
}

void *Staging::take(uint64_t s)
{
    if (deadline && s > 0) deadline->wait(st, ws->ev[7]);
    if (s + 1 < steps) copy(s + 1);
    LGPU_CUDA(cudaStreamWaitEvent(st, copied[s & 1], 0));
    return buf[s & 1].p;
}

void Staging::close()
{
    LGPU_CUDA(cudaEventRecord(ws->ev_join, ws->front));
    LGPU_CUDA(cudaStreamWaitEvent(st, ws->ev_join, 0));
    ws->front_open = false;
}

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

// The rows of a handle that were not deleted (lgpu_*_delete): a device bitmap over row ids [0, id_bound), id_bound the
// largest row id + 1, with the bit of every row id the handle holds set until that id is deleted (rowmask.cu).  The
// first delete builds it; a handle never deleted from holds none (active false) and searches as before.
struct RowLive {
    DevBuf bits;
    uint64_t id_bound = 0;
    bool active = false;
};

// `b` holds `used` bytes; make room for `need` (an append): capacity at least doubles, the contents move by a
// device-to-device copy.  The caller has drained the device, so nothing still reads the old buffer when it is released.
static void grow_keep(DevBuf &b, size_t used, size_t need)
{
    if (need <= b.bytes) return;
    DevBuf nb;
    nb.ensure(std::max(need, 2 * b.bytes));                    // bumps g_alloc_epoch
    if (used) LGPU_CUDA(cudaMemcpy(nb.p, b.p, used, cudaMemcpyDeviceToDevice));
    std::swap(b.p, nb.p);
    std::swap(b.bytes, nb.bytes);
}

// the most rows of a host handle one staging buffer holds, in bytes: large enough that the copy engine runs at the
// PCIe rate and a chunk's fixed scoring cost is small, small enough that the unoverlapped first copy is short
constexpr size_t FLAT_STAGE_BYTES = (size_t)128 << 20;

// One chunk of a RowStore walk or visit: step s, rows [r0, r1), X the rows as a kernel reads them.  resident: X is the
// store's own HBM (the handle's per-row terms apply as they are); else an HBM copy (the chunk's terms are built for it).
struct RowChunk {
    uint64_t s, r0, r1;
    const void *X;
    bool resident;
};

// Stored rows, [n][row bytes] -- a flat, binary or multivector handle's rows, an IVF index's codes or raw vectors: in
// HBM, or -- when the open found they do not fit there (rows_fit_hbm) -- in pinned host memory mapped into the device's
// address space, which searches stream through HBM or read over PCIe.  The placement is fixed at open.
struct RowStore {
    bool on_host = false;
    DevBuf hbm;
    PinnedBuf host;
    // `bytes` of rows, allocated exactly (HBM: at least 16)
    void open(bool in_host, size_t bytes)
    {
        on_host = in_host;
        if (on_host) host.alloc(bytes);
        else hbm.ensure(std::max<size_t>(bytes, 16), true);
    }
    // the rows as host code addresses them: an HBM pointer, or the pinned host memory
    char *data() const { return static_cast<char *>(on_host ? host.p : hbm.p); }
    // the rows as a kernel reads them: an HBM pointer, or the mapped alias of the pinned memory
    const void *dev() const { return on_host ? host.dev : hbm.p; }
    // bytes from a host pointer into the rows at byte `at`
    void fill(size_t at, const void *src, size_t bytes)
    {
        if (!bytes) return;
        if (on_host) memcpy(data() + at, src, bytes);
        else LGPU_CUDA(cudaMemcpy(data() + at, src, bytes, cudaMemcpyHostToDevice));
    }
    // room for `need` bytes of rows, `used` of them kept (an append)
    void grow(size_t used, size_t need)
    {
        if (!on_host) return grow_keep(hbm, used, need);
        if (need <= host.bytes) return;
        PinnedBuf nb;
        nb.alloc(std::max(need, 2 * host.bytes));
        if (used) memcpy(nb.p, host.p, used);
        std::swap(host.p, nb.p);
        std::swap(host.dev, nb.dev);
        std::swap(host.bytes, nb.bytes);
    }
    uint64_t device_bytes() const { return hbm.bytes; }
    uint64_t host_bytes() const { return host.bytes; }
    // the two staging buffers of a host store's walk, `bytes` each
    void reserve_stage(Workspace *ws, size_t bytes) const
    {
        if (on_host) for (auto &b : ws->stage.buf) b.ensure(bytes);
    }
    // use(RowChunk) for `passes` passes over the chunks cut[c]..cut[c + 1] (row r at byte at(r)), then after(s) once
    // step s's staging buffer is released.  An HBM store is one resident chunk [cut.front(), cut.back()) per pass, the
    // deadline checked between passes; a host store streams each chunk through Workspace::stage, which checks it
    // between steps.  Chunk s is copied into its staging buffer by `copier` when the caller gives one, else by a
    // cudaMemcpyAsync of its pinned rows.
    template <class At, class Use, class After>
    void walk(Workspace *ws, cudaStream_t st, const std::vector<uint64_t> &cut, uint64_t passes, At &&at,
              const Deadline *deadline, Use &&use, After &&after, Staging::Copier copier = nullptr) const
    {
        const uint64_t nc = cut.size() - 1;
        if (!on_host) {
            for (uint64_t s = 0; s < passes; s++) {
                if (deadline && s > 0) deadline->wait(st, ws->ev[7]);
                use(RowChunk{s, cut.front(), cut.back(), hbm.p, true});
                after(s);
            }
            return;
        }
        if (!copier)
            copier = [&](uint64_t s, void *buf, cudaStream_t fs) {
                const uint64_t c = s % nc, bytes = at(cut[c + 1]) - at(cut[c]);
                if (bytes)
                    LGPU_CUDA(cudaMemcpyAsync(buf, static_cast<const char *>(host.p) + at(cut[c]), bytes,
                                              cudaMemcpyHostToDevice, fs));
            };
        ws->stage.open(ws, st, passes * nc, deadline, std::move(copier));
        for (uint64_t s = 0; s < passes * nc; s++) {
            const uint64_t c = s % nc;
            use(RowChunk{s, cut[c], cut[c + 1], ws->stage.take(s), false});
            ws->stage.release(s);
            after(s);
        }
        ws->stage.close();
    }
    template <class At, class Use>
    void walk(Workspace *ws, cudaStream_t st, const std::vector<uint64_t> &cut, At &&at, const Deadline *deadline,
              Use &&use, Staging::Copier copier = nullptr) const
    {
        walk(ws, st, cut, 1, at, deadline, use, [](uint64_t) {}, std::move(copier));
    }
    // f(RowChunk) over rows [r0, r1) of `row_bytes` each, at open or append, synchronously on the legacy stream: an HBM
    // store once, X its resident row r0; a host store in chunks of at most FLAT_STAGE_BYTES, each copied into one
    // temporary HBM buffer.  Nothing runs for no rows.
    template <class F> void visit(uint64_t r0, uint64_t r1, size_t row_bytes, F &&f) const
    {
        if (r1 <= r0) return;
        if (!on_host) return f(RowChunk{0, r0, r1, static_cast<const char *>(hbm.p) + r0 * row_bytes, true});
        const uint64_t C = std::max<uint64_t>(1, std::min<uint64_t>(r1 - r0, FLAT_STAGE_BYTES / row_bytes));
        DevBuf x;
        x.ensure(C * row_bytes);
        for (uint64_t r = r0, s = 0; r < r1; r += C, s++) {
            const uint64_t m = std::min(C, r1 - r);
            LGPU_CUDA(cudaMemcpy(x.p, data() + r * row_bytes, m * row_bytes, cudaMemcpyHostToDevice));
            f(RowChunk{s, r, r + m, x.p, false});
        }
    }
};

// the cuts of N rows in chunks of C
static std::vector<uint64_t> uniform_cuts(uint64_t N, uint64_t C)
{
    std::vector<uint64_t> cut{0};
    for (uint64_t r = 0; r < N; r += C) cut.push_back(std::min(N, r + C));
    if (cut.size() == 1) cut.push_back(0);
    return cut;
}

}  // namespace lgpu

using namespace lgpu;

// ---- live-handle registry: every entry point resolves its handle through it, so a handle that was closed (or
// that belongs to the parent of a fork()), or a live handle of another kind, is rejected instead of dereferenced, and
// close waits for the calls still inside the handle (BaseTable is Send + Sync: rust/lancedb/src/table.rs:549; queries
// are re-executable from any tokio worker: rust/lancedb/src/query.rs:954-955).
namespace lgpu {
enum class HandleKind { index, ivf_binary, flat, binary, multivec, comm };
static const char *handle_name(HandleKind k)
{
    static const char *const names[] = {"index", "binary IVF index", "flat", "binary", "multivector", "communicator"};
    return names[(int)k];
}
template <class H> constexpr HandleKind handle_kind();
template <> constexpr HandleKind handle_kind<lgpu_index>() { return HandleKind::index; }
template <> constexpr HandleKind handle_kind<lgpu_ivf_binary>() { return HandleKind::ivf_binary; }
template <> constexpr HandleKind handle_kind<lgpu_flat>() { return HandleKind::flat; }
template <> constexpr HandleKind handle_kind<lgpu_binary>() { return HandleKind::binary; }
template <> constexpr HandleKind handle_kind<lgpu_multivec>() { return HandleKind::multivec; }
template <> constexpr HandleKind handle_kind<lgpu_comm>() { return HandleKind::comm; }

static std::mutex g_live_mu;
static std::condition_variable g_live_cv;
static std::unordered_map<const void *, HandleKind> g_live;
// handles an append holds exclusively (HandleExcl): a call that would enter one waits until the append is done, and so
// does the close of one (retire_handle)
static std::unordered_set<const void *> g_excl;
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
template <class H> static void register_handle(const H *h)
{
    static std::once_flag once;
    std::call_once(once, [] { pthread_atfork(atfork_prepare, atfork_parent, atfork_child); });
    std::lock_guard<std::mutex> g(g_live_mu);
    g_live[h] = handle_kind<H>();
}
// throws unless p is a live handle of kind `want` (g_live_mu held)
static void require_live(const void *p, HandleKind want)
{
    const auto it = p ? g_live.find(p) : g_live.end();
    if (it == g_live.end())
        set_error(std::string(handle_name(want)) + " handle is null, closed, or was opened in another process (fork)");
    else if (it->second != want)
        set_error(std::string(handle_name(want)) + " handle expected, got " +
                  (it->second == HandleKind::index ? "an " : "a ") + handle_name(it->second) + " handle");
    else
        return;
    throw Failure{LGPU_INVALID_INPUT};
}
template <class H> struct HandleRef {
    H *h;
    explicit HandleRef(H *p) : h(nullptr)
    {
        std::unique_lock<std::mutex> g(g_live_mu);
        g_live_cv.wait(g, [&] { return g_excl.empty() || !g_excl.count(p); });
        require_live(p, handle_kind<H>());
        p->refs.fetch_add(1);
        h = p;
    }
    ~HandleRef()
    {
        if (h && h->refs.fetch_sub(1) == 1) { std::lock_guard<std::mutex> g(g_live_mu); g_live_cv.notify_all(); }
    }
    H *operator->() const { return h; }
};
// the handle alone: waits for the calls inside it to finish and keeps new ones out until released (close waits too)
template <class H> struct HandleExcl {
    H *h;
    explicit HandleExcl(H *p) : h(nullptr)
    {
        std::unique_lock<std::mutex> g(g_live_mu);
        g_live_cv.wait(g, [&] { return !g_excl.count(p); });
        require_live(p, handle_kind<H>());
        g_excl.insert(p);
        g_live_cv.wait(g, [&] { return p->refs.load() == 0; });   // p stays allocated: close waits for g_excl
        if (!g_live.count(p)) {                                    // closed meanwhile: let the close go on
            g_excl.erase(p);
            g_live_cv.notify_all();
            set_error(std::string(handle_name(handle_kind<H>())) + " handle was closed during the append");
            throw Failure{LGPU_INVALID_INPUT};
        }
        p->refs.fetch_add(1);
        h = p;
    }
    ~HandleExcl()
    {
        if (!h) return;
        std::lock_guard<std::mutex> g(g_live_mu);
        h->refs.fetch_sub(1);
        g_excl.erase(h);
        g_live_cv.notify_all();
    }
    H *operator->() const { return h; }
};
// unregister and wait until no call is inside the handle any more; false = it was not a live handle of kind H
template <class H> static bool retire_handle(H *p)
{
    std::unique_lock<std::mutex> g(g_live_mu);
    const auto it = p ? g_live.find(p) : g_live.end();
    if (it == g_live.end() || it->second != handle_kind<H>()) return false;
    g_live.erase(it);
    // an append that claimed the handle (HandleExcl) before it was retired is let out first: it sees the handle gone
    // and backs off, or it finishes, before p can be freed
    g_live_cv.wait(g, [&] { return p->refs.load() == 0 && !g_excl.count(p); });
    return true;
}
// every *_close: unregister, drain the handle's device, free it.  A null or closed handle, a handle of another kind,
// or a parent-process handle in a fork child, is left alone.
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

namespace lgpu {
// the kinds of IVF index: 8-bit and 4-bit PQ codes, 8-bit scalar codes (scanned, or searched by per-partition HNSW
// graphs), 1-bit RaBitQ codes, packed binary rows
enum class IvfKind { pq8, pq4, sq, hnsw_sq, rq, ham };
}  // namespace lgpu

struct lgpu_index {
    std::atomic<int> refs{0};
    Coalescer coalescer;
    IvfKind kind = IvfKind::pq8;
    int device = 0, num_sms = 0;
    uint32_t dim = 0, nlist = 0, m = 0, dsub = 0, nch = 0;
    uint32_t max_nrb = 1;          // row blocks (of 1536 rows) of the largest partition: bounds the tile count
    int metric = 0;
    uint64_t nrows = 0, device_bytes = 0;
    DevBuf centroids, cb_tiled, code_base, part_n, part_npad, part_off, row_ids;
    // the stored codes, in the scan's layout.  IVF_SQ, IVF_RQ and binary IVF_FLAT place them at open (place_codes):
    // [nrows][code_row_bytes] in HBM, or in pinned host memory, which a search stages through HBM in chunks of
    // consecutive partitions, code_cut[c] .. code_cut[c + 1] (rows code_rows[c] .. code_rows[c + 1]), at most
    // code_stage bytes each.  The PQ kinds and IVF_HNSW_SQ keep them in `codes.hbm`.
    RowStore codes;
    uint32_t code_row_bytes = 0;
    size_t code_stage = 0;
    std::vector<uint32_t> code_cut;
    std::vector<uint64_t> code_rows;
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
    // the raw vectors (refine_factor), placed by place_vectors: [nrows][vec_stride] f32, vec_stride = dim in HBM, or dim
    // rounded up to 4 (padding zero) in pinned host memory
    RowStore vectors;
    uint32_t vec_stride = 0;
    // IVF_SQ (lgpu_ivf_sq_open): `codes` holds [nrows][dim_pad] u8 row codes, `sq_xx` the sum of each row's squared codes
    uint32_t dim_pad = 0;
    double sq_lo = 0.0, sq_hi = 0.0;
    DevBuf sq_xx;
    // IVF_HNSW_SQ (lgpu_ivf_hnsw_sq_open): IVF_SQ's arrays plus the graph, lgpu_ivf_hnsw_sq_desc's layout
    uint32_t hnsw_m = 0;
    DevBuf hn_levels, hn_adj0, hn_upper_index, hn_upper_adj, hn_entry, hn_top;
    // IVF_RQ (lgpu_ivf_rq_open): `codes` holds [nrows][rq_wpr] u32 sign bits; the rotation, the rotated centroids and
    // the per-row factors and popcounts
    uint32_t rq_wpr = 0;
    DevBuf rq_rot, rq_rc, rq_add, rq_scale, rq_popc;
    // 4-bit IVF_PQ (lgpu_index_open with nbits = 4): `codes` holds per partition [m/2][npad] packed bytes, `pq4_cb` the
    // codebook [m][dsub][16] (element-major); no filter tables
    DevBuf pq4_cb;
    // binary IVF_FLAT (lgpu_ivf_binary_open; `dim` = nbytes): `centroids` holds the packed centroids [nlist][nbytes_pad]
    // and `codes` the packed rows [nrows][nbytes_pad] in partition order, both zero-padded, and their popcounts
    uint32_t nbytes = 0, nbytes_pad = 0;
    DevBuf cent_pop, row_pop;
    std::vector<uint64_t> pad_prefix;   // prefix sums of pad4(n_p) sorted descending
    std::vector<uint32_t> h_part_n;
    RowLive live;
    WorkspacePool pool;
};

// the C header's handle type of a binary IVF_FLAT index (an lgpu_index of kind IvfKind::ham)
struct lgpu_ivf_binary : lgpu_index {};

// What the flat, binary and multivector handles share: their rows (RowStore, in HBM or pinned host memory), optional
// row ids (else the positions), the live bitmap and the workspaces of their searches
struct lgpu_rows {
    std::atomic<int> refs{0};
    int device = 0, num_sms = 0;
    uint64_t nrows = 0;
    RowStore rows;
    DevBuf row_ids;
    bool has_ids = false;
    RowLive live;
    WorkspacePool pool;
};

// a float vector column.  `rows` holds [nrows][dim] f32, or fp16 (f16, lgpu_flat_open_f16); ysqrt, vec_b and vec_n2
// stay empty for a host store
struct lgpu_flat : lgpu_rows {
    uint32_t dim = 0;
    bool f16 = false;
    DevBuf ysqrt;                       // |x| (cosine), built by the first cosine search of an HBM store
    // the tensor-core path: bf16 rows (f32 handles; an fp16 handle's rows are their own operand) + |x|^2
    DevBuf vec_b, vec_n2;
    float vec_max = 0.f, vec_err = 0.f;     // max |x|, max |h(x) - x| (h: bf16 or fp16 rounding, gemm.cu)
    bool has_tc = false;
    bool has_norms = false;
    std::mutex mu;
};

// a packed binary vector column (fixed_size_list<uint8, nbytes>) searched by Hamming distance.  `rows` holds
// [nrows][nbytes_pad] zero-padded rows; `pop` (HBM store only) their popcounts
struct lgpu_binary : lgpu_rows {
    uint32_t nbytes = 0, nbytes_pad = 0;   // caller's row bytes; stored row bytes (multiple of 32)
    DevBuf pop;
    // every (nrows / nsample)-th row: the threshold sample of the list path, in HBM for both placements
    DevBuf sample, sample_pop;
    uint64_t nsample = 0;                  // 0: no sample (nrows <= HAM_SAMPLE)
    DevBuf sample_ids;                     // the sample rows' ids (a row filter tests them in the sample's select)
};

// a multivector column (list<fixed_size_list<float, dim>>) searched by late interaction (MaxSim over cosine).  `rows`
// holds the vectors [T][dim] in the row type (f32, or fp16: lgpu_multivec_open_f16), `ops` (same placement) the fp16
// normalised tensor-core operand [T][dim] of an f32 handle of the tensor-core shape (an fp16 handle's vectors are
// their own operand)
struct lgpu_multivec : lgpu_rows {
    uint64_t total = 0;                    // stored vectors T = offsets[nrows]
    uint32_t dim = 0;
    uint64_t max_row = 0;                  // largest n_r
    bool f16 = false;
    RowStore ops;
    DevBuf ysqrt, offsets;                 // |v| = sqrt(dot(v, v)) per vector, [nrows+1]
    DevBuf col_row;                        // tensor-core path: row of each vector [T]
    bool tc_ok = false;                    // the tensor-core path may run (see multivec_search_device)
    std::vector<uint64_t> h_offsets;       // host copy: the row chunks of a search are cut on the host
};

// the bytes of one stored row
static size_t stored_row_bytes(const lgpu_flat *fl) { return (size_t)fl->dim * (fl->f16 ? 2 : 4); }


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

// bf16 copy + squared norms + max norm and max bf16 rounding error |bf16(x) - x| of a row-major f32 matrix (open time).
// Fp16 rows (f16) are their own operand: no copy (Xb unused), and the error is |h(x) - x| of the fp16 MMA's operand.
// Returns false when a row holds a NaN or inf, or its |x|^2 or rounding error overflows: the error band (tc_band) is
// then not finite for any query, and the caller leaves the operand to the exact kernels.
// The rows' part: Xb and n2 point at room for n rows (an append prepares its new rows only).
static bool tc_operand_rows(const void *X, bool f16, uint64_t n, uint32_t d, void *Xb, float *n2, float &xmax,
                            float &xerr, cudaStream_t st)
{
    DevBuf err;
    err.ensure(std::max<size_t>((size_t)n * 4, 16));
    if (f16) launch_f16_row_terms(X, n, d, n2, err.as<float>(), st);
    else launch_to_bf16(static_cast<const float *>(X), n, d, Xb, n2, st, err.as<float>());
    std::vector<float> h(n), he(n);
    LGPU_CUDA(cudaMemcpyAsync(h.data(), n2, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaMemcpyAsync(he.data(), err.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA(cudaStreamSynchronize(st));
    float m = 0.f, me = 0.f;
    bool finite = true;                        // (std::max skips a NaN: look at every value)
    for (float v : h) { m = std::max(m, v); finite &= std::isfinite(v); }
    for (float v : he) { me = std::max(me, v); finite &= std::isfinite(v); }
    xmax = std::sqrt(m) * 1.0001f;
    xerr = me;
    return finite && std::isfinite(xmax);
}
static bool prepare_tc_operand(const float *X, uint64_t n, uint32_t d, DevBuf &Xb, DevBuf &n2, float &xmax, float &xerr,
                               cudaStream_t st)
{
    Xb.ensure(std::max<size_t>((size_t)n * d * 2, 16));
    n2.ensure(std::max<size_t>((size_t)n * 4, 16));
    return tc_operand_rows(X, false, n, d, Xb.p, n2.as<float>(), xmax, xerr, st);
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

// the ids of the columns of a block of scores: ids[c], or base + c without ids (base: the position of the block's first
// row in its column, nonzero for a chunk of a streamed flat column)
struct Cols {
    const uint64_t *ids;
    uint64_t base;
    Cols(const uint64_t *i = nullptr, uint64_t b = 0) : ids(i), base(b) {}
};

// the ids of rows [r0, ..) of a handle: its explicit ids from r0, or the positions from r0
static Cols row_cols(const lgpu_rows *h, uint64_t r0)
{
    return h->has_ids ? Cols(static_cast<const uint64_t *>(h->row_ids.p) + r0) : Cols(nullptr, r0);
}

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
static void with_cols(SelectArgs &s, Cols c)
{
    s.col_ids = c.ids; s.col_base = c.base;
}
static void with_range(SelectArgs &s, const lgpu_search_params &sp)
{
    s.has_lower = sp.has_lower; s.has_upper = sp.has_upper; s.lower = sp.lower; s.upper = sp.upper;
}
// k > SELECT_KMAX: the large select's scratch, from the workspace (nothing for k <= SELECT_KMAX)
static SelectArgs &with_scratch(Workspace *ws, SelectArgs &s)
{
    if (s.k > SELECT_KMAX) {
        s.scratch_bytes = select_large_scratch_bytes(s.B, s.k, s.out_pos != nullptr);
        ws->sel_large.ensure(s.scratch_bytes);
        s.scratch = ws->sel_large.p;
    }
    return s;
}
// workspace bytes per query that grow with k: the large select's scratch above SELECT_KMAX (below it, every per-query
// buffer is bounded by SELECT_KMAX entries and stays outside the sub-batch budget, DESIGN.md section 2)
static size_t large_k_query_bytes(uint32_t k)
{
    return k > SELECT_KMAX ? select_large_scratch_bytes(1, k, true) : 0;
}

// The tail of tc_topk_l2 and tc_topk_l2_filtered: exact re-score of the [B][cap] candidate slots (ws->t_pos, t_ids;
// one pair per slot, empty slots included; every candidate passed the row filter), their top-k into the outputs, then
// the dense fix-up of the queries flagged in ws->flags under the row filter (no-ops when none is).  T: the stored row
// type (float, or __half for an fp16 flat handle, whose rows X are also the GEMM operand Xb).
template <class T>
static void tc_rescore_fixup(Workspace *ws, cudaStream_t st, const float *Q, uint32_t B, const T *X, uint64_t N,
                             uint32_t d, Cols cols, uint32_t k, uint32_t cap, TopkOut out, float *Dbuf, uint64_t ld,
                             RowFilter rf)
{
    launch_pair_distance(Q, X, ws->t_pos.as<uint64_t>(), B, cap, d, LGPU_L2, ws->t_exact.as<float>(), st);
    launch_select(select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), cap, B, k, out), st);
    launch_dist_matrix(Q, X, B, N, d, 0, nullptr, nullptr, Dbuf, ld, st, ws->flags.as<uint32_t>());
    SelectArgs sc = select_rows(Dbuf, N, ld, B, k, out);
    with_cols(sc, cols); sc.only = ws->flags.as<uint32_t>();
    sc.allow = rf.bits; sc.allow_bits = rf.nbits;
    launch_select(sc, st);
}

// Tensor-core shortlist + exact re-score (squared L2 only): the k best of the N rows of X that pass the row filter rf
// (none: every row) for each of B queries by exact lance-order distance, ids from cols,
// ascending by (distance, id).  Dbuf: [B][ld] f32 scratch.  The shortlist holds the kp best allowed rows by approximate
// score; queries whose shortlist cannot be proven complete (band_check: it is full and its last score is within the
// band of the k-th) are redone by the exact kernels in the same stream, without a host round trip.
// the 16-bit query operand of the tensor-core paths (bf16, or fp16 for fp16 rows), |q|^2 and |h(q) - q|
template <class T> static void tc_queries(Workspace *ws, cudaStream_t st, const float *Q, uint32_t B, uint32_t d)
{
    ws->qb.ensure((size_t)B * d * 2); ws->qn2.ensure((size_t)B * 4); ws->qerr.ensure((size_t)B * 4);
    if (std::is_same<T, __half>::value) launch_to_f16(Q, B, d, ws->qb.p, ws->qn2.as<float>(), ws->qerr.as<float>(), st);
    else launch_to_bf16(Q, B, d, ws->qb.p, ws->qn2.as<float>(), st, ws->qerr.as<float>());
}

template <class T>
static void tc_topk_l2(Workspace *ws, cudaStream_t st, int num_sms, const float *Q, uint32_t B, const T *X,
                       const void *Xb, const float *xnorm2, float xmax, float xerr, uint64_t N, uint32_t d,
                       Cols cols, uint32_t k, uint32_t kp, TopkOut out, float *Dbuf, uint64_t ld, RowFilter rf)
{
    constexpr bool f16 = std::is_same<T, __half>::value;
    ws->flags.ensure((size_t)B * 4);
    ws->t_ids.ensure((size_t)B * kp * 8); ws->t_dist.ensure((size_t)B * kp * 4);
    ws->t_pos.ensure((size_t)B * kp * 8); ws->t_cnt.ensure((size_t)B * 4); ws->t_exact.ensure((size_t)B * kp * 4);
    tc_queries<T>(ws, st, Q, B, d);
    launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, N, d, Dbuf, ld, num_sms, st, nullptr, f16);
    SelectArgs sa = select_rows(Dbuf, N, ld, B, kp, {ws->t_ids.as<uint64_t>(), ws->t_dist.as<float>(),
                                                     ws->t_cnt.as<uint32_t>(), ws->t_pos.as<uint64_t>()});
    with_cols(sa, cols);
    sa.allow = rf.bits; sa.allow_bits = rf.nbits;
    launch_select(sa, st);
    if (kp >= N) LGPU_CUDA(cudaMemsetAsync(ws->flags.p, 0, (size_t)B * 4, st));   // every row is a candidate
    else launch_band_check(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->qn2.as<float>(), ws->qerr.as<float>(),
                           xmax, xerr, d, B, k, kp, ws->flags.as<uint32_t>(), st);
    tc_rescore_fixup(ws, st, Q, B, X, N, d, cols, k, kp, out, Dbuf, ld, rf);
}

// Large-N variant of tc_topk_l2 (flat search): a tensor-core pass over a row sample fixes, per query, a
// score threshold that provably admits every true top-k row (from the k best sample rows that pass the row filter rf:
// with fewer, +inf); the pass over all rows then runs with the filtering epilogue (no dense score matrix), admitting
// the rows under the threshold that pass rf, the few admitted rows are re-scored exactly, and queries whose candidate
// list overflowed are redone by the exact kernels.
template <class T>
static void tc_topk_l2_filtered(Workspace *ws, cudaStream_t st, int num_sms, const float *Q, uint32_t B, const T *X,
                                const void *Xb, const float *xnorm2, float xmax, float xerr, uint64_t N, uint32_t d,
                                Cols cols, uint32_t k, TopkOut out, float *Dbuf, uint64_t ld, RowFilter rf,
                                uint64_t min_sample = 65536, uint32_t cap = 1024)
{
    constexpr bool f16 = std::is_same<T, __half>::value;
    const uint64_t Ns = std::min<uint64_t>(N, std::max<uint64_t>(min_sample, N / 8));
    const uint64_t lds = (Ns + 3) & ~3ull;               // Dbuf is [B][ld >= lds]
    ws->flags.ensure((size_t)B * 4);
    ws->t_ids.ensure((size_t)B * cap * 8); ws->t_dist.ensure((size_t)B * std::max<uint32_t>(k, 32) * 4);
    ws->t_pos.ensure((size_t)B * cap * 8); ws->t_cnt.ensure((size_t)B * 4); ws->t_exact.ensure((size_t)B * cap * 4);
    ws->probe_A.ensure((size_t)B * 4);                   // thr[q]
    ws->amax.ensure((size_t)B * 4);                      // candidate counters
    ws->sbound.ensure((size_t)B * std::max<uint32_t>(k, 32) * 8);   // sample ids (unused)
    tc_queries<T>(ws, st, Q, B, d);
    // 1. sample pass: dense scores of the first Ns rows, k-th best per query -> threshold
    launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, Ns, d, Dbuf, lds, num_sms, st, nullptr, f16);
    SelectArgs ss = select_rows(Dbuf, Ns, lds, B, k, {ws->sbound.as<uint64_t>(), ws->t_dist.as<float>(),
                                                      ws->t_cnt.as<uint32_t>()});
    if (rf.bits) { with_cols(ss, cols); ss.allow = rf.bits; ss.allow_bits = rf.nbits; }
    launch_select(ss, st);
    launch_sample_threshold(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), ws->qn2.as<float>(), ws->qerr.as<float>(),
                            xmax, xerr, d, B, k, ws->probe_A.as<float>(), st);
    // 2. full pass with the filtering epilogue
    LGPU_CUDA(cudaMemsetAsync(ws->amax.p, 0, (size_t)B * 4, st));
    LGPU_CUDA(cudaMemsetAsync(ws->t_pos.p, 0xff, (size_t)B * cap * 8, st));
    LGPU_CUDA(cudaMemsetAsync(ws->t_ids.p, 0xff, (size_t)B * cap * 8, st));
    GemmFilter flt{};
    flt.thr = ws->probe_A.as<float>(); flt.count = ws->amax.as<uint32_t>(); flt.cand_pos = ws->t_pos.as<uint64_t>();
    flt.cand_ids = ws->t_ids.as<uint64_t>(); flt.col_ids = cols.ids; flt.col_base = cols.base; flt.cap = cap;
    flt.allow = rf.bits; flt.allow_bits = rf.nbits;
    if (Ns == N) launch_filter_dense(Dbuf, lds, B, N, flt, st);      // the sample pass already scored every row
    else launch_gemm_dist(ws->qb.p, Xb, xnorm2, B, N, d, nullptr, 0, num_sms, st, &flt, f16);
    launch_overflow_flags(ws->amax.as<uint32_t>(), cap, ws->probe_A.as<float>(), B, ws->flags.as<uint32_t>(), st);
    // 3. exact re-score of the admitted rows, final top-k; 4. fix-up of overflowed queries
    tc_rescore_fixup(ws, st, Q, B, X, N, d, cols, k, cap, out, Dbuf, ld, rf);
}

// top-k by (distance, id) of the dense scores D [b][ld] over N columns, with the request's distance range and
// prefilter, into `out`
static void select_dense(Workspace *ws, const float *D, uint64_t N, uint64_t ld, Cols cols, uint32_t b,
                         const lgpu_search_params &sp, RowFilter rf, TopkOut out, cudaStream_t st)
{
    SelectArgs sa = select_rows(D, N, ld, b, sp.k, out);
    with_cols(sa, cols);
    with_range(sa, sp);
    sa.allow = rf.bits; sa.allow_bits = rf.nbits;
    launch_select(with_scratch(ws, sa), st);
}

// the arguments every search call takes: the parameters, then the query and output buffers of a call with queries.
// k = limit + offset, and k * refine_factor when the kind re-ranks, go up to LGPU_K_MAX on every single-GPU search:
// up to SELECT_KMAX on the shared-memory selects, above it on the large select (select_large.cu) over the kind's exact
// route.  refine: the kind selects k * refine_factor candidates (a kind whose distances are exact ignores
// refine_factor).  The sharded search adds its own bound (SELECT_KMAX, check_sharded_call).
static void check_call(const lgpu_search_params *p, uint32_t B, const void *q, const void *ids, const void *dist,
                       const void *cnt, bool refine = true)
{
    LGPU_REQUIRE(p != nullptr, "search params are null");
    LGPU_REQUIRE(p->k >= 1, "limit must be greater than 0");
    LGPU_REQUIRE(p->k <= LGPU_K_MAX, "limit+offset above 65536 (LGPU_K_MAX) is not supported");
    if (refine && p->refine_factor)
        LGPU_REQUIRE((uint64_t)p->k * p->refine_factor <= LGPU_K_MAX,
                     "limit*refine_factor above 65536 (LGPU_K_MAX) is not supported");
    LGPU_REQUIRE(B == 0 || (q && ids && dist && cnt), "null buffer");
}

// binary vectors (Hamming distance): the crossovers of the flat search (DESIGN.md section 6) and of the binary IVF
// coarse step
constexpr uint64_t HAM_SAMPLE = 65536;     // rows of the threshold sample
constexpr uint32_t HAM_TC_MIN_B = 128;     // dense tensor-core path from this many queries (measured: SIMT faster at
                                           // 64 queries x 60000 rows, wgmma at 256) ...
constexpr uint64_t HAM_TC_MIN_N = 4096;    // ... and this many rows (not measured)

// ---- IVF search (IVF_PQ 8-bit and 4-bit, IVF_SQ, IVF_RQ and binary IVF_FLAT).  One sub-batch runs [cosine:
// normalise] -> coarse step (probes) -> small scan | regroup -> filter scan + fix-up | exact scan + select -> [refine],
// on the paths ivf_plan picks before any launch ----
enum class Coarse { exact, tc_dense, tc_list };   // see ivf_coarse
enum class IvfScan { small, filter_cand, filter_dense, exact_pq, sq, rq, pq4, ham, hnsw };

// bytes of one stored row, as the scan reads them (profiling: lgpu_last_scanned_code_bytes)
static uint32_t ivf_row_bytes(const lgpu_index *ix)
{
    switch (ix->kind) {
    case IvfKind::pq8: return ix->m;
    case IvfKind::pq4: return ix->m / 2;
    case IvfKind::sq: case IvfKind::hnsw_sq: return ix->dim;
    case IvfKind::rq: return ix->rq_wpr * 4;
    case IvfKind::ham: return ix->nbytes_pad;
    }
    return 0;
}

// workspace bytes per query of a sub-batch that only the kind uses: the per-slot u8 tables (pq4), the per-slot
// bit-planes and the rotated query (rq), the probe slots' ids, distances, regroup and tile descriptors (ham), the probe
// slots' [kk] result lists (hnsw_sq; kk = 0: not known, the largest)
static size_t ivf_kind_query_bytes(const lgpu_index *ix, uint32_t nprobes, uint32_t np_eff, uint32_t kk)
{
    switch (ix->kind) {
    case IvfKind::hnsw_sq: return (size_t)nprobes * (kk ? kk : LGPU_HNSW_EF_MAX) * 20;
    case IvfKind::pq4: return (size_t)nprobes * (16 * ix->m + sizeof(Pq4Slot));
    case IvfKind::rq: return (size_t)nprobes * (16 * ix->rq_wpr + sizeof(RqSlot)) + (size_t)ix->dim * 4;
    case IvfKind::ham: return (size_t)np_eff * 36 + (size_t)np_eff * ix->max_nrb * (sizeof(TileDesc) / SCAN_G + 1) + 64;
    default: return 0;
    }
}

// the queries of an IVF sub-batch in the kind's format: f32 rows [B][dim], or (ham) rows packed to [B][nbytes_pad]
// bytes and their popcounts
struct IvfQueries {
    const float *f;
    const uint8_t *h;
    const uint32_t *pop;
    size_t ld;                // elements of one row
    IvfQueries at(uint32_t q0) const
    {
        return {f ? f + q0 * ld : nullptr, h ? h + q0 * ld : nullptr, pop ? pop + q0 : nullptr, ld};
    }
};

struct IvfPlan {
    uint32_t B, nprobes, slots;
    uint32_t np_eff;          // probes that can hold rows: min(nprobes, nlist)
    uint32_t k, kk;           // the request's k; the PQ top-kk (k, or k * refine_factor candidates for the re-rank)
    uint32_t lb_short;        // dense filter scan: the rows of the lb_short smallest lower bounds are re-scored
    bool refine;
    Coarse coarse;
    IvfScan scan;
    uint32_t cand_cap;        // candidate mode: candidates per query (power of two >= kk)
    uint32_t efp;             // hnsw: W's capacity, ef' = max(ef, kk)
    bool filter() const { return scan == IvfScan::filter_cand || scan == IvfScan::filter_dense; }
    uint32_t rows_tile() const
    {
        if (filter()) return SCAN3_ROWS_TILE;
        if (scan == IvfScan::pq4) return PQ4_ROWS_TILE;
        if (scan == IvfScan::ham) return HAM_ROWS_TILE;
        return scan == IvfScan::sq ? SQ_ROWS_TILE : (scan == IvfScan::rq ? RQ_ROWS_TILE : SCAN_ROWS_TILE_MID);
    }
};

// IVF_HNSW_SQ's ef' = max(ef, kk), ef = 0 meaning ceil(1.5 k) (query.rs:1290-1300)
static uint64_t hnsw_efp(const lgpu_search_params &sp)
{
    const uint64_t kk = sp.refine_factor ? (uint64_t)sp.k * sp.refine_factor : sp.k;
    return std::max<uint64_t>(sp.ef ? sp.ef : (3ull * sp.k + 1) / 2, kk);
}

// prefilter: the request carries an allow bitmap; widening: the sub-batch redoes the queries flagged by the
// maximum_nprobes widening (exact kernels only)
static IvfPlan ivf_plan(const lgpu_index *ix, uint32_t B, uint32_t nprobes, const lgpu_search_params &sp, bool prefilter,
                        bool widening, const ScanModes &modes)
{
    IvfPlan p{};
    const uint32_t nlist = ix->nlist;
    p.B = B; p.nprobes = nprobes; p.slots = B * nprobes; p.np_eff = std::min(nprobes, nlist);
    p.k = sp.k; p.kk = sp.refine_factor ? sp.k * sp.refine_factor : sp.k; p.refine = sp.refine_factor != 0;
    // kk above SELECT_KMAX: the exact scan (or the small path) feeds every row to the large select; the filter scan's
    // shortlists are sized to SELECT_KMAX (lb_short) and its candidate mode to CAND_TOPK_MAX
    const bool large_k = p.kk > SELECT_KMAX;
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
    // every kind but 8-bit PQ: one exact scan, never the small or the filter path.  Hamming distances are exact:
    // no refine.
    switch (ix->kind) {
    case IvfKind::pq4: p.scan = IvfScan::pq4; return p;
    case IvfKind::sq: p.scan = IvfScan::sq; return p;
    case IvfKind::hnsw_sq: p.scan = IvfScan::hnsw; p.efp = hnsw_efp(sp); return p;
    case IvfKind::rq: p.scan = IvfScan::rq; return p;
    case IvfKind::ham: p.scan = IvfScan::ham; p.kk = p.k; p.refine = false; return p;
    case IvfKind::pq8: break;
    }
    // tiny batches (a single query, a micro-batch): the small path, 4 launches instead of ~25; LGPU_SMALL_SLOTS = 0
    // disables it.  Otherwise filter + verify (scan3.cu) unless the request needs every exact distance.
    const bool small = !widening && p.slots <= modes.small_slots && small_scan_smem(ix->m, ix->dim) <= 200 * 1024 &&
                       (size_t)p.slots * ix->pad_prefix[1] * 4 <= workspace_budget();
    const bool filter = ix->has_tables && !modes.exact && !sp.has_lower && !sp.has_upper && p.lb_short > p.kk &&
                        ix->m <= 512 && !widening && !small && !large_k;
    if (small) p.scan = IvfScan::small;
    else if (!filter) p.scan = IvfScan::exact_pq;
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
// Binary IVF_FLAT: Hamming distances to the packed centroids, or every partition when nprobes covers them all.
static void ivf_coarse(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const IvfQueries &q, cudaStream_t cs,
                       cudaStream_t st, const StageMarks &mark)
{
    const uint32_t B = p.B, nprobes = p.nprobes, nlist = ix->nlist, dim = ix->dim;
    const float *qs = q.f;
    ws->probes.ensure((size_t)p.slots * 8);
    if (p.scan == IvfScan::ham && nprobes >= nlist) {   // every partition: no coarse step, no top-nprobes select
        launch_ham_all_probes(ws->probes.as<uint64_t>(), B, nlist, cs);
        mark(IVF_COARSE, cs);
        return;
    }
    ws->probe_dist.ensure((size_t)p.slots * 4);
    ws->probe_cnt.ensure((size_t)B * 4);
    const uint64_t ldc = (nlist + 3u) & ~3u;
    ws->D.ensure((size_t)B * ldc * 4);
    const TopkOut probes{ws->probes.as<uint64_t>(), ws->probe_dist.as<float>(), ws->probe_cnt.as<uint32_t>()};
    if (p.coarse == Coarse::exact) {
        // binary: the b1 wgmma kernel from the flat path's crossover (HAM_TC_MIN_B x HAM_TC_MIN_N); for the coarse
        // step's shapes the crossover is not measured
        if (p.scan != IvfScan::ham)
            launch_dist_matrix(qs, ix->centroids.as<float>(), B, nlist, dim, ix->metric == LGPU_DOT ? 1 : 0, nullptr,
                               nullptr, ws->D.as<float>(), ldc, cs);
        else if (tc_enabled() && B >= HAM_TC_MIN_B && nlist >= HAM_TC_MIN_N)
            launch_ham_gemm(q.h, ix->centroids.p, ix->cent_pop.as<uint32_t>(), q.pop, B, nlist, ix->nbytes_pad,
                            ws->D.as<float>(), ldc, ix->num_sms, cs);
        else
            launch_ham_dense(q.h, ix->centroids.as<uint8_t>(), B, nlist, ix->nbytes_pad, ws->D.as<float>(), ldc,
                             ix->num_sms, cs);
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
    ss.codes = ix->codes.hbm.as<unsigned char>(); ss.code_base = ix->code_base.as<uint64_t>();
    ss.part_n = ix->part_n.as<uint32_t>(); ss.part_npad = ix->part_npad.as<uint32_t>();
    ss.dim = ix->dim; ss.m = ix->m; ss.nch = ix->nch; ss.metric = (uint32_t)ix->metric; ss.nlist = ix->nlist;
    ss.nprobes = p.nprobes;
    ss.queries = qs; ss.probes = ws->probes.as<uint64_t>(); ss.seg_stride = stride;
    ss.seg_off = ws->seg_off.as<uint64_t>(); ss.dist_out = ws->dist_out.as<float>();
    launch_small_scan(ss, ix->dsub, p.slots, st);
    mark(IVF_SCAN, st);
    SelectArgs sa = select_segments(ix, ws, p, p.kk, pq_out(ws, p, out), rf);
    with_range(sa, sp);
    launch_select(with_scratch(ws, sa), st);
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
    sc.codes = ix->codes.hbm.as<unsigned char>(); sc.code_base = ix->code_base.as<uint64_t>();
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
    a.codes = ix->codes.hbm.as<uint32_t>(); a.tables = ws->pq4_tab.as<uint8_t>(); a.slots = ws->pq4_slots.as<Pq4Slot>();
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
    fa.codes = ix->codes.hbm.as<unsigned char>(); fa.code_base = ix->code_base.as<uint64_t>();
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
    launch_pq_rescore(qs, ws->s_pos.as<uint64_t>(), B, kp, ix->codes.hbm.as<unsigned char>(), ix->code_base.as<uint64_t>(),
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

// The scan of a row-major kind (sq, rq, ham) with `rows(a, X)` setting its rows to X, over the walk of its codes.  An
// HBM index: one launch over the whole tile queue of its own rows.  An index whose codes are in pinned host memory:
// chunk c's probed partitions (part_cnt of the regroup, so the flagged queries' probes in the maximum_nprobes pass) are
// copied into a staging buffer by launch_codes_copy_gated on the side stream while chunk c - 1 is scanned; then the
// scan runs over chunk c's tiles alone (TileRange, its own claim counter in code_ctr, after the walk's byte count),
// its rows read from the buffer.  Nothing waits on the host but the deadline, checked between chunks.
template <class Args, class Rows, class Launch>
static void scan_codes(lgpu_index *ix, Workspace *ws, const GroupArgs &ga, Args a, Rows &&rows, Launch &&launch,
                       const Deadline *deadline, cudaStream_t st)
{
    a.total_tiles = ga.total_tiles; a.tile_counter = ga.tile_counter; a.tile_desc = ga.tile_desc;
    a.dist_out = ws->dist_out.as<float>();
    const std::vector<uint32_t> &cut = ix->code_cut;
    const uint64_t rb = ix->code_row_bytes;
    ix->codes.reserve_stage(ws, ix->code_stage);
    if (ix->codes.on_host) LGPU_CUDA(cudaMemsetAsync(ws->code_ctr.as<uint32_t>() + 2, 0, (cut.size() - 1) * 4, st));
    ix->codes.walk(
        ws, st, ix->code_rows, [&](uint64_t r) { return r * rb; }, deadline,
        [&](const RowChunk &ch) {
            rows(a, ch.X);
            if (!ch.resident) {
                const uint64_t c = ch.s;
                a.range = {ga.tile_off + cut[c], ga.tile_off_b + cut[c], cut[c + 1] - cut[c], (uint32_t)ch.r0};
                a.tile_counter = ws->code_ctr.as<uint32_t>() + 2 + c;
            }
            launch(a, 2 * ix->num_sms, st);
        },
        [&](uint64_t c, void *buf, cudaStream_t fs) {
            launch_codes_copy_gated(static_cast<const uint8_t *>(ix->codes.dev()), static_cast<uint8_t *>(buf), rb,
                                    ix->part_off.as<uint64_t>(), ga.part_cnt, cut[c], cut[c + 1],
                                    (ix->code_rows[c + 1] - ix->code_rows[c]) * rb,
                                    ws->code_ctr.as<unsigned long long>(), ix->num_sms, fs);
        });
}

// IvfScan::exact_pq / sq / rq / pq4 / ham: the exact scan of every regrouped tile, then the PQ top-kk
static void ivf_exact(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const lgpu_search_params &sp,
                      const IvfQueries &q, const GroupArgs &ga, RowFilter rf, const uint32_t *only, TopkOut pq,
                      cudaStream_t st, const StageMarks &mark, const Deadline *deadline)
{
    if (p.scan == IvfScan::sq) {
        SqScanArgs qa{};
        qa.xx = ix->sq_xx.as<uint32_t>();
        qa.qcodes = ws->sq_q.as<uint8_t>(); qa.qq = ws->sq_qq.as<uint32_t>(); qa.dim_pad = ix->dim_pad;
        scan_codes(ix, ws, ga, qa, [](SqScanArgs &a, const void *X) { a.codes = static_cast<const uint8_t *>(X); },
                   launch_sq_scan, deadline, st);
    } else if (p.scan == IvfScan::rq) {
        RqScanArgs ra{};
        ra.add = ix->rq_add.as<float>(); ra.scale = ix->rq_scale.as<float>();
        ra.popc = ix->rq_popc.as<uint32_t>();
        ra.planes = ws->rq_planes.as<uint32_t>(); ra.slots = ws->rq_slots.as<RqSlot>();
        ra.dim = ix->dim; ra.wpr = ix->rq_wpr; ra.cosine = ix->metric == LGPU_COSINE;
        scan_codes(ix, ws, ga, ra, [](RqScanArgs &a, const void *X) { a.codes = static_cast<const uint32_t *>(X); },
                   launch_rq_scan, deadline, st);
    } else if (p.scan == IvfScan::pq4) {
        launch_pq4_scan(pq4_args(ix, ws, ga), 2 * ix->num_sms, st);
    } else if (p.scan == IvfScan::ham) {
        HamScanArgs ha{};
        ha.row_pop = ix->row_pop.as<uint32_t>(); ha.queries = q.h; ha.qpop = q.pop;
        ha.nbytes_pad = ix->nbytes_pad;
        scan_codes(ix, ws, ga, ha, [](HamScanArgs &a, const void *X) { a.rows = static_cast<const uint8_t *>(X); },
                   launch_ivf_ham_scan, deadline, st);
    } else {
        launch_scan2(scan_args(ix, ws, q.f, ga), ix->dsub, ix->num_sms, st);
    }
    mark(IVF_SCAN, st);
    SelectArgs sa = select_segments(ix, ws, p, p.kk, pq, rf);
    sa.only = only;
    with_range(sa, sp);
    launch_select(with_scratch(ws, sa), st);
    mark(IVF_TOPK, st);
}

// IvfScan::hnsw: the graph search of every probe slot into its [kk] list (hnsw_scan.cu), then the top-kk over a query's
// nprobes lists.  Each list already holds only rows that pass the row filter.
static void ivf_hnsw(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const lgpu_search_params &sp, RowFilter rf,
                     const uint32_t *only, TopkOut pq, cudaStream_t st, const StageMarks &mark)
{
    const size_t n = (size_t)p.slots * p.kk;
    ws->hn_ids.ensure(n * 8); ws->hn_dist.ensure(n * 4); ws->hn_pos.ensure(n * 8); ws->hn_ctr.ensure(16);
    LGPU_CUDA(cudaMemsetAsync(ws->hn_ctr.p, 0, 4, st));
    HnswArgs a{};
    a.codes = ix->codes.hbm.as<uint8_t>(); a.qcodes = ws->sq_q.as<uint8_t>(); a.dim_pad = ix->dim_pad;
    a.probes = ws->probes.as<uint64_t>(); a.slots = p.slots; a.nprobes = p.nprobes; a.nlist = ix->nlist;
    a.part_off = ix->part_off.as<uint64_t>(); a.row_ids = ix->row_ids.as<uint64_t>();
    a.levels = ix->hn_levels.as<uint8_t>(); a.adj0 = ix->hn_adj0.as<uint32_t>();
    a.upper_index = ix->hn_upper_index.as<uint32_t>(); a.upper_adj = ix->hn_upper_adj.as<uint32_t>();
    a.entry = ix->hn_entry.as<uint32_t>(); a.top_level = ix->hn_top.as<uint8_t>();
    a.m = ix->hnsw_m; a.efp = p.efp; a.kk = p.kk;
    a.has_lower = sp.has_lower; a.has_upper = sp.has_upper; a.lower = sp.lower; a.upper = sp.upper;
    a.allow = rf.bits; a.allow_bits = rf.nbits; a.only = only;
    a.counter = ws->hn_ctr.as<uint32_t>();
    a.out_ids = ws->hn_ids.as<uint64_t>(); a.out_dist = ws->hn_dist.as<float>(); a.out_pos = ws->hn_pos.as<uint64_t>();
    launch_hnsw_search(a, ix->num_sms, st);
    mark(IVF_SCAN, st);
    SelectArgs sa = select_cands(a.out_dist, a.out_ids, (uint64_t)p.nprobes * p.kk, p.B, p.kk, pq);
    sa.cand_pos = a.out_pos; sa.only = only;
    launch_select(sa, st);
    mark(IVF_TOPK, st);
}

// refine (query.rs:1302-1332): exact distance of the k * refine_factor candidates (ws->t_*), re-sort into `out`
static void ivf_refine(lgpu_index *ix, Workspace *ws, const IvfPlan &p, const float *d_q, TopkOut out,
                       const uint32_t *only, cudaStream_t st)
{
    const float *X = static_cast<const float *>(ix->vectors.dev());
    if (ix->vectors.on_host)
        launch_refine_host(d_q, X, ix->vec_stride, ws->t_pos.as<uint64_t>(), p.B, p.kk, ix->dim, ix->metric,
                           ws->t_exact.as<float>(), ix->num_sms, st);
    else
        launch_pair_distance(d_q, X, ws->t_pos.as<uint64_t>(), p.B, p.kk, ix->dim, ix->metric, ws->t_exact.as<float>(),
                             st);
    SelectArgs sr = select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), p.kk, p.B, p.k, out);
    sr.only = only;
    launch_select(with_scratch(ws, sr), st);
}

// one sub-batch of an IVF search, everything device-side on `st` (and `front`, joined).  only (device, [B]): redo just
// the flagged queries (maximum_nprobes widening) -- exact kernels, the other queries' outputs are left untouched.
void ivf_sub_batch(lgpu_index *ix, Workspace *ws, cudaStream_t st, const IvfQueries &q, uint32_t B,
                   const lgpu_search_params &sp, uint32_t nprobes, TopkOut out, bool prof, RowFilter rf,
                   const Deadline *deadline, const uint32_t *only = nullptr)
{
    const IvfPlan p = ivf_plan(ix, B, nprobes, sp, rf.bits != nullptr, only != nullptr, scan_modes());
    const StageMarks mark{ws, prof};
    mark(IVF_START, st);
    ws->stats_mode = 0;
    IvfQueries prep = q;
    prep.f = ivf_queries(ix, ws, st, q.f, B);
    const float *qs = prep.f;
    const cudaStream_t cs = p.filter() ? fork_front(ix, ws, st, B) : st;   // the coarse step's and the regroup's
    ivf_coarse(ix, ws, p, prep, cs, st, mark);
    if (p.scan == IvfScan::sq || p.scan == IvfScan::hnsw) {
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
    } else if (p.scan == IvfScan::hnsw) {
        ivf_hnsw(ix, ws, p, sp, rf, only, pq_out(ws, p, out), st, mark);
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
            ivf_exact(ix, ws, p, sp, prep, ga, rf, only, pq, st, mark, deadline);
        }
    }
    if (!p.refine) return;
    ivf_refine(ix, ws, p, q.f, out, only, st);
    mark(IVF_REFINE, st);
}

// kk: the PQ top-kk of the request (0: not known, lgpu_debug_sub_batch_size)
uint32_t ivf_sub_batch_size(lgpu_index *ix, uint32_t B, uint32_t nprobes, uint32_t kk = 0)
{
    uint32_t np_eff = std::min<uint32_t>(nprobes, ix->nlist);
    // distance segments, coarse scores, the filter scan's per-query tables, then the kind's own buffers; above
    // SELECT_KMAX the large select's scratch and the refine stage's [kk] candidates (ids, distances, positions, exact
    // distances) grow with kk and count too
    size_t per_q = std::max<size_t>(ix->pad_prefix[np_eff] * 4 + (size_t)ix->nlist * 4 + (size_t)ix->nch * 256 * 8 * 4, 4) +
                   ivf_kind_query_bytes(ix, nprobes, np_eff, kk) + large_k_query_bytes(kk) +
                   (kk > SELECT_KMAX ? (size_t)kk * 28 : 0);
    // an index whose codes are in pinned host memory leases its two staging buffers from the same budget
    const size_t budget = workspace_budget(), stage = ix->codes.on_host ? 2 * ix->code_stage : 0;
    size_t bs = (budget > stage ? budget - stage : 0) / per_q;
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

// the queries of an IVF call in the kind's format: the caller's f32 rows, or (ham) the caller's bytes [B][nbytes]
// packed once per call into ws->hq / hq_pop
static IvfQueries ivf_call_queries(lgpu_index *ix, Workspace *ws, cudaStream_t st, const void *d_q, uint32_t B)
{
    if (ix->kind != IvfKind::ham) return {static_cast<const float *>(d_q), nullptr, nullptr, ix->dim};
    const uint32_t nbp = ix->nbytes_pad;
    ws->hq.ensure((size_t)B * nbp); ws->hq_pop.ensure((size_t)B * 4);
    launch_ham_pack(static_cast<const uint8_t *>(d_q), ix->nbytes, ix->nbytes, B, ws->hq.as<uint8_t>(), nbp,
                    ws->hq_pop.as<uint32_t>(), st);
    return {nullptr, ws->hq.as<uint8_t>(), ws->hq_pop.as<uint32_t>(), nbp};
}

// d_q: the caller's queries in device memory, [B][dim] f32 or (binary IVF_FLAT) [B][nbytes] bytes
void ivf_search_device(lgpu_index *ix, Workspace *ws, cudaStream_t st, const void *d_q, uint32_t B,
                       const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                       RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint32_t nprobes = std::min<uint32_t>(std::max<uint32_t>(sp.nprobes, 1), ix->nlist);
    // maximum_nprobes (query.rs:1250-1275): under a prefilter, the queries that found fewer than k rows in their
    // minimum_nprobes partitions are searched again over their maximum_nprobes nearest (no work if none is)
    const uint32_t np_max = std::min<uint32_t>(sp.max_nprobes, ix->nlist);
    const bool widen = rf.bits && np_max > nprobes;
    if (widen)
        LGPU_REQUIRE(np_max <= SELECT_KMAX || np_max >= ix->nlist,
                     "maximum_nprobes above 2048 is not supported unless it covers every partition");
    const uint32_t kk = sp.refine_factor && ix->kind != IvfKind::ham ? sp.k * sp.refine_factor : sp.k;
    const uint32_t bs = ivf_sub_batch_size(ix, B, widen ? np_max : nprobes, kk);
    const bool prof = profiling_enabled();
    if (prof) {
        memset(g_stage_ms, 0, sizeof(g_stage_ms));
        memset(g_filter_stats, 0, sizeof(g_filter_stats));
        g_scanned_bytes = 0;
        g_streamed_bytes = 0;
    }
    if (ix->codes.on_host) {       // the walk's byte count (code_ctr[0]) and one tile counter per chunk (scan_codes)
        ws->code_ctr.ensure(8 + ix->code_cut.size() * 4);
        LGPU_CUDA(cudaMemsetAsync(ws->code_ctr.p, 0, 8, st));
    }
    const IvfQueries qs = ivf_call_queries(ix, ws, st, d_q, B);
    const TopkOut out{d_ids, d_dist, d_cnt};
    for (uint32_t q0 = 0; q0 < B; q0 += bs) {
        uint32_t b = std::min(bs, B - q0);
        if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);      // the previous sub-batch, or LGPU_TIMEOUT
        ivf_sub_batch(ix, ws, st, qs.at(q0), b, sp, nprobes, out.at(q0, sp.k), prof, rf, deadline);
        if (prof) g_scanned_bytes += add_ivf_profile(ws, st, b) * ivf_row_bytes(ix);
        if (widen) {
            ws->widen.ensure((size_t)b * 4);
            launch_count_below(out.at(q0, sp.k).cnt, b, sp.k, ws->widen.as<uint32_t>(), st);
            ivf_sub_batch(ix, ws, st, qs.at(q0), b, sp, np_max, out.at(q0, sp.k), false, rf, deadline,
                          ws->widen.as<uint32_t>());
        }
    }
    if (prof && ix->codes.on_host) {  // every pass's copies, the maximum_nprobes widening's included
        LGPU_CUDA(cudaMemcpyAsync(&g_streamed_bytes, ws->code_ctr.p, 8, cudaMemcpyDeviceToHost, st));
        LGPU_CUDA(cudaStreamSynchronize(st));
    }
}

// N rows of a flat handle as a search scores them: all the rows of an HBM handle, or one chunk of a host handle's
// staged in HBM.  X: the rows as stored (T = float, or __half for an fp16 handle; every path reads them as they are);
// Xop, n2: their tensor-core operand and |x|^2 (tc: present, and the handle's band is finite); ysqrt: |x| (cosine)
template <class T> struct FlatRows {
    const T *X;
    const void *Xop;
    const float *n2, *ysqrt;
    uint64_t N;
    Cols cols;
    bool tc;
};

// Whether b queries over N rows go to the l2 tensor-core path.  A row filter -- a prefilter, deleted rows -- stays on
// the tensor cores: the shortlists and thresholds are taken over the allowed rows, DESIGN.md section 3; k above
// SELECT_KMAX goes through the exact kernels: the shortlists are sized to SELECT_KMAX.
static bool flat_tc_route(bool tc, int metric, const lgpu_search_params &sp, uint32_t b, uint64_t N)
{
    return tc && tc_enabled() && metric == LGPU_L2 && !sp.has_lower && !sp.has_upper && b >= 8 && N >= 4096 &&
           sp.k <= SELECT_KMAX;
}

// the k best of the rows r for the b queries q into out (b rows of k)
template <class T>
static void flat_score(lgpu_flat *fl, Workspace *ws, cudaStream_t st, int metric, const float *q, uint32_t b,
                       const lgpu_search_params &sp, const FlatRows<T> &r, TopkOut out, RowFilter rf, bool prof)
{
    const uint64_t N = r.N, ld = (N + 3) & ~3ull;
    ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
    const float *xn = nullptr;
    if (metric == LGPU_COSINE) {
        ws->xnorm.ensure((size_t)b * 4);
        launch_row_norms(q, b, fl->dim, ws->xnorm.as<float>(), st);
        xn = ws->xnorm.as<float>();
    }
    const uint32_t kp = (uint32_t)std::min<uint64_t>(N, std::min<uint32_t>(SELECT_KMAX, std::max<uint32_t>(8 * sp.k, 256)));
    if (flat_tc_route(r.tc, metric, sp, b, N)) {
        if (N >= 262144 && !getenv("LGPU_FLAT_DENSE"))
            tc_topk_l2_filtered(ws, st, fl->num_sms, q, b, r.X, r.Xop, r.n2, fl->vec_max, fl->vec_err, N, fl->dim, r.cols,
                                sp.k, out, ws->D.as<float>(), ld, rf);
        else
            tc_topk_l2(ws, st, fl->num_sms, q, b, r.X, r.Xop, r.n2, fl->vec_max, fl->vec_err, N, fl->dim, r.cols, sp.k, kp,
                       out, ws->D.as<float>(), ld, rf);
        if (prof) g_filter_stats[1] += (uint64_t)b * N;
        return;
    }
    launch_dist_matrix(q, r.X, b, N, fl->dim, metric == LGPU_L2 ? 0 : (metric == LGPU_DOT ? 1 : 2), xn, r.ysqrt,
                       ws->D.as<float>(), ld, st);
    select_dense(ws, ws->D.as<float>(), N, ld, r.cols, b, sp, rf, out, st);
}

// The dense search of a flat or binary handle (stream_topk) reads its rows in chunks of C rows.  An HBM store is one
// resident chunk of all N rows, the queries in passes of P = bs that the budget holds the scores of.  A host store's
// chunks cross PCIe, copied into the workspace's two staging buffers on its side stream (RowStore::walk), chunk i + 1
// while chunk i is scored on the call's stream by the route an HBM handle of that chunk's rows takes.  Each chunk's
// exact top-k is merged into a running top-k per query by (distance, id).  Chunks are the outer loop: a pass over the
// column serves P queries, all B unless the budget cannot hold the running top-k of that many, in scoring groups of bs
// queries whose scores fit.  The staging buffers, the chunk's per-row terms and the running lists all count against
// the workspace budget.  timeout_ms is checked between chunks, and between the passes of an HBM store.
struct StreamShape {
    uint64_t C, nchunks;                // rows per chunk, chunks of the column
    uint32_t P, bs;                     // queries per pass, per scoring group
};
// row_b: workspace bytes per row of a staged chunk (its two staging copies and its per-row terms); row_bytes: the bytes
// of one stored row (a chunk stages at most FLAT_STAGE_BYTES of them).  A scoring group holds each query's [ldc] f32
// scores.
static StreamShape stream_shape(const RowStore &rows, uint64_t N, size_t row_b, size_t row_bytes, uint32_t B,
                                uint32_t k)
{
    const size_t budget = workspace_budget();
    StreamShape s;
    if (!rows.on_host) {
        const uint64_t ld = (N + 3) & ~3ull;
        const size_t per_q = std::max<size_t>(ld * 4, 4) + large_k_query_bytes(k);
        s.C = std::max<uint64_t>(N, 1);
        s.nchunks = 1;
        s.P = s.bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(budget / per_q, B));
        return s;
    }
    s.C = std::max<uint64_t>(1, std::min<uint64_t>(std::max<uint64_t>(N, 1),
                                                   std::min(budget / 2 / row_b, FLAT_STAGE_BYTES / row_bytes)));
    const uint64_t ldc = (s.C + 3) & ~3ull;
    s.nchunks = N ? (N + s.C - 1) / s.C : 1;
    const size_t rest = budget > s.C * row_b ? budget - s.C * row_b : 0;
    // per query: the running top-k (two buffers of two lists of k ids and distances, and their counts), and the scores
    // of a chunk
    const size_t run_q = (size_t)k * 48 + 16, score_q = ldc * 4 + large_k_query_bytes(k);
    s.P = (uint32_t)std::max<size_t>(1, std::min<size_t>(B, rest / 2 / run_q));
    const size_t left = rest > (size_t)s.P * run_q ? rest - (size_t)s.P * run_q : 0;
    s.bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(s.P, left / score_q));
    return s;
}

// The running top-k of pb queries over the chunks of a streamed column, in the workspace's run lists: list l of buffer
// r holds [pb][k] entries and [pb] counts.  Chunk 0's top-k goes to list 0 of buffer 0, chunk c > 0's to list 1 of
// buffer (c - 1) & 1, and merge(c) folds it with list 0 of that buffer into list 0 of the other, or into `out` after
// the last chunk.  A column of one chunk is scored straight into `out`.  only / gate (the fix-up of flagged queries):
// the merges touch the flagged queries alone, and return at once when none is.
struct RunningTopk {
    Workspace *ws;
    uint64_t nchunks;
    uint32_t pb, k;
    TopkOut out;
    const uint32_t *only = nullptr, *gate = nullptr;
    // room for passes of P queries
    static void reserve(Workspace *ws, uint64_t nchunks, uint32_t P, uint32_t k)
    {
        if (nchunks < 2) return;
        ws->run_ids.ensure((size_t)4 * P * k * 8); ws->run_dist.ensure((size_t)4 * P * k * 4);
        ws->run_cnt.ensure((size_t)4 * P * 4);
    }
    TopkOut run(uint64_t r, uint32_t l) const
    {
        const size_t off = (size_t)(2 * r + l) * pb;
        return {ws->run_ids.as<uint64_t>() + off * k, ws->run_dist.as<float>() + off * k, ws->run_cnt.as<uint32_t>() + off};
    }
    TopkOut dst(uint64_t c) const { return nchunks == 1 ? out : c == 0 ? run(0, 0) : run((c - 1) & 1, 1); }
    void merge(uint64_t c, cudaStream_t st) const
    {
        if (c == 0) return;
        const TopkOut a = run((c - 1) & 1, 0);
        SelectArgs m = select_cands(a.dist, a.ids, k, pb, k, c + 1 == nchunks ? out : run(c & 1, 0));
        m.ncols = 2 * (uint64_t)k; m.outer_stride = (uint64_t)pb * k; m.list_cnt = a.cnt;
        m.only = only; m.gate = gate;
        launch_select(with_scratch(ws, m), st);
    }
};

// The dense search of a flat or binary handle: its rows, N of row_bytes each, in chunks and passes of shape sh
// (stream_shape).  score(ch, p0, pb, dst) enqueues on the call's stream the k best of chunk ch (RowChunk) for the pb
// queries p0, p0 + 1, ... into dst ([pb][k], [pb]).
template <class Score>
static void stream_topk(const RowStore &rows, Workspace *ws, cudaStream_t st, size_t row_bytes, uint64_t N,
                        const StreamShape &sh, uint32_t B, uint32_t k, TopkOut out, const Deadline *deadline,
                        Score &&score)
{
    const uint64_t nchunks = sh.nchunks;
    const uint32_t P = sh.P;
    rows.reserve_stage(ws, std::max<size_t>(sh.C * row_bytes, 16));
    RunningTopk::reserve(ws, nchunks, P, k);
    // step s: pass s / nchunks, chunk s % nchunks
    auto run = [&](uint64_t s) {
        const uint32_t p0 = (uint32_t)(s / nchunks) * P;
        return RunningTopk{ws, nchunks, std::min(P, B - p0), k, out.at(p0, k)};
    };
    rows.walk(ws, st, uniform_cuts(N, sh.C), (B + P - 1) / P, [&](uint64_t r) { return r * row_bytes; }, deadline,
              [&](const RowChunk &ch) {
                  const RunningTopk r = run(ch.s);
                  score(ch, (uint32_t)(ch.s / nchunks) * P, r.pb, r.dst(ch.s % nchunks));
              },
              // after the chunk's staging buffer is released, so that the next copy does not wait for the merge
              [&](uint64_t s) { run(s).merge(s % nchunks, st); });
}

// |x| of the rows X of an HBM flat handle, built by its first cosine search
template <class T> static void flat_norms(lgpu_flat *fl, const T *X, cudaStream_t st)
{
    std::lock_guard<std::mutex> g(fl->mu);
    if (fl->has_norms) return;
    fl->ysqrt.ensure(std::max<size_t>(fl->nrows, 1) * 4, true);
    launch_row_norms(X, fl->nrows, fl->dim, fl->ysqrt.as<float>(), st);
    LGPU_CUDA(cudaStreamSynchronize(st));
    fl->has_norms = true;
}

// stream_topk, each chunk scored by flat_score: a resident chunk with the handle's per-row terms, a staged chunk with
// its terms built into the workspace
template <class T>
static void flat_search(lgpu_flat *fl, Workspace *ws, cudaStream_t st, int metric, const float *d_q, uint32_t B,
                        const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt, RowFilter rf,
                        const Deadline *deadline)
{
    const uint32_t d = fl->dim, k = sp.k;
    const size_t es = sizeof(T);
    // per row of a staged chunk: two staging copies, the bf16 operand (f32 rows), |x|^2 and |x|
    const size_t row_b = 2 * (size_t)d * es + (fl->f16 ? 0 : 2 * (size_t)d) + 8;
    const StreamShape sh = stream_shape(fl->rows, fl->nrows, row_b, (size_t)d * es, B, k);
    if (fl->rows.on_host) {
        if (fl->has_tc && !fl->f16) ws->chunk_xb.ensure(sh.C * d * 2);
        ws->chunk_n2.ensure(sh.C * 4);
        if (metric == LGPU_COSINE) ws->chunk_ysqrt.ensure(sh.C * 4);
    }
    const bool prof = profiling_enabled();
    if (prof) memset(g_filter_stats, 0, sizeof(g_filter_stats));      // [1] tensor-core distances, [3] queries
    stream_topk(fl->rows, ws, st, (size_t)d * es, fl->nrows, sh, B, k, TopkOut{d_ids, d_dist, d_cnt}, deadline,
                [&](const RowChunk &ch, uint32_t p0, uint32_t pb, TopkOut dst) {
        const T *X = static_cast<const T *>(ch.X);
        const uint64_t n = ch.r1 - ch.r0;
        FlatRows<T> rows{X, fl->f16 ? static_cast<const void *>(X) : fl->vec_b.p, fl->vec_n2.as<float>(), nullptr, n,
                         row_cols(fl, ch.r0), fl->has_tc};
        if (ch.resident) {
            if (metric == LGPU_COSINE) flat_norms(fl, X, st);
            rows.ysqrt = fl->ysqrt.as<float>();
        } else {
            // the operand only when a scoring group takes the tensor cores (the first group is the largest)
            rows.tc = flat_tc_route(fl->has_tc, metric, sp, std::min(sh.bs, pb), n);
            if (rows.tc && fl->f16) launch_f16_row_terms(X, n, d, ws->chunk_n2.as<float>(), nullptr, st);
            else if (rows.tc) launch_to_bf16(reinterpret_cast<const float *>(X), n, d, ws->chunk_xb.p, ws->chunk_n2.as<float>(), st);
            if (metric == LGPU_COSINE) launch_row_norms(X, n, d, ws->chunk_ysqrt.as<float>(), st);
            if (!fl->f16) rows.Xop = ws->chunk_xb.p;
            rows.n2 = ws->chunk_n2.as<float>();
            rows.ysqrt = ws->chunk_ysqrt.as<float>();
        }
        for (uint32_t g0 = 0; g0 < pb; g0 += sh.bs)
            flat_score(fl, ws, st, metric, d_q + (size_t)(p0 + g0) * d, std::min(sh.bs, pb - g0), sp, rows,
                       dst.at(g0, k), rf, prof);
    });
    if (prof) g_filter_stats[3] = B;
}

void flat_search_device(lgpu_flat *fl, Workspace *ws, cudaStream_t st, int metric, const float *d_q, uint32_t B,
                        const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                        RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    if (fl->f16) flat_search<__half>(fl, ws, st, metric, d_q, B, sp, d_ids, d_dist, d_cnt, rf, deadline);
    else flat_search<float>(fl, ws, st, metric, d_q, B, sp, d_ids, d_dist, d_cnt, rf, deadline);
}

// ---- binary vectors (Hamming distance) ----
// Paths, chosen from shape and request (DESIGN.md section 6):
//   SIMT dense    ham_dense_kernel -> D[b][N] -> select mode 1.  N < HAM_TC_MIN_N, or fewer than HAM_TC_MIN_B queries
//                 with N <= HAM_SAMPLE, distance_range, LGPU_NO_TENSOR_CORE=1.
//   wgmma dense   the b1 gemm_dist_kernel writes D[b][N] -> select mode 1 (N <= HAM_SAMPLE).
//   wgmma list    N > HAM_SAMPLE, any batch size: sample pass -> threshold -> filtering pass -> select mode 2 -> dense
//                 fix-up of the queries whose list overflowed (ham_topk_list).  On the H100 it beat the SIMT kernel at
//                 every batch size measured, one query included: a single query's select over a dense row of N
//                 columns runs on one SM.
// Every path computes exact integer distances, so all three return the same rows.  A row filter (prefilter, deleted
// rows) keeps the path: the selects, the sample's threshold and the filtering pass all skip the rows it leaves out.
// Candidate-list capacity of the list path.  Rows with d <= tau_q, tau_q the k-th smallest distance among the sample's
// rows, number about k N / ns (more under ties): 4x that, at least 1024, at most 16384.
static uint32_t ham_list_cap(uint32_t k, uint64_t N, uint64_t ns)
{
    const uint64_t want = 4 * (uint64_t)k * ((N + ns - 1) / ns);
    uint32_t cap = 1024;
    while (cap < want && cap < 16384) cap <<= 1;
    return cap;
}

// The per-row terms of a binary handle once rows [n0, n0 + n) are stored, at open (n0 = 0) or append (which hold the
// handle alone): the threshold sample of the list path, taken again from all nrows = n0 + n rows, every
// (nrows / HAM_SAMPLE)-th row, packed, with its popcount and its id.  A host handle's sample rows are gathered on the
// host and uploaded, so the sample is in HBM for both placements.  Enqueued on the legacy stream; the caller
// synchronises.
static void ham_sample(lgpu_binary *bx, uint64_t n0, uint64_t n)
{
    const uint64_t nrows = n0 + n;
    if (nrows <= HAM_SAMPLE) return;
    const uint64_t stride = nrows / HAM_SAMPLE;
    const uint32_t nbp = bx->nbytes_pad;
    bx->nsample = HAM_SAMPLE;
    bx->sample.ensure((size_t)HAM_SAMPLE * nbp);
    bx->sample_pop.ensure((size_t)HAM_SAMPLE * 4);
    bx->sample_ids.ensure((size_t)HAM_SAMPLE * 8);
    DevBuf gathered;
    const uint8_t *src = reinterpret_cast<const uint8_t *>(bx->rows.data());
    uint64_t src_stride = stride * nbp;
    if (bx->rows.on_host) {
        std::vector<uint8_t> h((size_t)HAM_SAMPLE * nbp);
        for (uint64_t s = 0; s < HAM_SAMPLE; s++) memcpy(h.data() + s * nbp, src + s * stride * nbp, nbp);
        gathered.ensure(h.size());
        LGPU_CUDA(cudaMemcpy(gathered.p, h.data(), h.size(), cudaMemcpyHostToDevice));
        src = gathered.as<uint8_t>();
        src_stride = nbp;
    }
    launch_ham_pack(src, src_stride, nbp, HAM_SAMPLE, bx->sample.as<uint8_t>(), nbp, bx->sample_pop.as<uint32_t>(),
                    nullptr);
    if (bx->has_ids) {
        LGPU_CUDA(cudaMemcpy2DAsync(bx->sample_ids.p, 8, bx->row_ids.p, stride * 8, 8, HAM_SAMPLE,
                                    cudaMemcpyDeviceToDevice, nullptr));
    } else {
        std::vector<uint64_t> ids(HAM_SAMPLE);
        for (uint64_t s = 0; s < HAM_SAMPLE; s++) ids[s] = s * stride;
        LGPU_CUDA(cudaMemcpy(bx->sample_ids.p, ids.data(), ids.size() * 8, cudaMemcpyHostToDevice));
    }
}

// The list path of one sub-batch (Q: padded queries [B][nbytes_pad], qpop [B]) over the rows that pass the row filter rf
// (none: every row), in four steps (ham_topk_list): the threshold (ham_list_threshold), the filtering pass over every
// row into the candidate lists, their top-k (ham_list_select), the dense fix-up of the queries whose list overflowed.
// 1. sample pass: exact distances to the sample rows, tau_q = the k-th smallest over the allowed ones (an upper bound of
// the true k-th over all rows; +inf with fewer than k).  Then the candidate counters are zeroed, and the filter of the
// filtering pass is returned: every allowed row with d <= tau_q is appended as (position, id, distance); the distance
// is final.
static GemmFilter ham_list_threshold(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *Q,
                                     const uint32_t *qpop, uint32_t B, uint32_t k, uint32_t cap, RowFilter rf)
{
    const uint64_t ns = bx->nsample, lds = (ns + 3) & ~3ull;
    launch_ham_gemm(Q, bx->sample.p, bx->sample_pop.as<uint32_t>(), qpop, B, ns, bx->nbytes_pad,
                    ws->h_sample.as<float>(), lds, bx->num_sms, st);
    SelectArgs ss = select_rows(ws->h_sample.as<float>(), ns, lds, B, k, {ws->sbound.as<uint64_t>(),
                                                                          ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>()});
    if (rf.bits) { ss.col_ids = bx->sample_ids.as<uint64_t>(); ss.allow = rf.bits; ss.allow_bits = rf.nbits; }
    launch_select(ss, st);
    launch_ham_threshold(ws->t_dist.as<float>(), ws->t_cnt.as<uint32_t>(), B, k, ws->probe_A.as<float>(), st);
    LGPU_CUDA(cudaMemsetAsync(ws->amax.p, 0, (size_t)B * 4, st));
    GemmFilter flt{};
    flt.thr = ws->probe_A.as<float>(); flt.count = ws->amax.as<uint32_t>(); flt.cand_pos = ws->t_pos.as<uint64_t>();
    flt.cand_ids = ws->t_ids.as<uint64_t>();
    flt.cap = cap; flt.cand_s = ws->t_exact.as<float>();
    flt.allow = rf.bits; flt.allow_bits = rf.nbits;
    return flt;
}

// 3. the overflow flags, and the top-k by (distance, id) of each list (an overflowed list is complete up to cap; its
// query is redone by the fix-up)
static void ham_list_select(Workspace *ws, cudaStream_t st, uint32_t B, uint32_t k, uint32_t cap, TopkOut out)
{
    launch_overflow_flags(ws->amax.as<uint32_t>(), cap, nullptr, B, ws->flags.as<uint32_t>(), st);
    SelectArgs sb = select_cands(ws->t_exact.as<float>(), ws->t_ids.as<uint64_t>(), cap, B, k, out);
    sb.ncols_q = ws->amax.as<uint32_t>();
    launch_select(sb, st);
}

// The list path of one sub-batch (above).  The one threshold tau_q bounds the k-th distance over every row, so the
// filtering GEMM runs over each chunk of the row store's walk (chunks of C rows: an HBM store's one resident chunk
// with its stored popcounts, a host store's staged chunks with theirs computed on the device, ids from the chunk's
// first row) into the sub-batch's candidate lists, whose counts add up across chunks: each row crosses PCIe once and
// the lists need no merge.  The dense fix-up of the overflowed queries differs by placement.  An HBM store: chunks of
// `bf` queries over a [bf][N] matrix; one launch lists each chunk's flagged queries, and each chunk's two launches
// return at once when its list is empty.  A host store: one list of all B flagged queries (its count gates every
// launch below), then a second walk of the chunks, each copied out of the mapped pinned memory by a gated copier,
// scored densely for the flagged queries ([B][C] matrix), and its top-k merged into a running top-k of the flagged
// queries; with nothing flagged each launch returns at once, and nothing waits on the host.
static void ham_topk_list(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *Q, const uint32_t *qpop,
                          uint32_t B, uint32_t k, uint32_t cap, uint64_t C, uint32_t bf, TopkOut out, RowFilter rf,
                          const Deadline *deadline)
{
    const uint64_t N = bx->nrows;
    const uint32_t nbp = bx->nbytes_pad;
    const std::vector<uint64_t> cut = uniform_cuts(N, C);
    // 1, 2. threshold, filtering pass
    GemmFilter flt = ham_list_threshold(bx, ws, st, Q, qpop, B, k, cap, rf);
    bx->rows.walk(ws, st, cut, [&](uint64_t r) { return r * nbp; }, deadline, [&](const RowChunk &ch) {
        const uint64_t n = ch.r1 - ch.r0;
        const uint32_t *xpop = bx->pop.as<uint32_t>();
        if (!ch.resident) {
            launch_ham_pack(static_cast<const uint8_t *>(ch.X), nbp, nbp, n, nullptr, nbp, ws->chunk_pop.as<uint32_t>(),
                            st);
            xpop = ws->chunk_pop.as<uint32_t>();
        }
        const Cols cols = row_cols(bx, ch.r0);
        flt.col_ids = cols.ids; flt.col_base = cols.base;
        launch_ham_gemm(Q, ch.X, xpop, qpop, B, n, nbp, nullptr, 0, bx->num_sms, st, &flt);
    });
    // 3. top-k of the lists
    ham_list_select(ws, st, B, k, cap, out);
    // 4. dense fix-up of the overflowed queries only
    if (!bx->rows.on_host) {
        const uint64_t ld = (N + 3) & ~3ull;
        launch_ham_flag_list(ws->flags.as<uint32_t>(), B, bf, ws->h_list.as<uint32_t>(), ws->h_cnt.as<uint32_t>(), st);
        for (uint32_t q0 = 0, c = 0; q0 < B; q0 += bf, c++) {
            const uint32_t b = std::min(bf, B - q0);
            launch_ham_dense(Q + (size_t)q0 * nbp, bx->rows.hbm.as<uint8_t>(), b, N, nbp, ws->D.as<float>(), ld,
                             bx->num_sms, st, ws->h_list.as<uint32_t>() + q0, ws->h_cnt.as<uint32_t>() + c);
            SelectArgs sc = select_rows(ws->D.as<float>(), N, ld, b, k, out.at(q0, k));
            sc.col_ids = row_cols(bx, 0).ids; sc.only = ws->flags.as<uint32_t>() + q0;
            sc.gate = ws->h_cnt.as<uint32_t>() + c;
            sc.allow = rf.bits; sc.allow_bits = rf.nbits;
            launch_select(sc, st);
        }
        return;
    }
    const uint64_t ldc = (C + 3) & ~3ull;
    launch_ham_flag_list(ws->flags.as<uint32_t>(), B, B, ws->h_list.as<uint32_t>(), ws->h_cnt.as<uint32_t>(), st);
    const uint32_t *gate = ws->h_cnt.as<uint32_t>();
    RunningTopk run{ws, cut.size() - 1, B, k, out};
    run.only = ws->flags.as<uint32_t>(); run.gate = gate;
    const uint8_t *mapped = static_cast<const uint8_t *>(bx->rows.dev());
    bx->rows.walk(ws, st, cut, 1, [&](uint64_t r) { return r * nbp; }, nullptr,
        [&](const RowChunk &ch) {
            const uint64_t n = ch.r1 - ch.r0;
            launch_ham_dense(Q, static_cast<const uint8_t *>(ch.X), B, n, nbp, ws->D.as<float>(), ldc, bx->num_sms, st,
                             ws->h_list.as<uint32_t>(), gate);
            SelectArgs sc = select_rows(ws->D.as<float>(), n, ldc, B, k, run.dst(ch.s));
            with_cols(sc, row_cols(bx, ch.r0));
            sc.only = run.only; sc.gate = gate;
            sc.allow = rf.bits; sc.allow_bits = rf.nbits;
            launch_select(sc, st);
        },
        [&](uint64_t s) { run.merge(s, st); },
        [&](uint64_t s, void *buf, cudaStream_t fs) {
            launch_mv_copy_gated(mapped + cut[s] * nbp, static_cast<uint8_t *>(buf), (cut[s + 1] - cut[s]) * nbp, gate,
                                 bx->num_sms, fs);
        });
}

// b queries (Q, qpop) against N rows X of a binary handle (ids from cols) by the dense route of an HBM handle of those
// rows, xpop their popcounts (tc only), into out: the b1 wgmma kernel (tc) or the SIMT kernel writes D [b][ld], then the
// top-k with the request's range and row filter
static void ham_dense_topk(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *Q, const uint32_t *qpop,
                           uint32_t b, const uint8_t *X, const uint32_t *xpop, uint64_t N, Cols cols, bool tc,
                           const lgpu_search_params &sp, RowFilter rf, TopkOut out)
{
    const uint64_t ld = (N + 3) & ~3ull;
    ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
    if (tc) launch_ham_gemm(Q, X, xpop, qpop, b, N, bx->nbytes_pad, ws->D.as<float>(), ld, bx->num_sms, st);
    else launch_ham_dense(Q, X, b, N, bx->nbytes_pad, ws->D.as<float>(), ld, bx->num_sms, st);
    select_dense(ws, ws->D.as<float>(), N, ld, cols, b, sp, rf, out, st);
}

// d_q: raw queries [B][nbytes] in device memory.  Both placements take the same route: the list route through
// ham_topk_list, the dense routes through stream_topk, each staged chunk scored as an HBM handle of the chunk's rows
// would score it.
void binary_search_device(lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *d_q, uint32_t B,
                          const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                          RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint64_t N = bx->nrows, ld = (N + 3) & ~3ull;
    const uint32_t nbp = bx->nbytes_pad, k = sp.k;
    const TopkOut out{d_ids, d_dist, d_cnt};
    const bool prof = profiling_enabled();
    if (prof) memset(g_filter_stats, 0, sizeof(g_filter_stats));
    ws->hq.ensure((size_t)B * nbp); ws->hq_pop.ensure((size_t)B * 4);
    launch_ham_pack(d_q, bx->nbytes, bx->nbytes, B, ws->hq.as<uint8_t>(), nbp, ws->hq_pop.as<uint32_t>(), st);
    const uint8_t *Q = ws->hq.as<uint8_t>();
    const uint32_t *qpop = ws->hq_pop.as<uint32_t>();
    const bool tc_ok = tc_enabled() && !sp.has_lower && !sp.has_upper;
    // k above SELECT_KMAX: a dense path (the list path's capacity stops at 16384 rows)
    const bool list = tc_ok && bx->nsample > 0 && k <= SELECT_KMAX;
    const bool tc = list || (tc_ok && B >= HAM_TC_MIN_B && N >= HAM_TC_MIN_N);
    const size_t budget = workspace_budget();
    uint64_t tc_dists = 0;          // profiling: distances computed on the tensor cores
    if (list) {
        // Workspace, all inside LGPU_WS_BYTES.  An HBM handle: the fix-up matrix [bf][N] gets at most half the budget
        // and 1 GiB (it is rarely used); the rest is split into sub-batches of bs queries, each holding its sample
        // scores [bs][ns] and candidate lists [bs][cap] (at the default 8 GiB, 1024 queries x 10M rows run as one
        // sub-batch).  A host handle: chunks of C rows take the two staging copies and popcounts of at most half the
        // budget; each query of a sub-batch adds to the above its running top-k and its row of the fix-up matrix
        // [bs][C].
        const uint64_t ns = bx->nsample, lds = (ns + 3) & ~3ull;
        const uint32_t cap = ham_list_cap(k, N, ns);
        const size_t per_q0 = lds * 4 + (size_t)cap * 20 + (size_t)k * 12 + 16;
        uint32_t bf = 0, bs = 0;
        uint64_t C = N;
        if (bx->rows.on_host) {
            const size_t row_b = 2 * (size_t)nbp + 4;
            C = std::max<uint64_t>(1, std::min<uint64_t>(N, std::min(budget / 2 / row_b, FLAT_STAGE_BYTES / nbp)));
            const uint64_t ldc = (C + 3) & ~3ull;
            const size_t per_q = per_q0 + (size_t)k * 48 + 16 + ldc * 4;
            const size_t left = budget > C * row_b ? budget - C * row_b : 0;
            bs = bf = (uint32_t)std::max<size_t>(1, std::min<size_t>(left / per_q, B));
            bx->rows.reserve_stage(ws, C * nbp);
            ws->chunk_pop.ensure(C * 4);
            RunningTopk::reserve(ws, (N + C - 1) / C, bs, k);
            ws->D.ensure((size_t)bs * ldc * 4);
        } else {
            bf = (uint32_t)std::max<size_t>(1, std::min<size_t>(std::min<size_t>(budget / 2, (size_t)1 << 30) / (ld * 4), B));
            const size_t left = budget > (size_t)bf * ld * 4 ? budget - (size_t)bf * ld * 4 : 0;
            bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(left / per_q0, B));
            ws->D.ensure((size_t)bf * ld * 4);
        }
        ws->h_sample.ensure((size_t)bs * lds * 4);
        ws->t_dist.ensure((size_t)bs * k * 4); ws->sbound.ensure((size_t)bs * k * 8); ws->t_cnt.ensure((size_t)bs * 4);
        ws->probe_A.ensure((size_t)bs * 4); ws->amax.ensure((size_t)bs * 4); ws->flags.ensure((size_t)bs * 4);
        ws->t_pos.ensure((size_t)bs * cap * 8); ws->t_ids.ensure((size_t)bs * cap * 8);
        ws->t_exact.ensure((size_t)bs * cap * 4);
        ws->h_list.ensure((size_t)bs * 4);
        ws->h_cnt.ensure((size_t)((bs + bf - 1) / bf) * 4);
        for (uint32_t q0 = 0; q0 < B; q0 += bs) {
            const uint32_t b = std::min(bs, B - q0);
            if (deadline && q0 > 0) deadline->wait(st, ws->ev[7]);
            ham_topk_list(bx, ws, st, Q + (size_t)q0 * nbp, qpop + q0, b, k, cap, C, bf, out.at(q0, k), rf, deadline);
            if (prof) {             // [0] list appends, [2] queries redone densely (over every sub-batch)
                std::vector<uint32_t> cnt(b), fl(b);
                LGPU_CUDA(cudaMemcpyAsync(cnt.data(), ws->amax.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaMemcpyAsync(fl.data(), ws->flags.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
                LGPU_CUDA(cudaStreamSynchronize(st));
                for (uint32_t q = 0; q < b; q++) { g_filter_stats[0] += cnt[q]; g_filter_stats[2] += fl[q] ? 1 : 0; }
            }
        }
        tc_dists = (uint64_t)B * (N + ns);
    } else {
        // per row of a staged chunk: two staging copies and its popcount
        const StreamShape sh = stream_shape(bx->rows, N, 2 * (size_t)nbp + 4, nbp, B, k);
        if (bx->rows.on_host) ws->chunk_pop.ensure(sh.C * 4);
        stream_topk(bx->rows, ws, st, nbp, N, sh, B, k, out, deadline,
                    [&](const RowChunk &ch, uint32_t p0, uint32_t pb, TopkOut dst) {
            const uint8_t *X = static_cast<const uint8_t *>(ch.X);
            const uint64_t n = ch.r1 - ch.r0;
            // The two placements choose the tensor cores differently: the resident chunk from the call's B (tc), a
            // staged chunk per scoring group.  Both choices are kept as they are; making them agree changes which
            // kernels a call launches.
            auto group_tc = [&](uint32_t b) {
                return ch.resident ? tc : tc_ok && b >= HAM_TC_MIN_B && n >= HAM_TC_MIN_N;
            };
            const uint32_t *xpop = bx->pop.as<uint32_t>();
            if (!ch.resident) {
                // the popcounts only when a scoring group takes the tensor cores (the first group is the largest)
                if (group_tc(std::min(sh.bs, pb)))
                    launch_ham_pack(X, nbp, nbp, n, nullptr, nbp, ws->chunk_pop.as<uint32_t>(), st);
                xpop = ws->chunk_pop.as<uint32_t>();
            }
            for (uint32_t g0 = 0; g0 < pb; g0 += sh.bs) {
                const uint32_t b = std::min(sh.bs, pb - g0);
                ham_dense_topk(bx, ws, st, Q + (size_t)(p0 + g0) * nbp, qpop + p0 + g0, b, X, xpop, n,
                               row_cols(bx, ch.r0), group_tc(b), sp, rf, dst.at(g0, k));
                if (group_tc(b)) tc_dists += (uint64_t)b * n;
            }
        });
    }
    if (prof) {                     // [1] distances computed on the tensor cores, [3] queries
        LGPU_CUDA(cudaStreamSynchronize(st));
        g_filter_stats[1] = tc_dists;
        g_filter_stats[3] = B;
    }
}

// ---- multivector columns (late interaction: sum over the query's vectors of the min cosine distance) ----
// Limits of one call: a query holds 1..MV_MAX_NQ vectors, a row 0..MV_MAX_ROW, a vector at most MV_MAX_DIM components.
constexpr uint32_t MV_MAX_NQ = 4096;
constexpr uint64_t MV_MAX_ROW = (uint64_t)1 << 20;
constexpr uint32_t MV_MAX_DIM = 65536;

// Paths (multivec.cu, DESIGN.md section 6), chosen per call:
//   tensor cores  the F16MaxSim gemm_dist_kernel scores fp16 copies of the normalised vectors (an fp16 handle: the
//                 F16RowMaxSim policy, fp16 normalised queries against the stored vectors, each similarity scaled by
//                 1 / |v|) and keeps the largest similarity per (query vector, row); approximate distances -> the k-th
//                 smallest (select mode 1) -> every row within 2 E_q of it (mv_band, mv_band_f16) -> exact re-score of
//                 those rows (dist.cu) -> select mode 2; a query whose list overflowed or that holds a zero /
//                 non-finite vector is redone by the exact path below in the same stream (flags / gate: nothing runs
//                 when no query is flagged).  Taken when the column holds at least MV_TC_MIN_T vectors (all of them
//                 finite and non-zero), dim is a multiple of 8, there is no distance_range, LGPU_NO_TENSOR_CORE is
//                 not set and one query's scores fit the workspace.  Under a row filter (a prefilter, deleted rows:
//                 the RowFilter of the call) the k-th select sees the allowed rows only and mv_admit_kernel admits
//                 only allowed rows, so a filtered row never costs a shortlist slot or a re-score.  The band is
//                 unchanged: leaving rows out of the select can only raise the k-th approximate distance tau, and
//                 the k allowed rows with A <= tau have D <= tau + E, so the allowed exact k-th distance D_k is at
//                 most tau + E and every allowed row of the exact top-k has A <= D + E <= D_k + E <= tau + 2 E.
//                 With fewer than k allowed rows the select returns fewer than k, tau is +inf and every
//                 allowed row is admitted; a list that overflows goes to the fix-up, which filters as the exact
//                 route does.
//   exact         for every sub-batch of queries, blocks of consecutive query vectors against chunks of whole rows --
//                 dist_matrix_kernel (cosine, lance order) -> per-row minimum -> in-order running sum into D[b][N] --
//                 then select mode 1 (distance_range, prefilter, (_distance, _rowid) order, NaN dropped).
// Workspace stays inside LGPU_WS_BYTES.
constexpr uint64_t MV_TC_MIN_T = 65536;   // stored vectors from which the tensor-core path runs (not measured)

// the exact distances of queries [qa, qb) to rows [ra, rb) into D[b - qa][ra..rb) (only / vflags / gate: the fix-up of
// flagged queries).  X holds the vectors of those rows in the row type, from the first vector of row ra (a host
// handle's staged chunk); the order of the additions per row depends only on the blocking of the query vectors, not
// on [ra, rb).
static void mv_exact_dense(lgpu_multivec *mv, Workspace *ws, cudaStream_t st, const float *d_q, const uint32_t *h_qoff,
                           uint32_t qa, uint32_t qb, float *D, uint64_t ld, const void *X, uint64_t ra, uint64_t rb,
                           const uint32_t *only = nullptr, const uint32_t *vflags = nullptr,
                           const uint32_t *gate = nullptr)
{
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
        for (uint64_t r0 = ra; r0 < rb;) {
            uint64_t r1 = r0 + 1;
            while (r1 < rb && (off[r1 + 1] - off[r0]) + (r1 + 1 - r0) <= cap) r1++;
            const uint64_t span = off[r1] - off[r0], ldP = (span + 3) & ~3ull;
            const uint32_t nr = (uint32_t)(r1 - r0);
            ws->mv_P.ensure(std::max<size_t>((size_t)nqv * ldP, 4) * 4);
            ws->mv_M.ensure((size_t)nqv * nr * 4);
            auto dist = [&](auto *x) {
                launch_dist_matrix(d_q + (size_t)i0 * dim, x + (size_t)(off[r0] - off[ra]) * dim, nqv, span, dim, 2,
                                   ws->xnorm.as<float>() + i0, mv->ysqrt.as<float>() + off[r0], ws->mv_P.as<float>(),
                                   ldP, st, vflags ? vflags + (i0 - h_qoff[qa]) : nullptr, gate);
            };
            if (span) {
                if (mv->f16) dist(static_cast<const __half *>(X));
                else dist(static_cast<const float *>(X));
            }
            launch_mv_rowmin(ws->mv_P.as<float>(), ldP, nqv, mv->offsets.as<uint64_t>(), r0, nr, ws->mv_M.as<float>(),
                             nr, mv->num_sms, st, gate);
            launch_mv_rowsum(ws->mv_M.as<float>(), nr, ws->mv_qoff.as<uint32_t>(), blo, bhi, qa, i0, i1, nr, D, ld, r0,
                             mv->num_sms, st, only, gate);
            r0 = r1;
        }
    }
}

// ---- a host multivector handle (RowStore::on_host): its row data crosses PCIe in chunks of whole rows ----
// The bytes of one staging buffer: FLAT_STAGE_BYTES, or an eighth of the budget when that is smaller, and never less
// than the longest row's vectors in the row type.  Two such buffers must fit the budget (mv_check_stage, before any
// device work).
static size_t mv_elem_bytes(const lgpu_multivec *mv) { return mv->f16 ? 2 : 4; }

static size_t mv_stage_bytes(const lgpu_multivec *mv)
{
    const size_t longest = (size_t)mv->max_row * mv->dim * mv_elem_bytes(mv);
    return std::max<size_t>(std::min(FLAT_STAGE_BYTES, workspace_budget() / 8), std::max<size_t>(longest, 16));
}

static void mv_check_stage(const lgpu_multivec *mv)
{
    const size_t longest = (size_t)mv->max_row * mv->dim * mv_elem_bytes(mv);
    if (mv->rows.on_host && 2 * longest > workspace_budget()) {
        set_error("a multivector row of " + std::to_string(mv->max_row) + " vectors (" + std::to_string(longest) +
                  " bytes) does not fit twice in the workspace budget (LGPU_WS_BYTES) that streams a host handle");
        throw Failure{LGPU_OOM};
    }
}

// the rows of each chunk: bounds cut[c]..cut[c + 1], whole rows of at most `cap_vec` vectors in all (a longer row
// is a chunk of its own)
static std::vector<uint64_t> mv_chunks(const lgpu_multivec *mv, uint64_t cap_vec)
{
    const uint64_t *off = mv->h_offsets.data();
    std::vector<uint64_t> cut{0};
    for (uint64_t r = 0; r < mv->nrows;) {
        uint64_t r1 = r + 1;
        while (r1 < mv->nrows && off[r1 + 1] - off[r] <= cap_vec) r1++;
        cut.push_back(r1);
        r = r1;
    }
    return cut;
}

// h_qoff: HOST [B+1] offsets of each query's vectors in d_q (validated by the caller).
// Both routes (above) read the row data in chunks of whole rows, bounds cut[c]..cut[c + 1]: an HBM handle's one
// resident chunk [0, N); a host handle's mv_chunks of one staging buffer each, streamed through Workspace::stage in
// every sub-batch, so each vector crosses PCIe once per sub-batch.  The tensor-core GEMM keeps chunk-local keys
// (row_base = the chunk's first row) and fills the chunk's columns of A.  A host handle re-scores the shortlist from the
// pinned vectors, and its fix-up walks the chunks again with a copier kernel that returns at once when the gate is 0:
// no host synchronisation decides anything.  The vectors are in the row type (es bytes per element); an
// fp16 handle's vectors are also its tensor-core operand, so both routes stream the same 2-byte rows.  Half the budget
// goes to the distance blocks of mv_exact_dense; the other half, less a host handle's two staging buffers, is `left`.
void multivec_search_device(lgpu_multivec *mv, Workspace *ws, cudaStream_t st, const float *d_q, const uint32_t *h_qoff,
                            uint32_t B, const lgpu_search_params &sp, uint64_t *d_ids, float *d_dist, uint32_t *d_cnt,
                            RowFilter rf = RowFilter(), const Deadline *deadline = nullptr)
{
    const uint64_t N = mv->nrows, ld = (N + 3) & ~3ull;
    const uint32_t dim = mv->dim, k = sp.k, Tq = h_qoff[B];
    const uint64_t *off = mv->h_offsets.data();
    const uint64_t *ids = mv->has_ids ? mv->row_ids.as<uint64_t>() : nullptr;
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
    const bool tc = mv->tc_ok && tc_enabled() && !sp.has_lower && !sp.has_upper && k <= SELECT_KMAX &&
                    (size_t)(max_nq + 1) * ld * 4 <= quarter;
    const size_t S = mv->rows.on_host ? mv_stage_bytes(mv) : 0, left = budget / 2 > 2 * S ? budget / 2 - 2 * S : 0;
    mv->rows.reserve_stage(ws, S);
    // the chunks of a copy of the vectors at `vb` bytes each, and the byte of each row's first vector in it
    auto chunks = [&](size_t vb) { return S ? mv_chunks(mv, S / (dim * vb)) : std::vector<uint64_t>{0, N}; };
    auto at = [&](size_t vb) { return [&, vb](uint64_t r) { return off[r] * vb; }; };
    const size_t es = mv_elem_bytes(mv);
    const std::vector<uint64_t> cutv = chunks(es);                  // chunks of the vectors in the row type
    if (!tc) {
        const size_t per_q = std::max<size_t>(ld * 4, 4) + large_k_query_bytes(k);
        const uint32_t bs = (uint32_t)std::max<size_t>(1, std::min<size_t>(left / per_q, B));
        for (uint32_t qa = 0; qa < B; qa += bs) {
            const uint32_t qb = std::min(B, qa + bs), b = qb - qa;
            if (deadline && qa > 0) deadline->wait(st, ws->ev[7]);
            ws->D.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
            mv->rows.walk(ws, st, cutv, at((size_t)dim * es), deadline, [&](const RowChunk &ch) {
                mv_exact_dense(mv, ws, st, d_q, h_qoff, qa, qb, ws->D.as<float>(), ld, ch.X, ch.r0, ch.r1);
            });
            select_dense(ws, ws->D.as<float>(), N, ld, ids, b, sp, rf, out.at(qa, k), st);
        }
    } else {
        // fp16 normalised queries (and the queries holding a bad vector)
        ws->mv_qh.ensure(std::max<size_t>((size_t)Tq * dim * 2, 16));
        ws->mv_qbad.ensure(std::max<size_t>(Tq, 1) * 4);
        launch_mv_normalize_f16(d_q, Tq, dim, ws->mv_qh.p, ws->mv_qbad.as<uint32_t>(), st);
        uint32_t cap = 1024;
        while (cap < 8 * k && cap < 16384) cap <<= 1;
        const std::vector<uint64_t> cut16 = chunks(2);
        uint64_t R = 1;                                   // the most rows of an operand chunk
        for (size_t c = 0; c + 1 < cut16.size(); c++) R = std::max(R, cut16[c + 1] - cut16[c]);
        const uint64_t ldR = (R + 3) & ~3ull;
        // may queries [qa, qb] form one sub-batch?  An HBM handle: if their keys M [vectors][ld] u32 and approximate
        // distances A [queries][ld] f32 take a quarter of the budget each.  A host handle: if their per-query state
        // (A, the k-th select, threshold, counters, the shortlist and its exact scores) and per query vector the keys
        // of one chunk fit `left`.
        const size_t per_q = ld * 4 + (size_t)k * 12 + (size_t)cap * 16 + 32, per_v = ldR * 4 + 4;
        auto fits = [&](uint32_t qa, uint32_t qb) {
            const size_t nq = qb + 1 - qa, nv = h_qoff[qb + 1] - h_qoff[qa];
            return mv->rows.on_host ? nq * per_q + nv * per_v <= left : nv * ld * 4 <= quarter && nq * ld * 4 <= quarter;
        };
        const void *V = mv->rows.dev();                                 // the vectors, for the re-score
        const RowStore &op = mv->f16 ? mv->rows : mv->ops;             // the operand
        for (uint32_t qa = 0; qa < B;) {
            uint32_t qb = qa + 1;
            while (qb < B && fits(qa, qb)) qb++;
            if (deadline && qa > 0) deadline->wait(st, ws->ev[7]);
            const uint32_t b = qb - qa, va = h_qoff[qa], nqv = h_qoff[qb] - va;
            ws->mv_Mk.ensure((size_t)nqv * ldR * 4);
            ws->mv_A.ensure(std::max<size_t>((size_t)b * ld, 4) * 4);
            ws->mv_kd.ensure((size_t)b * k * 4); ws->mv_ki.ensure((size_t)b * k * 8); ws->mv_kc.ensure((size_t)b * 4);
            ws->mv_thr.ensure((size_t)b * 4); ws->mv_cnt.ensure((size_t)b * 4); ws->mv_cand.ensure((size_t)b * cap * 4);
            ws->mv_flags.ensure((size_t)b * 4); ws->mv_vflags.ensure((size_t)nqv * 4); ws->mv_gate.ensure(16);
            ws->mv_ex.ensure((size_t)b * cap * 4); ws->mv_exid.ensure((size_t)b * cap * 8);
            float *A = ws->mv_A.as<float>();
            op.walk(ws, st, cut16, at((size_t)dim * 2), deadline, [&](const RowChunk &ch) {
                const uint64_t ra = ch.r0, rb = ch.r1, span = off[rb] - off[ra], ldc = (rb - ra + 3) & ~3ull;
                LGPU_CUDA(cudaMemsetAsync(ws->mv_Mk.p, 0, (size_t)nqv * ldc * 4, st));
                MaxSimOut mo{};
                mo.col_row = mv->col_row.as<uint32_t>() + off[ra]; mo.M = ws->mv_Mk.as<uint32_t>(); mo.ldM = ldc;
                mo.row_base = (uint32_t)ra; mo.vnorm = mv->ysqrt.as<float>() + off[ra];
                launch_maxsim_gemm(ws->mv_qh.as<char>() + (size_t)va * dim * 2, ch.X, nqv, span, dim, mo, mv->f16,
                                   mv->num_sms, st);
                launch_mv_approx_sum(ws->mv_Mk.as<uint32_t>(), ldc, ws->mv_qoff.as<uint32_t>(), qa, qb, va, rb - ra,
                                     A + ra, ld, mv->num_sms, st);
            });
            // the k-th smallest approximate distance of each query over the allowed rows (A's column r is row r of
            // the handle in both placements, so its id is ids[r], or r)
            SelectArgs sk = select_rows(A, N, ld, b, k, {ws->mv_ki.as<uint64_t>(), ws->mv_kd.as<float>(),
                                                         ws->mv_kc.as<uint32_t>()});
            if (rf.bits) { with_cols(sk, ids); sk.allow = rf.bits; sk.allow_bits = rf.nbits; }
            launch_select(sk, st);
            launch_mv_threshold(ws->mv_kd.as<float>(), ws->mv_kc.as<uint32_t>(), ws->mv_qoff.as<uint32_t>(), qa, b, k, dim,
                                mv->f16, ws->mv_thr.as<float>(), st);
            LGPU_CUDA(cudaMemsetAsync(ws->mv_cnt.p, 0, (size_t)b * 4, st));
            launch_mv_admit(A, ld, b, N, ws->mv_thr.as<float>(), cap, ws->mv_cnt.as<uint32_t>(),
                            ws->mv_cand.as<uint32_t>(), ids, rf.bits, rf.nbits, st);
            launch_mv_flags(ws->mv_cnt.as<uint32_t>(), cap, ws->mv_qbad.as<uint32_t>(), ws->mv_qoff.as<uint32_t>(), qa, b,
                            ws->mv_flags.as<uint32_t>(), ws->mv_vflags.as<uint32_t>(), ws->mv_gate.as<uint32_t>(), st);
            auto rescore = [&](auto *v) {
                if (mv->rows.on_host)
                    launch_mv_rescore_host(d_q, ws->mv_qoff.as<uint32_t>(), qa, ws->xnorm.as<float>(), v,
                                           mv->ysqrt.as<float>(), mv->offsets.as<uint64_t>(), ids, dim, b,
                                           ws->mv_cand.as<uint32_t>(), ws->mv_cnt.as<uint32_t>(), cap,
                                           ws->mv_ex.as<float>(), ws->mv_exid.as<uint64_t>(), mv->num_sms, st);
                else
                    launch_mv_rescore(d_q, ws->mv_qoff.as<uint32_t>(), qa, ws->xnorm.as<float>(), v, mv->ysqrt.as<float>(),
                                      mv->offsets.as<uint64_t>(), ids, dim, b, ws->mv_cand.as<uint32_t>(),
                                      ws->mv_cnt.as<uint32_t>(), cap, ws->mv_ex.as<float>(), ws->mv_exid.as<uint64_t>(),
                                      st);
            };
            if (mv->f16) rescore(static_cast<const __half *>(V));
            else rescore(static_cast<const float *>(V));
            launch_select(select_cands(ws->mv_ex.as<float>(), ws->mv_exid.as<uint64_t>(), cap, b, k, out.at(qa, k)), st);
            // exact fix-up of the flagged queries into A (free again: it holds their exact distances).  A host handle's
            // chunks are copied by a gated copier; with no query flagged, every launch returns at once
            const uint32_t *gate = ws->mv_gate.as<uint32_t>();
            mv->rows.walk(ws, st, cutv, at((size_t)dim * es), nullptr,
                [&](const RowChunk &ch) {
                    mv_exact_dense(mv, ws, st, d_q, h_qoff, qa, qb, A, ld, ch.X, ch.r0, ch.r1,
                                   ws->mv_flags.as<uint32_t>(), ws->mv_vflags.as<uint32_t>(), gate);
                },
                [&](uint64_t s, void *buf, cudaStream_t fs) {
                    const uint64_t j0 = off[cutv[s]], n = (off[cutv[s + 1]] - j0) * dim;
                    if (mv->f16)
                        launch_mv_copy_gated(static_cast<const __half *>(V) + j0 * dim, static_cast<__half *>(buf), n,
                                             gate, mv->num_sms, fs);
                    else
                        launch_mv_copy_gated(static_cast<const float *>(V) + j0 * dim, static_cast<float *>(buf), n,
                                             gate, mv->num_sms, fs);
                });
            SelectArgs sc = select_rows(A, N, ld, b, k, out.at(qa, k));
            sc.col_ids = ids;
            sc.only = ws->mv_flags.as<uint32_t>(); sc.gate = gate;
            sc.allow = rf.bits; sc.allow_bits = rf.nbits;
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
    // tags are below 2^16; ef in bits 16..31 (values above 0xffff share a key: IVF_HNSW_SQ refuses ef above
    // LGPU_HNSW_EF_MAX and every other kind ignores ef)
    key[0] = tag ^ ((uint64_t)std::min<uint32_t>(p.ef, 0xffffu) << 16) ^ ((uint64_t)B << 32);
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

// The row filter of a call on a handle, given the call's own (rf, none when rf.bits is null): rf itself when nothing
// was deleted; the handle's live bitmap when the call has none (no copy, no launch); else their AND, made on `st` into
// the workspace once per call and charged to the call's workspace budget (WsCharge).  A row passes the result exactly
// when it passes rf and was not deleted.
static RowFilter with_live(Workspace *ws, cudaStream_t st, RowFilter rf, const RowLive &live)
{
    if (!live.active) return rf;
    const uint32_t *lb = static_cast<const uint32_t *>(live.bits.p);
    if (!rf.bits) return {lb, live.id_bound};
    const uint64_t nbits = std::min(rf.nbits, live.id_bound), words = (nbits + 31) / 32;
    ws->live_and.ensure(std::max<size_t>(words, 1) * 4);
    g_ws_charged += std::max<size_t>(words, 1) * 4;
    launch_rowmask_and(rf.bits, lb, words, ws->live_and.as<uint32_t>(), st);
    return {ws->live_and.as<uint32_t>(), nbits};
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

// Whether the host route may capture a handle's calls into a CUDA graph: not a handle whose rows are on the host,
// whose calls stream from pinned memory that an append moves, on a side stream (RowStore::walk), nor an IVF index whose
// codes are on the host, whose calls stage them on a side stream too (scan_codes) and check timeout_ms between chunks
template <class H> static bool graph_capturable(const H *h)
{
    if constexpr (std::is_base_of_v<lgpu_rows, H>) return !h->rows.on_host;
    else if constexpr (std::is_base_of_v<lgpu_index, H>) return !h->codes.on_host;
    else return true;
}

// The sequence of every search entry point: resolve the handle; the kind's own checks, `check(h)`, which return how
// many query elements (T) the call reads; the bitmap of a filtered call; nothing more for B == 0; the device; then
// the kind's `search(h, ws, st, d_q, B, params, d_ids, d_dist, d_cnt, rf, deadline)` on a workspace leased for the
// caller's stream, or staged through host_submit.
template <class H, class T, class Check, class Search>
int search_call(H *hp, const Route &r, const T *queries, uint32_t B, const lgpu_search_params *p,
                uint64_t *ids, float *dist, uint32_t *cnt, Check &&check, Search &&search)
{
    return guarded([&] {
        const WsCharge charge;
        HandleRef<H> h(hp);
        const size_t q_elems = check(h.h);
        if (r.via == Route::FILTERED) LGPU_REQUIRE(r.allow != nullptr || r.allow_bits == 0, "allow bitmap is null");
        if (B == 0) return;
        require_device(h->device);
        if (r.via == Route::DEVICE) {
            WsLease lease(h->pool, (cudaStream_t)r.stream, true);
            search(h.h, lease.ws, lease.st, queries, B, *p, ids, dist, cnt,
                   with_live(lease.ws, lease.st, RowFilter(), h->live), nullptr);
            return;
        }
        uint64_t key[4];
        const bool graph = r.graph_tag && graph_capturable(h.h);
        if (graph) make_key(key, r.graph_tag, B, *p);
        host_call(h->pool, queries, q_elems, B, p->k, ids, dist, cnt, graph ? key : nullptr, p->timeout_ms,
                  [&](Workspace *ws, cudaStream_t st, const T *dq, uint64_t *di, float *dd, uint32_t *dc,
                      const Deadline &dl) {
                      const RowFilter rf = r.via == Route::FILTERED ? upload_allow(ws, st, r.allow, r.allow_bits)
                                                                    : RowFilter();
                      search(h.h, ws, st, dq, B, *p, di, dd, dc, with_live(ws, st, rf, h->live), &dl);
                  });
    });
}

// what the flat, binary and multivector opens share: the device's SM count and the optional row ids
static void open_rows(lgpu_rows *h, const uint64_t *row_ids, uint64_t nrows)
{
    cudaDeviceProp prop;
    LGPU_CUDA(cudaGetDeviceProperties(&prop, h->device));
    h->num_sms = prop.multiProcessorCount;
    if (row_ids && nrows) {
        h->row_ids.ensure((size_t)nrows * 8, true);
        LGPU_CUDA(cudaMemcpy(h->row_ids.p, row_ids, (size_t)nrows * 8, cudaMemcpyHostToDevice));
        h->has_ids = true;
    }
}

// The byte accounting of a flat, binary or multivector handle (lgpu_*_device_bytes, lgpu_*_host_bytes): its row stores,
// ids and live bitmap, and its kind's per-row buffers in HBM
static uint64_t sum_bytes(std::initializer_list<const DevBuf *> bufs)
{
    uint64_t n = 0;
    for (const DevBuf *b : bufs) n += b->bytes;
    return n;
}
static uint64_t own_device_bytes(const lgpu_flat *fl) { return sum_bytes({&fl->ysqrt, &fl->vec_b, &fl->vec_n2}); }
static uint64_t own_device_bytes(const lgpu_binary *bx)
{
    return sum_bytes({&bx->pop, &bx->sample, &bx->sample_pop, &bx->sample_ids});
}
static uint64_t own_device_bytes(const lgpu_multivec *mv)
{
    return sum_bytes({&mv->ysqrt, &mv->offsets, &mv->col_row}) + mv->ops.device_bytes();
}
static uint64_t own_host_bytes(const lgpu_rows *) { return 0; }
static uint64_t own_host_bytes(const lgpu_multivec *mv) { return mv->ops.host_bytes(); }
template <class H> static int rows_device_bytes(const H *hp, uint64_t *bytes)
{
    return guarded([&] {
        HandleRef<H> h(const_cast<H *>(hp));
        LGPU_REQUIRE(bytes != nullptr, "null argument");
        *bytes = h->rows.device_bytes() + h->row_ids.bytes + h->live.bits.bytes + own_device_bytes(h.h);
    });
}
// lgpu_*_host_bytes, lgpu_*_code_bytes: of(h) gives a handle's row store (null: it keeps none, LGPU_VECTORS_NONE) and
// the pinned bytes it holds beside it; the call reports the store's pinned bytes plus those, and where the store is
template <class H, class Of> static int host_placement(const H *hp, uint64_t *bytes, int *placement, Of &&of)
{
    return guarded([&] {
        LGPU_REQUIRE(bytes || placement, "null argument");
        HandleRef<H> h(const_cast<H *>(hp));
        const auto [s, extra] = of(h.h);
        if (bytes) *bytes = (s ? s->host_bytes() : 0) + extra;
        if (placement) *placement = !s ? LGPU_VECTORS_NONE : s->on_host ? LGPU_VECTORS_HOST : LGPU_VECTORS_HBM;
    });
}
template <class H> static int rows_host_bytes(const H *hp, uint64_t *bytes, int *placement)
{
    return host_placement(hp, bytes, placement,
                          [](const H *h) { return std::pair<const RowStore *, uint64_t>{&h->rows, own_host_bytes(h)}; });
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

// copy a host array into a device buffer of at least 16 bytes, on the legacy stream
static void upload(DevBuf &b, const void *src, size_t bytes)
{
    b.ensure(std::max<size_t>(bytes, 16));
    if (bytes) LGPU_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, nullptr));
}

// The partition arrays every IVF index holds (part_n, part_npad, part_off, row_ids, code_base, the host-side tile bound
// max_nrb and pad_prefix), uploaded on the legacy stream; `rows_tile` is the scan's tile height.  code_base: the byte
// offset of each partition's codes, which the regroup copies into the tile descriptors -- padded_code_base for the PQ
// layouts, zeros for the row-major kinds (sq, rq, ham), whose scans address rows by part_off.
template <class Desc>
static void open_ivf_partitions(lgpu_index *ix, const Desc *d, uint32_t rows_tile, const std::vector<uint64_t> &code_base)
{
    const uint32_t nlist = d->nlist;
    ix->device = d->device;
    cudaDeviceProp prop;
    LGPU_CUDA(cudaGetDeviceProperties(&prop, ix->device));
    ix->num_sms = prop.multiProcessorCount;
    ix->nlist = nlist; ix->nrows = d->nrows;
    std::vector<uint32_t> part_n(nlist), part_npad(nlist);
    std::vector<uint64_t> pads(nlist);
    for (uint32_t p = 0; p < nlist; p++) {
        const uint32_t n = (uint32_t)(d->part_offsets[p + 1] - d->part_offsets[p]);
        part_n[p] = n; part_npad[p] = (n + 31u) & ~31u;
        pads[p] = (n + 3ull) & ~3ull;
        ix->max_nrb = std::max(ix->max_nrb, scan_nrb(n, rows_tile));
    }
    ix->h_part_n = part_n;
    std::sort(pads.begin(), pads.end(), std::greater<uint64_t>());
    ix->pad_prefix.assign(nlist + 1, 0);
    for (uint32_t p = 0; p < nlist; p++) ix->pad_prefix[p + 1] = ix->pad_prefix[p] + pads[p];
    upload(ix->part_n, part_n.data(), (size_t)nlist * 4);
    upload(ix->part_npad, part_npad.data(), (size_t)nlist * 4);
    upload(ix->part_off, d->part_offsets, (size_t)(nlist + 1) * 8);
    upload(ix->row_ids, d->row_ids, (size_t)d->nrows * 8);
    upload(ix->code_base, code_base.data(), (size_t)nlist * 8);
    LGPU_CUDA(cudaStreamSynchronize(nullptr));
}

// What the float IVF indexes add, uploaded on the legacy stream: centroids (and their bf16 copy for the tensor-core
// coarse step).  The optional raw vectors are placed last, by place_vectors, once the rest of the index is in HBM.
template <class Desc>
static void open_ivf_common(lgpu_index *ix, const Desc *d, uint32_t rows_tile, const std::vector<uint64_t> &code_base)
{
    const uint32_t dim = d->dim, nlist = d->nlist;
    ix->dim = dim; ix->metric = d->metric;
    cudaStream_t st = nullptr;
    upload(ix->centroids, d->centroids, (size_t)nlist * dim * 4);
    open_ivf_partitions(ix, d, rows_tile, code_base);
    if (gemm_shape_supported(dim) && d->metric != LGPU_DOT) {
        LGPU_CUDA(cudaStreamSynchronize(st));
        const bool finite =
            prepare_tc_operand(ix->centroids.as<float>(), nlist, dim, ix->cent_b, ix->cent_n2, ix->cent_max, ix->cent_err, st);
        if (!finite) { ix->cent_b.reset(); ix->cent_n2.reset(); }     // never read: the exact coarse kernels serve it
        if (finite && nlist >= 1024) {
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
        }
        ix->has_tc = finite;                   // a non-finite centroid: the exact coarse kernels
    }
    LGPU_CUDA(cudaStreamSynchronize(st));
}

// IVF_SQ stored rows: dim zero-padded to the scan's K step
static uint32_t sq_dim_pad(uint32_t dim) { return (uint32_t)round_up64(dim, SQ_K_CHUNK); }

// codes [n][dim] (host) -> dst [n][dim_pad] (device, zero padding) and xx[r] = sum of row r's squared codes, on the
// legacy stream
static void fill_sq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, uint8_t *dst, uint32_t *xx)
{
    const uint32_t dim_pad = sq_dim_pad(dim);
    LGPU_CUDA(cudaMemsetAsync(dst, 0, n * dim_pad, nullptr));
    LGPU_CUDA(cudaMemcpy2DAsync(dst, dim_pad, codes, dim, dim, n, cudaMemcpyHostToDevice, nullptr));
    launch_sq_row_norms(dst, n, dim_pad, xx, nullptr);
}
static void upload_sq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, DevBuf &dst, DevBuf &xx)
{
    dst.ensure(std::max<size_t>((size_t)n * sq_dim_pad(dim), 16));
    xx.ensure(std::max<size_t>((size_t)n * 4, 16));
    if (n) fill_sq_rows(codes, n, dim, dst.as<uint8_t>(), xx.as<uint32_t>());
    LGPU_CUDA(cudaStreamSynchronize(nullptr));
}

// IVF_RQ stored rows: dim zero-padded to the scan's K step, in 32-bit words
static uint32_t rq_wpr(uint32_t dim) { return (uint32_t)round_up64(dim, RQ_K_BITS) / 32; }

// codes [n][ceil(dim / 8)] (host) -> dst [n][wpr] u32 (device, zero padding, bits past dim cleared) and popc[r], on the
// legacy stream
static void fill_rq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, uint32_t *dst, uint32_t *popc)
{
    const uint32_t wpr = rq_wpr(dim), nb = (dim + 7) / 8;
    LGPU_CUDA(cudaMemsetAsync(dst, 0, n * wpr * 4, nullptr));
    LGPU_CUDA(cudaMemcpy2DAsync(dst, (size_t)wpr * 4, codes, nb, nb, n, cudaMemcpyHostToDevice, nullptr));
    launch_rq_row_prep(dst, n, dim, wpr, popc, nullptr);
}
static void upload_rq_rows(const uint8_t *codes, uint64_t n, uint32_t dim, DevBuf &dst, DevBuf &popc)
{
    dst.ensure(std::max<size_t>((size_t)n * rq_wpr(dim) * 4, 16));
    popc.ensure(std::max<size_t>((size_t)n * 4, 16));
    if (n) fill_rq_rows(codes, n, dim, dst.as<uint32_t>(), popc.as<uint32_t>());
    LGPU_CUDA(cudaStreamSynchronize(nullptr));
}

// The padded PQ layouts: partition p's codes at code_base[p] = row_bytes x the 32-row padded heights of the partitions
// before it ((nch + 1) x 8 bytes per row for the 8-bit streams, m/2 for 4-bit codes).  Returns the total bytes.
static uint64_t padded_code_base(const uint64_t *part_offsets, uint32_t nlist, uint64_t row_bytes,
                                 std::vector<uint64_t> &code_base)
{
    code_base.resize(nlist);
    uint64_t cb = 0;
    for (uint32_t p = 0; p < nlist; p++) {
        code_base[p] = cb;
        cb += row_bytes * (((part_offsets[p + 1] - part_offsets[p]) + 31u) & ~31ull);
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

// after the desc's checks: the device, then a new index of `kind`
template <class H = lgpu_index> static H *new_ivf(int device, IvfKind kind)
{
    require_device(device);
    H *ix = new H();
    ix->kind = kind;
    return ix;
}

// lgpu_index_open with nbits = 8 (the desc's common fields are checked): the IVF arrays, the codebook tiled for the
// scans, the codes re-laid out as skewed streams (retile.cu) and the filter scan's tables (tables.cu)
static void open_pq8(const lgpu_index_desc *d, lgpu_index *&ix)
{
    const uint32_t nlist = d->nlist, nch = (d->m + 7) / 8;
    std::vector<uint64_t> code_base;
    const uint64_t cb = padded_code_base(d->part_offsets, nlist, (uint64_t)(nch + 1) * 8, code_base);
    ix = new_ivf(d->device, IvfKind::pq8);
    ix->m = d->m; ix->dsub = d->dim / d->m; ix->nch = nch;
    open_ivf_common(ix, d, SCAN_ROWS_TILE_MID, code_base);
    cudaStream_t st = nullptr;
    {   // codebook -> [nch][256][8][dsub]
        DevBuf tmp;
        upload(tmp, d->codebook, (size_t)d->m * 256 * ix->dsub * 4);
        ix->cb_tiled.ensure((size_t)ix->nch * 256 * 8 * ix->dsub * 4);
        launch_retile_codebook(tmp.as<float>(), d->m, ix->dsub, ix->nch, ix->cb_tiled.as<float>(), st);
        LGPU_CUDA(cudaStreamSynchronize(st));
    }
    {   // codes -> skewed streams
        ix->codes.hbm.ensure(std::max<uint64_t>(cb, 16));
        LGPU_CUDA(cudaMemsetAsync(ix->codes.hbm.p, 0, ix->codes.hbm.bytes, st));
        DevBuf tmp;
        if (d->nrows) {
            upload(tmp, d->codes, (size_t)d->nrows * d->m);
            launch_retile_codes(tmp.as<unsigned char>(), d->codes_layout, ix->part_off.as<uint64_t>(), nlist, d->nrows,
                                d->m, ix->nch, ix->code_base.as<uint64_t>(), ix->part_npad.as<uint32_t>(),
                                ix->codes.hbm.as<unsigned char>(), st);
        }
        LGPU_CUDA(cudaStreamSynchronize(st));
    }
    {   // |b|^2 of the tiled codebook entries and CB2 = sum_i max_c |b|^2 (filter scan, tables.cu)
        ix->cb_n2.ensure((size_t)ix->nch * 256 * 8 * 4);
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
    float rmax = 0.f;
    if (d->metric != LGPU_DOT) {   // per-row constants of the filter scan (tables.cu)
        ix->row_R.ensure(std::max<size_t>((size_t)d->nrows * 4, 16));
        ix->rmax_bits.ensure(16);
        launch_row_const(ix->codes.hbm.as<unsigned char>(), ix->code_base.as<uint64_t>(), ix->part_npad.as<uint32_t>(),
                         ix->part_off.as<uint64_t>(), nlist, d->nrows, ix->centroids.as<float>(),
                         ix->cb_tiled.as<float>(), d->dim, d->m, ix->dsub, ix->row_R.as<float>(),
                         ix->rmax_bits.as<int>(), st);
        LGPU_CUDA(cudaStreamSynchronize(st));
        int bits = 0;
        LGPU_CUDA(cudaMemcpy(&bits, ix->rmax_bits.p, 4, cudaMemcpyDeviceToHost));
        rmax = __builtin_bit_cast(float, bits);
    }
    // the filter scan's error band (kernels.cuh scan_band) is finite only with a finite CB2 and max |R|: a NaN / inf
    // centroid or codeword leaves the index on the exact scan
    ix->has_tables = std::isfinite(ix->cb2) && std::isfinite(rmax);
}

// lgpu_index_open with nbits = 4 (the desc's common fields are checked): the IVF arrays, the codebook and the codes
// re-laid out for pq4_tables / pq4_scan.  No filter tables: the scan is exact.
static void open_pq4(const lgpu_index_desc *d, lgpu_index *&ix)
{
    LGPU_REQUIRE(d->m % 2 == 0, "num_sub_vectors must be even for 4-bit PQ codes");
    LGPU_REQUIRE(d->m <= LGPU_PQ4_MAX_M, "4-bit PQ codes support num_sub_vectors up to 256");
    std::vector<uint64_t> code_base;
    const uint64_t total = padded_code_base(d->part_offsets, d->nlist, d->m / 2, code_base);
    ix = new_ivf(d->device, IvfKind::pq4);
    ix->m = d->m; ix->dsub = d->dim / d->m; ix->nch = (d->m + 7) / 8;
    open_ivf_common(ix, d, PQ4_ROWS_TILE, code_base);
    // codebook [m][16][dsub] -> [m][dsub][16], the layout the table kernel reads
    const uint32_t m = d->m, dsub = ix->dsub;
    std::vector<float> cbt((size_t)m * 16 * dsub);
    for (uint32_t i = 0; i < m; i++)
        for (uint32_t j = 0; j < 16; j++)
            for (uint32_t t = 0; t < dsub; t++)
                cbt[((size_t)i * dsub + t) * 16 + j] = d->codebook[((size_t)i * 16 + j) * dsub + t];
    upload(ix->pq4_cb, cbt.data(), cbt.size() * 4);
    upload_pq4_codes(d->codes, d->codes_layout, d->nrows, d->m, d->nlist, ix->part_off.as<uint64_t>(),
                     ix->code_base.as<uint64_t>(), ix->part_npad.as<uint32_t>(), total, ix->codes.hbm);
}

// the HBM an index holds: every buffer its open allocated
static uint64_t index_device_bytes(const lgpu_index *ix)
{
    return ix->codes.device_bytes() + ix->vectors.device_bytes() +
           sum_bytes({&ix->centroids, &ix->cb_tiled, &ix->code_base, &ix->part_n, &ix->part_npad, &ix->part_off,
                      &ix->row_ids, &ix->row_R, &ix->rmax_bits, &ix->cb_n2, &ix->cent_b, &ix->cent_n2, &ix->cent_sb,
                      &ix->cent_sn2, &ix->sq_xx, &ix->rq_rot, &ix->rq_rc, &ix->rq_add, &ix->rq_scale, &ix->rq_popc,
                      &ix->pq4_cb, &ix->cent_pop, &ix->row_pop, &ix->hn_levels, &ix->hn_adj0, &ix->hn_upper_index,
                      &ix->hn_upper_adj, &ix->hn_entry, &ix->hn_top});
}

// lgpu_index_code_bytes, lgpu_ivf_binary_code_bytes: the pinned bytes of an index's codes and where they are
template <class H> static int code_bytes(const H *hp, uint64_t *bytes, int *placement)
{
    return host_placement(hp, bytes, placement,
                          [](const H *ix) { return std::pair<const RowStore *, uint64_t>{&ix->codes, 0}; });
}

// Whether `bytes` of a handle's rows go to HBM at open: at most the cap the variable `cap_var` sets (read at every open;
// unset = no cap, 0 = never HBM), and the device's free memory covers them plus the workspace budget (LGPU_WS_BYTES)
// the handle's searches may lease
static bool rows_fit_hbm(const char *cap_var, uint64_t bytes)
{
    const char *e = getenv(cap_var);
    const uint64_t cap = (e && *e) ? strtoull(e, nullptr, 10) : UINT64_MAX;
    size_t free_b = 0, total_b = 0;
    LGPU_CUDA(cudaMemGetInfo(&free_b, &total_b));
    return cap > 0 && bytes <= cap && (uint64_t)free_b >= bytes + workspace_budget();
}

// Where an IVF_SQ, IVF_RQ or binary IVF_FLAT index keeps its codes, nrows x row_bytes in the scan's layout: in HBM when
// they fit with room to spare (rows_fit_hbm under LGPU_CODES_HBM_BYTES), allocated exactly, so that device bytes of the
// two placements differ by the code bytes; otherwise in pinned, mapped host memory the index owns, in the same layout.
// fill(dst, r0, n) lays rows r0 .. r0 + n out at device address dst and runs the kind's per-row kernel on them.  An HBM
// store is one chunk of every row, laid out in place; a host store is built in chunks of CODE_PREP_BYTES in one HBM
// buffer, each copied into the pinned rows (never a device copy of the whole index), so the stored bytes and the
// per-row terms of the two placements are the same.  The chunks of consecutive partitions a search walks are cut here:
// one for an HBM store; for a host store, each at most code_stage bytes (FLAT_STAGE_BYTES, or an eighth of the
// workspace budget when that is smaller, never less than the largest partition), and two staging buffers of the
// largest partition must fit the budget, or the open fails with LGPU_OOM.  IVF_HNSW_SQ (its graph walk reads rows at
// random) and the PQ kinds keep their codes in HBM: they never come here.
constexpr size_t CODE_PREP_BYTES = (size_t)64 << 20;

template <class Fill> static void place_codes(lgpu_index *ix, uint32_t row_bytes, Fill &&fill)
{
    const uint64_t n = ix->nrows, bytes = n * row_bytes;
    const uint32_t nlist = ix->nlist;
    const bool host = !rows_fit_hbm("LGPU_CODES_HBM_BYTES", bytes);
    ix->code_row_bytes = row_bytes;
    ix->code_cut.assign(1, 0);
    ix->code_rows.assign(1, 0);
    if (host) {
        uint64_t largest = 0;
        for (uint32_t p = 0; p < nlist; p++) largest = std::max<uint64_t>(largest, (uint64_t)ix->h_part_n[p] * row_bytes);
        const size_t budget = workspace_budget();
        if (2 * largest > budget) {
            set_error("the largest partition's codes (" + std::to_string(largest) + " bytes) do not fit twice in the " +
                      "workspace budget (LGPU_WS_BYTES) that stages an index whose codes are in host memory");
            throw Failure{LGPU_OOM};
        }
        ix->code_stage = std::max<size_t>(std::min(FLAT_STAGE_BYTES, budget / 8), std::max<size_t>(largest, 16));
        uint64_t in_chunk = 0, r = 0;
        for (uint32_t p = 0; p < nlist; p++) {
            const uint64_t b = (uint64_t)ix->h_part_n[p] * row_bytes;
            if (in_chunk && in_chunk + b > ix->code_stage) {
                ix->code_cut.push_back(p);
                ix->code_rows.push_back(r);
                in_chunk = 0;
            }
            in_chunk += b;
            r += ix->h_part_n[p];
        }
    }
    ix->code_cut.push_back(nlist);
    ix->code_rows.push_back(n);
    ix->codes.open(host, bytes);
    const uint64_t C = host ? std::max<uint64_t>(1, CODE_PREP_BYTES / row_bytes) : n;
    DevBuf tmp;
    if (host) tmp.ensure((size_t)std::min(n, C) * row_bytes + 16);
    uint8_t *rows = reinterpret_cast<uint8_t *>(ix->codes.data());
    for (uint64_t r0 = 0; r0 < n; r0 += C) {
        const uint64_t c = std::min(C, n - r0);
        uint8_t *dst = host ? tmp.as<uint8_t>() : rows;
        fill(dst, r0, c);
        if (host)
            LGPU_CUDA(cudaMemcpyAsync(rows + r0 * row_bytes, dst, c * row_bytes, cudaMemcpyDeviceToHost, nullptr));
        LGPU_CUDA(cudaStreamSynchronize(nullptr));
    }
}

// Where an index keeps its raw vectors ([nrows][dim] f32 on the host, borrowed for the open call), decided after
// everything else the index holds is in HBM.  HBM when they fit with room to spare: at most LGPU_VECTORS_HBM_BYTES of
// them (read at every open; unset = no cap, 0 = never HBM), and the device's free memory covers them plus the
// workspace budget (LGPU_WS_BYTES) its searches may lease.  HBM rows are allocated exactly, so that device bytes of the
// two placements differ by nrows x dim x 4.  Otherwise a pinned, mapped host copy that the index owns,
// rows padded to a multiple of 4 floats, which refine reads over PCIe (launch_refine_host).
static void place_vectors(lgpu_index *ix, const float *vectors)
{
    if (!vectors) return;
    ix->has_vectors = true;
    const uint64_t n = ix->nrows, dim = ix->dim;
    const bool host = !rows_fit_hbm("LGPU_VECTORS_HBM_BYTES", n * dim * 4);
    const uint64_t stride = host ? round_up64(dim, 4) : dim;
    ix->vec_stride = (uint32_t)stride;
    ix->vectors.open(host, n * stride * 4);
    if (stride == dim) return ix->vectors.fill(0, vectors, n * dim * 4);
    float *dst = reinterpret_cast<float *>(ix->vectors.data());
    for (uint64_t r = 0; r < n; r++) {
        memcpy(dst + r * stride, vectors + r * dim, dim * 4);
        memset(dst + r * stride + dim, 0, (stride - dim) * 4);
    }
}

// The sequence of every IVF open: `open(ix)` checks the desc, then creates the index (new_ivf) and fills it, and returns
// the raw vectors it keeps for refine_factor (or null), which place_vectors places last; the index is then registered
// and returned, or deleted if any step failed.
template <class H, class Open> static int open_ivf(H **out, Open &&open)
{
    H *ix = nullptr;
    const int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr, "null argument");
        const float *vectors = open(ix);
        LGPU_CUDA(cudaStreamSynchronize(nullptr));
        place_vectors(ix, vectors);
        LGPU_CUDA(cudaStreamSynchronize(nullptr));
        ix->device_bytes = index_device_bytes(ix);
        register_handle(ix);
        *out = ix;
    });
    if (rc != LGPU_OK) delete ix;
    return rc;
}

// The tile queue of a kernel-alone debug entry: B queries, query b alone in probe slot b of one partition of N rows
// (at row 0, padded to 32 rows), cut into the regroup's row blocks for `rows_tile`; query b's output at b * stride.
// The descriptors go to `tiles`, the {total, 0} counter to `ctr`.  Returns the tile count.
static uint32_t debug_tiles(uint32_t B, uint32_t N, uint32_t rows_tile, uint64_t stride, DevBuf &tiles, DevBuf &ctr)
{
    const uint32_t nrb = scan_nrb(N, rows_tile), rbr = scan_rb_rows(N, nrb);
    std::vector<TileDesc> h;
    for (uint32_t q0 = 0; q0 < B; q0 += SCAN_G)
        for (uint32_t rb = 0; rb < nrb; rb++) {
            TileDesc t{};
            t.row0 = rb * rbr; t.nrows = std::min(rbr, N - t.row0);
            t.ng = std::min<uint32_t>(SCAN_G, B - q0); t.n_p = N; t.npad = (N + 31u) & ~31u;
            for (uint32_t g = 0; g < t.ng; g++) { t.q[g] = t.slot[g] = q0 + g; t.out[g] = (uint32_t)((q0 + g) * stride); }
            h.push_back(t);
        }
    const uint32_t total = (uint32_t)h.size(), counter[2] = {total, 0u};
    upload(tiles, h.data(), h.size() * sizeof(TileDesc));
    upload(ctr, counter, 8);
    LGPU_CUDA(cudaStreamSynchronize(nullptr));
    return total;
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
    return open_ivf(out, [&](lgpu_index *&ix) -> const float * {
        LGPU_REQUIRE(d != nullptr, "null argument");
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
        if (d->nbits == 4) open_pq4(d, ix);
        else open_pq8(d, ix);
        return d->vectors;
    });
}

int lgpu_ivf_sq_open(const lgpu_ivf_sq_desc *d, lgpu_index **out)
{
    return open_ivf(out, [&](lgpu_index *&ix) -> const float * {
        LGPU_REQUIRE(d != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->metric != LGPU_DOT, "IVF_SQ supports the l2 and cosine distance types, not dot");
        LGPU_REQUIRE(d->dim <= LGPU_SQ_MAX_DIM, "IVF_SQ supports dimensions up to 65536");
        LGPU_REQUIRE(std::isfinite(d->lo) && std::isfinite(d->hi) && d->lo <= d->hi,
                     "IVF_SQ bounds must be finite with lo <= hi");
        check_ivf_layout(d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->codes, d->row_ids);
        ix = new_ivf(d->device, IvfKind::sq);
        ix->dim_pad = sq_dim_pad(d->dim);
        ix->sq_lo = d->lo; ix->sq_hi = d->hi;
        open_ivf_common(ix, d, SQ_ROWS_TILE, std::vector<uint64_t>(d->nlist));
        const uint32_t dim = d->dim;
        ix->sq_xx.ensure(std::max<size_t>((size_t)d->nrows * 4, 16));       // (as upload_sq_rows sizes it)
        place_codes(ix, ix->dim_pad, [&](uint8_t *dst, uint64_t r0, uint64_t n) {
            fill_sq_rows(d->codes + r0 * dim, n, dim, dst, ix->sq_xx.as<uint32_t>() + r0);
        });
        return d->vectors;
    });
}

// IVF_HNSW_SQ's graph, checked on the host before any device work: every position in its partition, every upper-level
// block inside upper_adj, every upper-level neighbour at least on the level it is listed at, every entry row on its
// partition's top level
static void check_hnsw_graph(const lgpu_ivf_hnsw_sq_desc *d)
{
    const uint32_t m = d->m, nlist = d->sq.nlist;
    LGPU_REQUIRE(m >= 1 && m <= LGPU_HNSW_MAX_M, "IVF_HNSW_SQ: m must be in [1, 64]");
    LGPU_REQUIRE(d->sq.nrows == 0 || (d->levels && d->adj0 && d->upper_index), "null graph array");
    LGPU_REQUIRE(d->entry && d->top_level, "null graph array");
    LGPU_REQUIRE(d->upper_blocks == 0 || d->upper_adj, "null graph array");
    LGPU_REQUIRE(d->upper_blocks < (1ull << 32), "IVF_HNSW_SQ: more than 2^32 upper-level blocks");
    for (uint32_t p = 0; p < nlist; p++) {
        const uint64_t off = d->sq.part_offsets[p], n = d->sq.part_offsets[p + 1] - off;
        if (n == 0) continue;
        const uint32_t top = d->top_level[p];
        LGPU_REQUIRE(top <= LGPU_HNSW_MAX_LEVEL, "IVF_HNSW_SQ: a top level above 15");
        LGPU_REQUIRE(d->entry[p] < n && d->levels[off + d->entry[p]] == top,
                     "IVF_HNSW_SQ: an entry row outside its partition or not on the top level");
        for (uint64_t r = off; r < off + n; r++) {
            const uint32_t lv = d->levels[r];
            LGPU_REQUIRE(lv <= top, "IVF_HNSW_SQ: a row above its partition's top level");
            for (uint32_t j = 0; j < 2 * m; j++) {
                const uint32_t v = d->adj0[r * 2 * m + j];
                LGPU_REQUIRE(v == LGPU_HNSW_NONE || v < n, "IVF_HNSW_SQ: a level-0 neighbour outside its partition");
            }
            if (lv == 0) continue;
            const uint64_t u = d->upper_index[r];
            LGPU_REQUIRE(u + lv <= d->upper_blocks, "IVF_HNSW_SQ: an upper_index outside upper_adj");
            for (uint32_t L = 1; L <= lv; L++)
                for (uint32_t j = 0; j < m; j++) {
                    const uint32_t v = d->upper_adj[(u + L - 1) * m + j];
                    LGPU_REQUIRE(v == LGPU_HNSW_NONE || (v < n && d->levels[off + v] >= L),
                                 "IVF_HNSW_SQ: an upper-level neighbour outside its partition or below its level");
                }
        }
    }
}

int lgpu_ivf_hnsw_sq_open(const lgpu_ivf_hnsw_sq_desc *d, lgpu_index **out)
{
    return open_ivf(out, [&](lgpu_index *&ix) -> const float * {
        LGPU_REQUIRE(d != nullptr, "null argument");
        const lgpu_ivf_sq_desc *s = &d->sq;
        LGPU_REQUIRE(s->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(s->metric != LGPU_DOT, "IVF_HNSW_SQ supports the l2 and cosine distance types, not dot");
        LGPU_REQUIRE(s->dim <= LGPU_SQ_MAX_DIM, "IVF_HNSW_SQ supports dimensions up to 65536");
        LGPU_REQUIRE(std::isfinite(s->lo) && std::isfinite(s->hi) && s->lo <= s->hi,
                     "IVF_HNSW_SQ bounds must be finite with lo <= hi");
        check_ivf_layout(s->dim, s->nlist, s->metric, s->nrows, s->centroids, s->part_offsets, s->codes, s->row_ids);
        check_hnsw_graph(d);
        ix = new_ivf(s->device, IvfKind::hnsw_sq);
        ix->dim_pad = sq_dim_pad(s->dim);
        ix->sq_lo = s->lo; ix->sq_hi = s->hi;
        ix->hnsw_m = d->m;
        open_ivf_common(ix, s, SQ_ROWS_TILE, std::vector<uint64_t>(s->nlist));
        upload_sq_rows(s->codes, s->nrows, s->dim, ix->codes.hbm, ix->sq_xx);
        upload(ix->hn_levels, d->levels, (size_t)s->nrows);
        upload(ix->hn_adj0, d->adj0, (size_t)s->nrows * 2 * d->m * 4);
        upload(ix->hn_upper_index, d->upper_index, (size_t)s->nrows * 4);
        upload(ix->hn_upper_adj, d->upper_adj, (size_t)d->upper_blocks * d->m * 4);
        upload(ix->hn_entry, d->entry, (size_t)s->nlist * 4);
        upload(ix->hn_top, d->top_level, (size_t)s->nlist);
        LGPU_CUDA(cudaStreamSynchronize(nullptr));
        return s->vectors;
    });
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
        debug_tiles(B, (uint32_t)N, SQ_ROWS_TILE, N, tiles, ctr);
        D.ensure((size_t)B * N * 4);
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
        // the one partition's codes laid out as in an index; query b's sums at b * ld (segments padded to 4, as in a
        // search)
        const uint64_t off[2] = {0, N}, ld = (N + 3) & ~3ull;
        const uint32_t npad = (uint32_t)((N + 31) & ~31ull);
        std::vector<uint64_t> code_base;
        const uint64_t total_bytes = padded_code_base(off, 1, m / 2, code_base);
        DevBuf d_off, d_cb, d_npad, X, tab, sl, D, tiles, ctr;
        upload(d_off, off, 16); upload(d_cb, code_base.data(), 8); upload(d_npad, &npad, 4);
        upload_pq4_codes(codes, LGPU_CODES_ROW_MAJOR, N, m, 1, d_off.as<uint64_t>(), d_cb.as<uint64_t>(),
                         d_npad.as<uint32_t>(), total_bytes, X);
        upload(tab, tables, (size_t)B * m * 16);
        sl.ensure((size_t)B * sizeof(Pq4Slot));
        debug_tiles(B, (uint32_t)N, PQ4_ROWS_TILE, ld, tiles, ctr);
        D.ensure((size_t)B * ld * 4);
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
    return open_ivf(out, [&](lgpu_index *&ix) -> const float * {
        LGPU_REQUIRE(d != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->metric != LGPU_DOT, "IVF_RQ supports the l2 and cosine distance types, not dot");
        LGPU_REQUIRE(d->num_bits == 1, "IVF_RQ supports num_bits = 1 only");
        LGPU_REQUIRE(d->dim <= LGPU_RQ_MAX_DIM, "IVF_RQ supports dimensions up to 4096");
        LGPU_REQUIRE(d->rotation != nullptr, "null index array");
        LGPU_REQUIRE(d->nrows == 0 || (d->add_factors && d->scale_factors), "null index array");
        check_ivf_layout(d->dim, d->nlist, d->metric, d->nrows, d->centroids, d->part_offsets, d->codes, d->row_ids);
        ix = new_ivf(d->device, IvfKind::rq);
        ix->rq_wpr = rq_wpr(d->dim);
        open_ivf_common(ix, d, RQ_ROWS_TILE, std::vector<uint64_t>(d->nlist));
        const uint32_t dim = d->dim, nb = (dim + 7) / 8;
        ix->rq_popc.ensure(std::max<size_t>((size_t)d->nrows * 4, 16));     // (as upload_rq_rows sizes it)
        place_codes(ix, ix->rq_wpr * 4, [&](uint8_t *dst, uint64_t r0, uint64_t n) {
            fill_rq_rows(d->codes + r0 * nb, n, dim, reinterpret_cast<uint32_t *>(dst), ix->rq_popc.as<uint32_t>() + r0);
        });
        upload(ix->rq_add, d->add_factors, (size_t)d->nrows * 4);
        upload(ix->rq_scale, d->scale_factors, (size_t)d->nrows * 4);
        upload(ix->rq_rot, d->rotation, (size_t)d->dim * d->dim * 4);
        ix->rq_rc.ensure((size_t)d->nlist * d->dim * 4);
        // rc_p = P c_p, once: each probe slot's residual is then one subtraction per dimension
        launch_rq_rotate(ix->rq_rot.as<float>(), ix->centroids.as<float>(), d->nlist, d->dim, ix->rq_rc.as<float>(),
                         nullptr);
        return d->vectors;
    });
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
        upload(add, add_factors, (size_t)N * 4); upload(scale, scale_factors, (size_t)N * 4);
        upload(Q, q_res, (size_t)B * dim * 4);
        zero.ensure((size_t)dim * 4); probes.ensure((size_t)B * 8);
        planes.ensure((size_t)B * 4 * wpr * 4); slots.ensure((size_t)B * sizeof(RqSlot));
        LGPU_CUDA(cudaMemset(zero.p, 0, (size_t)dim * 4));
        LGPU_CUDA(cudaMemset(probes.p, 0, (size_t)B * 8));
        // query b is one probe slot of partition 0 whose rotated centroid is 0: q' = the given residual
        launch_rq_planes(Q.as<float>(), zero.as<float>(), probes.as<uint64_t>(), B, 1, 1, dim, wpr,
                         planes.as<uint32_t>(), slots.as<RqSlot>(), nullptr);
        const uint32_t total = debug_tiles(B, (uint32_t)N, RQ_ROWS_TILE, N, tiles, ctr), counter[2] = {total, 0u};
        D.ensure((size_t)B * N * 4);
        RqScanArgs a{};
        a.codes = X.as<uint32_t>(); a.add = add.as<float>(); a.scale = scale.as<float>(); a.popc = popc.as<uint32_t>();
        a.planes = planes.as<uint32_t>(); a.slots = slots.as<RqSlot>(); a.dim = dim; a.wpr = wpr;
        a.cosine = metric == LGPU_COSINE;
        a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1;
        a.tile_desc = tiles.as<TileDesc>(); a.dist_out = D.as<float>();
        for (int mode = 0; mode < 2; mode++) {
            void *dst = mode ? (void *)out_ip : (void *)out_est;
            if (!dst) continue;
            LGPU_CUDA(cudaMemcpy(ctr.p, counter, 8, cudaMemcpyHostToDevice));
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
        HandleRef<lgpu_index> ix(const_cast<lgpu_index *>(ixh));
        *bytes = ix->device_bytes;
    });
}

int lgpu_index_host_bytes(const lgpu_index *ixh, uint64_t *bytes, int *placement)
{
    return host_placement(ixh, bytes, placement, [](const lgpu_index *ix) {
        return std::pair<const RowStore *, uint64_t>{ix->has_vectors ? &ix->vectors : nullptr, 0};
    });
}

int lgpu_index_code_bytes(const lgpu_index *ix, uint64_t *host_bytes, int *placement)
{
    return code_bytes(ix, host_bytes, placement);
}

int lgpu_debug_refine_host(const float *queries, uint32_t B, const float *rows, uint64_t N, uint32_t dim,
                           const uint64_t *pos, uint32_t nc, int metric, int device, float *out)
{
    return guarded([&] {
        LGPU_REQUIRE(dim >= 1, "dim must be positive");
        LGPU_REQUIRE(metric == LGPU_L2 || metric == LGPU_COSINE || metric == LGPU_DOT, "unknown distance type");
        LGPU_REQUIRE(B == 0 || nc == 0 || (queries && pos && out && (N == 0 || rows)), "null buffer");
        for (uint64_t i = 0; i < (uint64_t)B * nc; i++)
            LGPU_REQUIRE(pos[i] < N || pos[i] == UINT64_MAX, "a position outside the rows");
        if (B == 0 || nc == 0) return;
        require_device(device);
        int sms = 0;
        LGPU_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        const uint32_t stride = (uint32_t)round_up64(dim, 4);
        RowStore h;
        h.open(true, (size_t)N * stride * 4);
        float *X = reinterpret_cast<float *>(h.data());
        memset(X, 0, h.host_bytes());
        for (uint64_t r = 0; r < N; r++) memcpy(X + r * stride, rows + r * dim, (size_t)dim * 4);
        DevBuf q, p, o;
        upload(q, queries, (size_t)B * dim * 4);
        upload(p, pos, (size_t)B * nc * 8);
        o.ensure((size_t)B * nc * 4);
        launch_refine_host(q.as<float>(), static_cast<const float *>(h.dev()), stride, p.as<uint64_t>(), B, nc, dim, metric,
                           o.as<float>(), sms, nullptr);
        LGPU_CUDA(cudaMemcpy(out, o.p, (size_t)B * nc * 4, cudaMemcpyDeviceToHost));
    });
}

int lgpu_last_scanned_code_bytes(uint64_t *bytes)
{
    return guarded([&] { LGPU_REQUIRE(bytes, "null argument"); *bytes = g_scanned_bytes; });
}

int lgpu_last_streamed_code_bytes(uint64_t *bytes)
{
    return guarded([&] { LGPU_REQUIRE(bytes, "null argument"); *bytes = g_streamed_bytes; });
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
        HandleRef<lgpu_index> ix(ixh);
        *out = ivf_sub_batch_size(ix.h, B, nprobes);
    });
}

// lgpu_debug_select(_large): the checks of the arguments (k_lo <= k <= k_hi) and the SelectArgs they describe
static SelectArgs debug_select_args(const lgpu_debug_select_args *a, int device, cudaStream_t st, uint32_t k_lo,
                                    uint32_t k_hi, const char *k_msg)
{
    LGPU_REQUIRE(a != nullptr, "null argument");
    LGPU_REQUIRE(a->mode >= 0 && a->mode <= 2, "select mode must be 0, 1 or 2");
    LGPU_REQUIRE(a->k >= k_lo && a->k <= k_hi, k_msg);
    auto a16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    LGPU_REQUIRE(a->out_count && (a->out_rec || (a->out_ids && a->out_dist)), "null output buffer");
    LGPU_REQUIRE(a16(a->out_rec), "out_rec must be 16-byte aligned");
    if (a->mode == 0) {
        LGPU_REQUIRE(a->dist && a->seg_off && a->probes && a->part_n && a->part_off, "null mode-0 buffer");
        LGPU_REQUIRE(a16(a->dist), "mode 0: dist must be 16-byte aligned");   // float4 loads
    } else if (a->mode == 1) {
        LGPU_REQUIRE(a->dense, "null mode-1 buffer");
    } else {
        LGPU_REQUIRE(a->cand_rec || (a->dense && a->cand_ids), "null mode-2 buffer");
        LGPU_REQUIRE(a16(a->cand_rec), "cand_rec must be 16-byte aligned");
        LGPU_REQUIRE(a->inner >= 1, "mode 2: inner must be at least 1");
    }
    require_device(device);
    if (a->mode == 0 && a->B > 0 && a->nprobes > 0) {
        // the kernels load every probed segment as float4 up to its length rounded up to 4
        const size_t ns = (size_t)a->B * a->nprobes;
        std::vector<uint64_t> probes(ns), seg(ns);
        std::vector<uint32_t> part_n(a->nlist);
        LGPU_CUDA(cudaStreamSynchronize(st));
        LGPU_CUDA(cudaMemcpy(probes.data(), a->probes, ns * 8, cudaMemcpyDeviceToHost));
        LGPU_CUDA(cudaMemcpy(seg.data(), a->seg_off, ns * 8, cudaMemcpyDeviceToHost));
        if (a->nlist) LGPU_CUDA(cudaMemcpy(part_n.data(), a->part_n, (size_t)a->nlist * 4, cudaMemcpyDeviceToHost));
        for (size_t s = 0; s < ns; s++) {
            if (probes[s] >= a->nlist) continue;
            LGPU_REQUIRE(seg[s] % 4 == 0, "mode 0: seg_off must be a multiple of 4");
            LGPU_REQUIRE(seg[s] <= a->dist_len && round_up64(part_n[probes[s]], 4) <= a->dist_len - seg[s],
                         "mode 0: a segment padded to 4 floats runs past dist_len");
        }
    }
    SelectArgs s{};
    s.mode = a->mode;
    s.dist = a->dist; s.seg_off = a->seg_off; s.probes = a->probes; s.nprobes = a->nprobes; s.nlist = a->nlist;
    s.part_n = a->part_n; s.part_off = a->part_off; s.row_ids = a->row_ids;
    s.dense = a->dense; s.ncols = a->ncols; s.row_stride = a->row_stride;
    s.inner = a->inner; s.outer_stride = a->outer_stride;
    s.col_ids = a->col_ids; s.cand_ids = a->cand_ids; s.cand_pos = a->cand_pos; s.ncols_q = a->ncols_q;
    s.cand_rec = static_cast<const TopkRecord *>(a->cand_rec);
    s.B = a->B; s.k = a->k;
    s.has_lower = a->has_lower; s.has_upper = a->has_upper; s.lower = a->lower; s.upper = a->upper;
    s.out_ids = a->out_ids; s.out_dist = a->out_dist; s.out_count = a->out_count;
    s.out_rec = static_cast<TopkRecord *>(a->out_rec); s.out_pos = a->out_pos;
    s.only = a->only; s.gate = a->gate; s.allow = a->allow; s.allow_bits = a->allow_bits;
    return s;
}

int lgpu_debug_select(const lgpu_debug_select_args *a, int device, void *cuda_stream)
{
    return guarded([&] {
        cudaStream_t st = (cudaStream_t)cuda_stream;
        launch_select(debug_select_args(a, device, st, 1, SELECT_KMAX, "k must be in [1, 2048]"), st);
    });
}

int lgpu_debug_select_large(const lgpu_debug_select_args *a, int device, void *cuda_stream)
{
    return guarded([&] {
        cudaStream_t st = (cudaStream_t)cuda_stream;
        SelectArgs s = debug_select_args(a, device, st, SELECT_KMAX + 1, LGPU_K_MAX,
                                         "k must be in [2049, 65536] (above 2048, at most LGPU_K_MAX)");
        DevBuf scratch;
        s.scratch_bytes = select_large_scratch_bytes(s.B, s.k, s.out_pos != nullptr);
        scratch.ensure(s.scratch_bytes);
        s.scratch = scratch.p;
        launch_select_large(s, st);
        LGPU_CUDA(cudaStreamSynchronize(st));                // before the scratch is freed
    });
}

static void check_ivf_call(lgpu_index *ix, const void *q, uint32_t B, const lgpu_search_params *p,
                           const void *a, const void *b, const void *c)
{
    const bool refine = ix->kind != IvfKind::ham;     // Hamming distances are exact: refine_factor is ignored
    check_call(p, B, q, a, b, c, refine);
    LGPU_REQUIRE(p->nprobes >= 1, "minimum_nprobes must be greater than 0");
    LGPU_REQUIRE(p->nprobes <= SELECT_KMAX || p->nprobes >= ix->nlist,
                 "nprobes above 2048 is not supported unless it covers every partition");
    LGPU_REQUIRE(!refine || p->refine_factor == 0 || ix->has_vectors,
                 "refine_factor needs the raw vectors: open the index with desc.vectors");
    if (ix->kind == IvfKind::hnsw_sq)
        LGPU_REQUIRE(hnsw_efp(*p) <= LGPU_HNSW_EF_MAX,
                     "IVF_HNSW_SQ: ef and limit*refine_factor (or limit+offset) above 2048 (LGPU_HNSW_EF_MAX) are not "
                     "supported");
}

static int ivf_call(lgpu_index *ixh, const Route &r, const float *q, uint32_t B, const lgpu_search_params *p,
                    uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(ixh, r, q, B, p, ids, dist, cnt,
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
        HandleRef<lgpu_index> ix(ixh);
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
        : ix(h), lease(ix->pool, nullptr, false), deadline(timeout_ms) {}
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
            HandleRef<lgpu_index> ix(ixh);
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
                            const Deadline &) {
                            ivf_search_device(ix, ws, st, dq, B, sp, di, dd, dc, with_live(ws, st, RowFilter(), ix->live));
                        },
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

// The row data of a flat handle of n rows in HBM: the rows, and the tensor-core operand the handle builds for them (a
// bf16 copy for f32 rows; fp16 rows are their own) and |x|^2
static uint64_t flat_row_data_bytes(uint64_t n, uint32_t d, bool f16)
{
    const uint64_t rows = n * d * (f16 ? 2 : 4);
    if (!gemm_shape_supported(d) || n < 4096) return rows;
    return rows + (f16 ? 0 : n * d * 2) + n * 4;
}

// n of the caller's rows into rows n0.. of a flat handle's store, grown to hold them
static void flat_store_rows(lgpu_flat *fl, const void *src, uint64_t n0, uint64_t n)
{
    const size_t row = stored_row_bytes(fl);
    fl->rows.grow(n0 * row, (n0 + n) * row);
    fl->rows.fill(n0 * row, src, n * row);
}

// The per-row terms of a flat handle once rows [n0, n0 + n) are stored, at open (n0 = 0) or append.  In HBM, |x| once
// a cosine search built it.  Once a column of a GEMM shape holds 4096 rows, the tensor-core band (vec_max and vec_err,
// the maxima over every row) and, in HBM, the operand (vec_b, vec_n2): of every row when the column first gets there,
// else of the new rows while the band is finite.  Each chunk of the row store's visit gets tc_operand_rows, into the
// operand at its rows when the chunk is resident, else into scratch that only the band outlives.  A non-finite or
// overflowing row leaves the column to the exact kernels.
static void flat_row_terms(lgpu_flat *fl, uint64_t n0, uint64_t n)
{
    const uint64_t n1 = n0 + n;
    const uint32_t d = fl->dim;
    const bool f16 = fl->f16;
    const bool hbm = !fl->rows.on_host;
    if (hbm && fl->has_norms) {
        grow_keep(fl->ysqrt, (size_t)n0 * 4, (size_t)n1 * 4);
        const char *x = fl->rows.data() + n0 * stored_row_bytes(fl);
        if (f16) launch_row_norms(reinterpret_cast<const __half *>(x), n, d, fl->ysqrt.as<float>() + n0, nullptr);
        else launch_row_norms(reinterpret_cast<const float *>(x), n, d, fl->ysqrt.as<float>() + n0, nullptr);
    }
    if (!gemm_shape_supported(d) || n1 < 4096) return;
    const uint64_t a = n0 < 4096 ? 0 : n0;          // the first row whose terms are taken
    if (a > 0 && !fl->has_tc) return;
    if (hbm) {
        // room for the operand of rows [a, n1): an open has sized it exactly; an append that first reaches 4096 rows
        // gives the bf16 copy headroom (fp16 |x|^2 none), and later appends grow it as the rows grow
        if (!f16) grow_keep(fl->vec_b, (size_t)a * d * 2, (size_t)n1 * d * 2);
        if (a == 0) fl->vec_n2.ensure((size_t)n1 * 4, f16);
        else grow_keep(fl->vec_n2, (size_t)a * 4, (size_t)n1 * 4);
    }
    DevBuf xb, n2;
    bool finite = true;
    float xmax = 0.f, xerr = 0.f;
    fl->rows.visit(a, n1, stored_row_bytes(fl), [&](const RowChunk &ch) {
        const uint64_t m = ch.r1 - ch.r0;
        if (!ch.resident) {
            if (!f16) xb.ensure(m * d * 2);
            n2.ensure(m * 4);
        }
        void *b = f16 ? nullptr : ch.resident ? fl->vec_b.as<char>() + ch.r0 * d * 2 : xb.p;
        float *q = ch.resident ? fl->vec_n2.as<float>() + ch.r0 : n2.as<float>();
        float cm = 0.f, ce = 0.f;
        finite &= tc_operand_rows(ch.X, f16, m, d, b, q, cm, ce, nullptr);
        xmax = std::max(xmax, cm);
        xerr = std::max(xerr, ce);
    });
    fl->has_tc = finite;
    fl->vec_max = std::max(fl->vec_max, xmax);      // (both 0 before the column first reaches 4096 rows)
    fl->vec_err = std::max(fl->vec_err, xerr);
    if (!fl->has_tc) { fl->vec_b.reset(); fl->vec_n2.reset(); }
}

// lgpu_flat_open and lgpu_flat_open_f16: rows f32 or fp16 (f16), kept as given in HBM when their row data fits there
// (LGPU_FLAT_HBM_BYTES, rows_fit_hbm), else in pinned host memory the handle owns: an append of nrows rows to an empty
// store.  HBM rows and their operand are allocated exactly, so that device bytes of the two placements differ by the
// row data.
static int flat_open(const void *vectors, bool f16, uint64_t nrows, uint32_t dim, const uint64_t *row_ids, int device,
                     lgpu_flat **out)
{
    lgpu_flat *fl = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr && dim > 0, "null argument / zero dimension");
        LGPU_REQUIRE(nrows == 0 || vectors != nullptr, "null vectors");
        require_device(device);
        fl = new lgpu_flat();
        fl->device = device; fl->nrows = nrows; fl->dim = dim; fl->f16 = f16;
        fl->rows.open(!rows_fit_hbm("LGPU_FLAT_HBM_BYTES", flat_row_data_bytes(nrows, dim, f16)),
                      nrows * stored_row_bytes(fl));
        if (!fl->rows.on_host && gemm_shape_supported(dim) && nrows >= 4096) {
            if (!f16) fl->vec_b.ensure((size_t)nrows * dim * 2, true);
            fl->vec_n2.ensure((size_t)nrows * 4, true);
        }
        flat_store_rows(fl, vectors, 0, nrows);
        open_rows(fl, row_ids, nrows);
        flat_row_terms(fl, 0, nrows);
        register_handle(fl);
        *out = fl;
    });
    if (rc != LGPU_OK && fl) delete fl;
    return rc;
}

int lgpu_flat_open(const float *vectors, uint64_t nrows, uint32_t dim, const uint64_t *row_ids, int device,
                   lgpu_flat **out)
{
    return flat_open(vectors, false, nrows, dim, row_ids, device, out);
}

int lgpu_flat_open_f16(const uint16_t *vectors, uint64_t nrows, uint32_t dim, const uint64_t *row_ids, int device,
                       lgpu_flat **out)
{
    return flat_open(vectors, true, nrows, dim, row_ids, device, out);
}

int lgpu_flat_device_bytes(const lgpu_flat *fl, uint64_t *bytes) { return rows_device_bytes(fl, bytes); }
int lgpu_flat_host_bytes(const lgpu_flat *fl, uint64_t *bytes, int *placement)
{
    return rows_host_bytes(fl, bytes, placement);
}

void lgpu_flat_close(lgpu_flat *fl) { close_handle(fl); }

static int flat_call(lgpu_flat *flh, int metric, const Route &r, const float *q, uint32_t B,
                     const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(flh, r, q, B, p, ids, dist, cnt,
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

// n rows [n][nbytes] packed on the host as a binary handle stores them, [n][nbytes_pad] zero-padded: the layout the b1
// GEMM's TMA reads, so a host handle's staged chunk is the operand as it is
static void ham_pack_host(const uint8_t *src, uint64_t n, uint32_t nbytes, uint32_t nbytes_pad, uint8_t *dst)
{
    if (nbytes == nbytes_pad) { memcpy(dst, src, (size_t)n * nbytes); return; }
    for (uint64_t r = 0; r < n; r++) {
        memcpy(dst + r * nbytes_pad, src + r * nbytes, nbytes);
        memset(dst + r * nbytes_pad + nbytes, 0, nbytes_pad - nbytes);
    }
}

// n of the caller's rows [n][nbytes] into rows n0.. of a binary handle's store (grown to hold them), packed: on the host
// into pinned memory, or in HBM from an upload, with their popcounts into `pop` (grown to hold them)
static void ham_store_rows(lgpu_binary *bx, const void *src, uint64_t n0, uint64_t n)
{
    const uint32_t nbytes = bx->nbytes, nbp = bx->nbytes_pad;
    bx->rows.grow((size_t)n0 * nbp, (size_t)(n0 + n) * nbp);
    uint8_t *dst = reinterpret_cast<uint8_t *>(bx->rows.data()) + (size_t)n0 * nbp;
    if (bx->rows.on_host) return ham_pack_host(static_cast<const uint8_t *>(src), n, nbytes, nbp, dst);
    grow_keep(bx->pop, (size_t)n0 * 4, (size_t)(n0 + n) * 4);
    DevBuf raw;
    upload(raw, src, (size_t)n * nbytes);
    launch_ham_pack(raw.as<uint8_t>(), nbytes, nbytes, n, dst, nbp, bx->pop.as<uint32_t>() + n0, nullptr);
}

// The packed rows and their popcounts go to HBM when they fit there (LGPU_BINARY_HBM_BYTES, rows_fit_hbm), else the
// rows are packed into pinned host memory the handle owns: an append of nrows rows to an empty store.  HBM rows and
// popcounts are allocated exactly, so that device bytes of the two placements differ by nrows x (nbytes_pad + 4); an
// empty HBM handle holds 16 bytes of each, with headroom.
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
        const bool host = !rows_fit_hbm("LGPU_BINARY_HBM_BYTES", nrows * (nbp + 4));
        if (host || nrows) bx->rows.open(host, (size_t)nrows * nbp);
        else bx->rows.hbm.ensure(16);
        if (!host) bx->pop.ensure(nrows ? (size_t)nrows * 4 : 16, nrows > 0);
        ham_store_rows(bx, vectors, 0, nrows);
        open_rows(bx, row_ids, nrows);
        ham_sample(bx, 0, nrows);
        LGPU_CUDA(cudaDeviceSynchronize());
        register_handle(bx);
        *out = bx;
    });
    if (rc != LGPU_OK && bx) delete bx;
    return rc;
}

int lgpu_binary_device_bytes(const lgpu_binary *bx, uint64_t *bytes) { return rows_device_bytes(bx, bytes); }
int lgpu_binary_host_bytes(const lgpu_binary *bx, uint64_t *bytes, int *placement)
{
    return rows_host_bytes(bx, bytes, placement);
}

void lgpu_binary_close(lgpu_binary *bx) { close_handle(bx); }

static int binary_call(lgpu_binary *bxh, const Route &r, const uint8_t *q, uint32_t B, const lgpu_search_params *p,
                       uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(bxh, r, q, B, p, ids, dist, cnt,
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
    return open_ivf(out, [&](lgpu_ivf_binary *&ix) -> const float * {
        LGPU_REQUIRE(d != nullptr, "null argument");
        LGPU_REQUIRE(d->abi_version == LGPU_ABI_VERSION, "ABI version mismatch");
        LGPU_REQUIRE(d->nbytes > 0, "zero bytes per vector");
        LGPU_REQUIRE((uint64_t)d->nbytes * 8 <= ((uint64_t)1 << 24), "binary vectors above 2^24 bits are not supported");
        check_ivf_layout(d->nbytes, d->nlist, LGPU_L2, d->nrows, d->centroids, d->part_offsets, d->vectors, d->row_ids);
        ix = new_ivf<lgpu_ivf_binary>(d->device, IvfKind::ham);
        ix->nbytes = d->nbytes; ix->nbytes_pad = (d->nbytes + 31) & ~31u;
        ix->dim = d->nbytes;
        open_ivf_partitions(ix, d, HAM_ROWS_TILE, std::vector<uint64_t>(d->nlist));
        // centroids and rows zero-padded to nbytes_pad at dst, with their popcounts (ham_pack), from an upload
        const uint32_t nb = d->nbytes, nbp = ix->nbytes_pad;
        auto pack = [&](const uint8_t *src, uint64_t n, uint8_t *dst, uint32_t *pop) {
            DevBuf raw;
            upload(raw, src, (size_t)n * nb);
            launch_ham_pack(raw.as<uint8_t>(), nb, nb, n, dst, nbp, pop, nullptr);
            LGPU_CUDA(cudaStreamSynchronize(nullptr));
        };
        ix->centroids.ensure(std::max<size_t>((size_t)d->nlist * nbp, 16));
        ix->cent_pop.ensure(std::max<size_t>((size_t)d->nlist * 4, 16));
        pack(d->centroids, d->nlist, ix->centroids.as<uint8_t>(), ix->cent_pop.as<uint32_t>());
        ix->row_pop.ensure(std::max<size_t>((size_t)d->nrows * 4, 16));
        place_codes(ix, nbp, [&](uint8_t *dst, uint64_t r0, uint64_t n) {
            pack(d->vectors + r0 * nb, n, dst, ix->row_pop.as<uint32_t>() + r0);
        });
        return nullptr;             // the packed rows are the index: no separate raw vectors
    });
}

void lgpu_ivf_binary_close(lgpu_ivf_binary *ix) { close_handle(ix); }

int lgpu_ivf_binary_code_bytes(const lgpu_ivf_binary *ix, uint64_t *host_bytes, int *placement)
{
    return code_bytes(ix, host_bytes, placement);
}

static int ivf_binary_call(lgpu_ivf_binary *ixh, const Route &r, const uint8_t *q, uint32_t B,
                           const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(ixh, r, q, B, p, ids, dist, cnt,
                       [&](lgpu_ivf_binary *ix) { check_ivf_call(ix, q, B, p, ids, dist, cnt); return (size_t)B * ix->nbytes; },
                       ivf_search_device);
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

}  // extern "C"

// ---- appends to a flat or binary handle (the unindexed rows of a table, DESIGN.md section 3) ----
// The row ids after an append of n rows to n0: explicit ids stay explicit (positions n0.. when none are given), and
// ids given to a handle that had none make the old rows' positions explicit.
static void append_ids(lgpu_rows *h, uint64_t n0, uint64_t n, const uint64_t *row_ids)
{
    if (!row_ids && !h->has_ids) return;
    grow_keep(h->row_ids, h->has_ids ? n0 * 8 : 0, (n0 + n) * 8);
    std::vector<uint64_t> ids;
    if (!h->has_ids && n0) {
        ids.resize(n0);
        for (uint64_t i = 0; i < n0; i++) ids[i] = i;
        LGPU_CUDA(cudaMemcpy(h->row_ids.p, ids.data(), n0 * 8, cudaMemcpyHostToDevice));
    }
    if (!row_ids) {
        ids.resize(n);
        for (uint64_t i = 0; i < n; i++) ids[i] = n0 + i;
        row_ids = ids.data();
    }
    LGPU_CUDA(cudaMemcpy(static_cast<uint64_t *>(h->row_ids.p) + n0, row_ids, n * 8, cudaMemcpyHostToDevice));
    h->has_ids = true;
}

// What every append and delete does first, with the handle held exclusively: drain the device (a search enqueued
// earlier on a caller's stream may still read the buffers that move, the sample that is rewritten or the live bitmap
// that changes), and invalidate every captured graph, which bakes the row count and the row filter in even when no
// buffer moves.
static void begin_append(int device)
{
    require_device(device);
    LGPU_CUDA(cudaDeviceSynchronize());
    g_alloc_epoch++;
}

// ---- deleted rows (lgpu_*_delete): the live bitmap of a handle (RowLive) ----
// the row ids of a handle in device memory, or null when they are the positions 0 .. nrows - 1
static const uint64_t *device_row_ids(lgpu_index *ix) { return ix->row_ids.as<uint64_t>(); }
static const uint64_t *device_row_ids(const lgpu_rows *h) { return row_cols(h, 0).ids; }

static void require_id_bound(uint64_t max_id)
{
    LGPU_REQUIRE(max_id < LGPU_DELETE_ID_BOUND, "deleting rows needs every row id of the handle below "
                                                "LGPU_DELETE_ID_BOUND (2^32): the live bitmap holds one bit per id");
}

// the first delete: id_bound, and a bitmap with the bit of every row id the handle holds
template <class H> static void build_live(H *h)
{
    if (h->live.active) return;
    const uint64_t *ids = device_row_ids(h);
    uint64_t bound = h->nrows;
    if (ids && h->nrows) {
        DevBuf m;
        m.ensure(8);
        LGPU_CUDA(cudaMemset(m.p, 0, 8));
        launch_rowmask_max(ids, h->nrows, m.as<unsigned long long>(), nullptr);
        uint64_t mx = 0;
        LGPU_CUDA(cudaMemcpy(&mx, m.p, 8, cudaMemcpyDeviceToHost));
        require_id_bound(mx);
        bound = mx + 1;
    } else if (bound) {
        require_id_bound(bound - 1);
    }
    h->live.bits.ensure(std::max<size_t>((bound + 31) / 32, 1) * 4);
    LGPU_CUDA(cudaMemset(h->live.bits.p, 0, h->live.bits.bytes));
    launch_rowmask_set(h->live.bits.template as<uint32_t>(), bound, ids, 0, h->nrows, nullptr);
    LGPU_CUDA(cudaDeviceSynchronize());
    h->live.id_bound = bound;
    h->live.active = true;
}

// An append to a handle with deleted rows, checked before anything changes: the id_bound after the n rows (row_ids:
// host, null = the positions that follow).  An appended row may not take the id of a deleted row the handle still
// holds: the id's bit would make that row live again, and nothing is undeleted.  (Ids at or above id_bound name no
// row, so the usual append -- ids above every held one -- needs no device work for this.)
template <class H> static uint64_t live_bound_after(H *h, uint64_t n, const uint64_t *row_ids)
{
    if (!h->live.active) return 0;
    uint64_t mn = h->nrows, mx = h->nrows + n - 1;
    if (row_ids) {
        mn = UINT64_MAX; mx = 0;
        for (uint64_t i = 0; i < n; i++) { mn = std::min(mn, row_ids[i]); mx = std::max(mx, row_ids[i]); }
    }
    require_id_bound(mx);
    const uint64_t nbits = h->live.id_bound;
    if (mn < nbits) {
        DevBuf mark, ids, cnt;
        mark.ensure(std::max<size_t>((nbits + 31) / 32, 1) * 4);
        LGPU_CUDA(cudaMemset(mark.p, 0, mark.bytes));
        if (row_ids) upload(ids, row_ids, (size_t)n * 8);
        launch_rowmask_set(mark.as<uint32_t>(), nbits, row_ids ? ids.as<uint64_t>() : nullptr, h->nrows, n, nullptr);
        cnt.ensure(8);
        LGPU_CUDA(cudaMemsetAsync(cnt.p, 0, 8, nullptr));
        launch_rowmask_revived(mark.as<uint32_t>(), static_cast<const uint32_t *>(h->live.bits.p), nbits,
                               device_row_ids(h), h->nrows, cnt.as<unsigned long long>(), nullptr);
        uint64_t revived = 0;
        LGPU_CUDA(cudaMemcpy(&revived, cnt.p, 8, cudaMemcpyDeviceToHost));
        LGPU_REQUIRE(revived == 0, "an appended row takes the id of a deleted row of the handle: appending it would "
                                   "undelete that row");
    }
    return std::max(nbits, mx + 1);
}

// ... and the appended rows marked live, once their ids are in place
template <class H> static void grow_live(H *h, uint64_t n0, uint64_t n, uint64_t bound)
{
    if (!h->live.active) return;
    const size_t w0 = (h->live.id_bound + 31) / 32, w1 = (bound + 31) / 32;
    if (w1 > w0) {
        grow_keep(h->live.bits, w0 * 4, w1 * 4);
        LGPU_CUDA(cudaMemset(h->live.bits.template as<uint32_t>() + w0, 0, (w1 - w0) * 4));
    }
    launch_rowmask_set(h->live.bits.template as<uint32_t>(), bound,
                       h->has_ids ? h->row_ids.template as<uint64_t>() + n0 : nullptr, n0, n, nullptr);
    h->live.id_bound = bound;
}

template <class H> static int delete_rows(H *hp, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return guarded([&] {
        HandleExcl<H> h(hp);
        LGPU_REQUIRE(n == 0 || row_ids != nullptr, "null row ids");
        if (n_deleted) *n_deleted = 0;
        if (n == 0) return;
        begin_append(h->device);
        build_live(h.h);
        DevBuf ids, cnt;
        upload(ids, row_ids, (size_t)n * 8);
        cnt.ensure(8);
        LGPU_CUDA(cudaMemsetAsync(cnt.p, 0, 8, nullptr));
        launch_rowmask_clear(h->live.bits.template as<uint32_t>(), h->live.id_bound, ids.as<uint64_t>(), n,
                             cnt.as<unsigned long long>(), nullptr);
        uint64_t c = 0;
        LGPU_CUDA(cudaMemcpy(&c, cnt.p, 8, cudaMemcpyDeviceToHost));
        if (n_deleted) *n_deleted = c;
    });
}

// The sequence of a flat, binary or multivector append of n rows (row_ids: host, null = the positions that follow):
// hold the handle alone, `check(h)`, `store(h, rows, n0, n)` the rows into the row store, grown to hold them, set
// their ids and live bits, then the kind's per-row terms `terms(h, n0, n)`, drain the device and publish the new row
// count.  The kind's open runs the same store and terms on an empty store of the placement it chose.
template <class H, class R, class Check, class Store, class Terms>
static int append_rows(H *hp, const R *rows, uint64_t n, const uint64_t *row_ids, Check &&check, Store &&store,
                       Terms &&terms)
{
    return guarded([&] {
        HandleExcl<H> h(hp);
        check(h.h);
        LGPU_REQUIRE(n == 0 || rows != nullptr, "null rows");
        if (n == 0) return;
        const uint64_t bound = live_bound_after(h.h, n, row_ids);
        begin_append(h->device);
        const uint64_t n0 = h->nrows, n1 = n0 + n;
        store(h.h, rows, n0, n);
        append_ids(h.h, n0, n, row_ids);
        grow_live(h.h, n0, n, bound);
        terms(h.h, n0, n);
        LGPU_CUDA(cudaDeviceSynchronize());
        h->nrows = n1;
    });
}

extern "C" {

// lgpu_flat_append and lgpu_flat_append_f16: the rows must have the handle's row type (f16)
static int flat_append(lgpu_flat *flh, const void *rows, bool f16, uint64_t n, const uint64_t *row_ids)
{
    return append_rows(flh, rows, n, row_ids,
        [&](lgpu_flat *fl) {
            LGPU_REQUIRE(fl->f16 == f16, fl->f16 ? "the handle holds fp16 rows: append them with lgpu_flat_append_f16"
                                                 : "the handle holds f32 rows: append them with lgpu_flat_append");
        },
        flat_store_rows, flat_row_terms);
}

int lgpu_flat_append(lgpu_flat *flh, const float *rows, uint64_t n, const uint64_t *row_ids)
{
    return flat_append(flh, rows, false, n, row_ids);
}

int lgpu_flat_append_f16(lgpu_flat *flh, const uint16_t *rows, uint64_t n, const uint64_t *row_ids)
{
    return flat_append(flh, rows, true, n, row_ids);
}

int lgpu_binary_append(lgpu_binary *bxh, const uint8_t *rows, uint64_t n, const uint64_t *row_ids)
{
    return append_rows(bxh, rows, n, row_ids, [](lgpu_binary *) {}, ham_store_rows, ham_sample);
}

int lgpu_index_delete(lgpu_index *ix, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return delete_rows(ix, row_ids, n, n_deleted);
}

int lgpu_ivf_binary_delete(lgpu_ivf_binary *ix, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return delete_rows(ix, row_ids, n, n_deleted);
}

int lgpu_flat_delete(lgpu_flat *fl, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return delete_rows(fl, row_ids, n, n_deleted);
}

int lgpu_binary_delete(lgpu_binary *bx, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return delete_rows(bx, row_ids, n, n_deleted);
}

int lgpu_multivec_delete(lgpu_multivec *mv, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted)
{
    return delete_rows(mv, row_ids, n, n_deleted);
}

}  // extern "C"

// ---- union search: an IVF index and a flat tail holding the rows added after it was built ([unindexed fragments &
// !fast_search] flat KNN over them, union, TopK again; SURVEY.md section 3.1).  The tail's exact scan runs on the tail
// workspace's stream, forked from the caller's, while the IVF step runs on the caller's; both write into the index
// workspace's [2][B][k] lists, and one select by (_distance, _rowid) merges them by their counts. ----
// the tail's row width and its exact scan: a float tail under the index's metric, a binary tail by Hamming distance
static uint32_t row_elems(const lgpu_flat *fl) { return fl->dim; }
static uint32_t row_elems(const lgpu_binary *bx) { return bx->nbytes; }
static void tail_search(lgpu_index *ix, lgpu_flat *fl, Workspace *ws, cudaStream_t st, const float *d_q, uint32_t B,
                        const lgpu_search_params &sp, uint64_t *ids, float *dist, uint32_t *cnt, RowFilter rf,
                        const Deadline *dl)
{
    flat_search_device(fl, ws, st, ix->metric, d_q, B, sp, ids, dist, cnt, rf, dl);
}
static void tail_search(lgpu_ivf_binary *, lgpu_binary *bx, Workspace *ws, cudaStream_t st, const uint8_t *d_q,
                        uint32_t B, const lgpu_search_params &sp, uint64_t *ids, float *dist, uint32_t *cnt,
                        RowFilter rf, const Deadline *dl)
{
    binary_search_device(bx, ws, st, d_q, B, sp, ids, dist, cnt, rf, dl);
}

template <class IX, class TL, class T>
static void union_search_device(IX *ix, Workspace *ws, cudaStream_t st, TL *tl, Workspace *wt, const T *d_q, uint32_t B,
                                const lgpu_search_params &sp, RowFilter rf, uint64_t *d_ids, float *d_dist,
                                uint32_t *d_cnt, const Deadline *dl)
{
    const uint32_t k = sp.k;
    const size_t bk = (size_t)B * k;
    ws->u_ids.ensure(2 * bk * 8); ws->u_dist.ensure(2 * bk * 4); ws->u_cnt.ensure((size_t)2 * B * 4);
    uint64_t *ids = ws->u_ids.as<uint64_t>();
    float *dist = ws->u_dist.as<float>();
    uint32_t *cnt = ws->u_cnt.as<uint32_t>();
    // each handle's own deleted rows (rf: the call's filter)
    const RowFilter rf_ix = with_live(ws, st, rf, ix->live);
    // ivf_search_device's own refusal, checked before the fork (no tail work is left behind by it)
    if (rf_ix.bits && std::min<uint32_t>(sp.max_nprobes, ix->nlist) > std::min<uint32_t>(std::max<uint32_t>(sp.nprobes, 1), ix->nlist))
        LGPU_REQUIRE(std::min<uint32_t>(sp.max_nprobes, ix->nlist) <= SELECT_KMAX || sp.max_nprobes >= ix->nlist,
                     "maximum_nprobes above 2048 is not supported unless it covers every partition");
    // joins the tail's stream back into st on every exit, a throw included (a timeout between sub-batches, a CUDA
    // error): the index workspace's `done` event, recorded on st, then fences the tail's writes into u_ids / u_dist
    struct Join {
        Workspace *wt;
        cudaStream_t st;
        bool forked = false;
        ~Join()
        {
            if (forked && (cudaEventRecord(wt->ev_join, wt->stream) != cudaSuccess ||
                           cudaStreamWaitEvent(st, wt->ev_join, 0) != cudaSuccess))
                cudaGetLastError();
        }
    } join{wt, st};
    if (tl->nrows) {
        LGPU_CUDA(cudaEventRecord(wt->ev_fork, st));
        LGPU_CUDA(cudaStreamWaitEvent(wt->stream, wt->ev_fork, 0));
        join.forked = true;
        tail_search(ix, tl, wt, wt->stream, d_q, B, sp, ids + bk, dist + bk, cnt + B,
                    with_live(wt, wt->stream, rf, tl->live), dl);
    } else {                                    // an empty tail contributes an empty list
        LGPU_CUDA(cudaMemsetAsync(cnt + B, 0, (size_t)B * 4, st));
    }
    ivf_search_device(ix, ws, st, d_q, B, sp, ids, dist, cnt, rf_ix, dl);
    if (join.forked) {
        join.forked = false;
        LGPU_CUDA(cudaEventRecord(wt->ev_join, wt->stream));
        LGPU_CUDA(cudaStreamWaitEvent(st, wt->ev_join, 0));
    }
    SelectArgs s = select_cands(dist, ids, k, B, k, {d_ids, d_dist, d_cnt});
    s.ncols = 2 * (uint64_t)k; s.outer_stride = bk; s.list_cnt = cnt;
    launch_select(with_scratch(ws, s), st);
}

// The entry sequence of the four union entry points: resolve both handles, check the call, then run
// union_search_device on workspaces leased from both handles' pools, on the caller's stream (device route; `allow` is
// then a device bitmap) or staged through host_call (host route: eager, honours timeout_ms).
template <class IX, class TL, class T>
static int union_call(IX *ixh, TL *tlh, bool device, const T *q, uint32_t B, const lgpu_search_params *p,
                      const uint32_t *allow, uint64_t allow_bits, uint64_t *ids, float *dist, uint32_t *cnt,
                      void *stream)
{
    return guarded([&] {
        const WsCharge charge;
        HandleRef<IX> ix(ixh);
        HandleRef<TL> tl(tlh);
        check_ivf_call(ix.h, q, B, p, ids, dist, cnt);
        LGPU_REQUIRE(row_elems(tl.h) == ix->dim, "the tail's vectors do not have the index's dimension");
        LGPU_REQUIRE(tl->device == ix->device, "the tail and the index are on different devices");
        LGPU_REQUIRE(allow != nullptr || allow_bits == 0, "allow bitmap is null");
        if (B == 0) return;
        require_device(ix->device);
        if (device) {
            WsLease li(ix->pool, (cudaStream_t)stream, true);
            WsLease lt(tl->pool, nullptr, false);
            const RowFilter rf{allow, allow ? allow_bits : 0};
            union_search_device(ix.h, li.ws, li.st, tl.h, lt.ws, q, B, *p, rf, ids, dist, cnt, nullptr);
            return;
        }
        host_call(ix->pool, q, (size_t)B * ix->dim, B, p->k, ids, dist, cnt, nullptr, p->timeout_ms,
                  [&](Workspace *ws, cudaStream_t st, const T *dq, uint64_t *di, float *dd, uint32_t *dc,
                      const Deadline &dl) {
                      const RowFilter rf = allow ? upload_allow(ws, st, allow, allow_bits) : RowFilter();
                      WsLease lt(tl->pool, nullptr, false);
                      union_search_device(ix.h, ws, st, tl.h, lt.ws, dq, B, *p, rf, di, dd, dc, &dl);
                  });
    });
}

extern "C" {

int lgpu_search_unindexed(lgpu_index *ixh, lgpu_flat *tail, const float *queries, uint32_t B,
                          const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                          uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return union_call(ixh, tail, false, queries, B, params, allow, allow_bits, out_ids, out_dist, out_count, nullptr);
}

int lgpu_search_unindexed_device(lgpu_index *ixh, lgpu_flat *tail, const float *d_queries, uint32_t B,
                                 const lgpu_search_params *params, const uint32_t *d_allow, uint64_t allow_bits,
                                 uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count, void *cuda_stream)
{
    return union_call(ixh, tail, true, d_queries, B, params, d_allow, allow_bits, d_out_ids, d_out_dist, d_out_count,
                      cuda_stream);
}

int lgpu_ivf_binary_search_unindexed(lgpu_ivf_binary *ixh, lgpu_binary *tail, const uint8_t *queries, uint32_t B,
                                     const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                     uint64_t *out_ids, float *out_dist, uint32_t *out_count)
{
    return union_call(ixh, tail, false, queries, B, params, allow, allow_bits, out_ids, out_dist, out_count, nullptr);
}

int lgpu_ivf_binary_search_unindexed_device(lgpu_ivf_binary *ixh, lgpu_binary *tail, const uint8_t *d_queries,
                                            uint32_t B, const lgpu_search_params *params, const uint32_t *d_allow,
                                            uint64_t allow_bits, uint64_t *d_out_ids, float *d_out_dist,
                                            uint32_t *d_out_count, void *cuda_stream)
{
    return union_call(ixh, tail, true, d_queries, B, params, d_allow, allow_bits, d_out_ids, d_out_dist, d_out_count,
                      cuda_stream);
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
        q.ensure((size_t)B * nbp); x.ensure((size_t)N * nbp); qp.ensure((size_t)B * 4); xp.ensure((size_t)N * 4);
        upload(rq, queries, (size_t)B * nbytes); upload(rx, vectors, (size_t)N * nbytes);
        launch_ham_pack(rq.as<uint8_t>(), nbytes, nbytes, B, q.as<uint8_t>(), nbp, qp.as<uint32_t>(), nullptr);
        launch_ham_pack(rx.as<uint8_t>(), nbytes, nbytes, N, x.as<uint8_t>(), nbp, xp.as<uint32_t>(), nullptr);
        debug_tiles(B, (uint32_t)N, HAM_ROWS_TILE, N, tiles, ctr);
        D.ensure((size_t)B * N * 4);
        HamScanArgs a{};
        a.rows = x.as<uint8_t>(); a.row_pop = xp.as<uint32_t>(); a.queries = q.as<uint8_t>(); a.qpop = qp.as<uint32_t>();
        a.nbytes_pad = nbp;
        a.total_tiles = ctr.as<uint32_t>(); a.tile_counter = ctr.as<uint32_t>() + 1;
        a.tile_desc = tiles.as<TileDesc>(); a.dist_out = D.as<float>(); a.out_u32 = 1;
        launch_ivf_ham_scan(a, 2 * prop.multiProcessorCount, nullptr);
        LGPU_CUDA(cudaMemcpy(out, D.p, (size_t)B * N * 4, cudaMemcpyDeviceToHost));
    });
}

// |v| of stored vectors [skip, n) of n in HBM (f32, or fp16 when f16) into ysqrt and, when `check`, whether every one of
// the n is
// finite and non-zero (false: the tensor-core path may not run), with the fp16 normalised operand of f32 vectors into
// Xh.  fp16 vectors are their own operand: the same kernels read their exact f32 upcast, so |v| and the check are an
// f32 handle's on those values.
static bool mv_vector_terms(const void *X, bool f16, uint64_t n, uint32_t dim, float *ysqrt, uint64_t skip, bool check,
                            void *Xh)
{
    if (f16) launch_row_norms(static_cast<const __half *>(X) + skip * dim, n - skip, dim, ysqrt + skip, nullptr);
    else launch_row_norms(static_cast<const float *>(X) + skip * dim, n - skip, dim, ysqrt + skip, nullptr);
    if (!check) return true;
    DevBuf bad;
    bad.ensure(n * 4);
    if (f16) launch_mv_normalize_f16(static_cast<const __half *>(X), n, dim, nullptr, bad.as<uint32_t>(), nullptr);
    else launch_mv_normalize_f16(static_cast<const float *>(X), n, dim, Xh, bad.as<uint32_t>(), nullptr);
    std::vector<uint32_t> hb(n);
    LGPU_CUDA(cudaMemcpy(hb.data(), bad.p, n * 4, cudaMemcpyDeviceToHost));
    return std::none_of(hb.begin(), hb.end(), [](uint32_t b) { return b != 0; });
}

// the rows an open or append hands a multivector handle: values [offsets[n]][dim] in the row type, offsets [n + 1]
struct MvRows {
    const void *values;
    const uint64_t *offsets;
};

// The checks of n rows an open or append hands a handle that holds `held` vectors, before anything changes: offsets
// that start at 0 and do not decrease, rows of at most MV_MAX_ROW vectors, a column of at most 2^40 vectors, and
// values for any vector.
static void check_multivec_rows(const MvRows &src, uint64_t n, uint64_t held)
{
    const uint64_t *offsets = src.offsets;
    LGPU_REQUIRE(offsets != nullptr, "null argument");
    LGPU_REQUIRE(offsets[0] == 0, "row offsets must start at 0");
    for (uint64_t r = 0; r < n; r++) {
        LGPU_REQUIRE(offsets[r + 1] >= offsets[r], "row offsets must not decrease");
        LGPU_REQUIRE(offsets[r + 1] - offsets[r] <= MV_MAX_ROW, "a multivector row holds at most 2^20 vectors");
    }
    const uint64_t T = offsets[n];
    LGPU_REQUIRE(T <= ((uint64_t)1 << 40) - held, "a multivector column holds at most 2^40 vectors");
    LGPU_REQUIRE(T == 0 || src.values != nullptr, "null vectors");
}

// whether a column of T vectors in nrows rows has the tensor-core shape
static bool mv_tc_shape(uint64_t T, uint64_t nrows, uint32_t dim)
{
    return T >= MV_TC_MIN_T && T < ((uint64_t)1 << 31) && nrows < 0xffffffffull && gemm_shape_supported(dim);
}

// n of the caller's rows into rows n0.. of a multivector handle: their offsets (host and device) and their vectors into
// the row store, grown to hold them
static void mv_store_rows(lgpu_multivec *mv, const MvRows *src, uint64_t n0, uint64_t n)
{
    const uint64_t T0 = mv->h_offsets[n0], T = src->offsets[n];
    const size_t vb = (size_t)mv->dim * mv_elem_bytes(mv);
    mv->h_offsets.resize(n0 + 1);                         // (a failed append may have left more)
    for (uint64_t r = 1; r <= n; r++) mv->h_offsets.push_back(T0 + src->offsets[r]);
    grow_keep(mv->offsets, (n0 + 1) * 8, (n0 + n + 1) * 8);
    LGPU_CUDA(cudaMemcpy(mv->offsets.as<uint64_t>() + n0, mv->h_offsets.data() + n0, (n + 1) * 8,
                         cudaMemcpyHostToDevice));
    mv->rows.grow(T0 * vb, (T0 + T) * vb);
    mv->rows.fill(T0 * vb, src->values, T * vb);
}

// The per-vector terms of a multivector handle once rows [n0, n0 + n) are stored, at open (n0 = 0) or append: |v| of
// their vectors, the longest row and the vector count.  Once the column has the tensor-core shape (mv_tc_shape), the row
// of each vector (col_row), an f32 handle's fp16 normalised operand (`ops`, the rows' placement) and tc_ok, whether
// every stored vector normalises (a zero or non-finite vector has NaN pairs, which the approximate score cannot skip as
// the exact min does): of every vector when the column first gets there, else of the new vectors while tc_ok holds, so
// tc_ok ends as an open of the whole column sets it.  Each chunk of the row store's visit gets mv_vector_terms (each
// vector's terms depend on that vector alone): a resident chunk's operand is written in place, a staged chunk's copied
// back into the pinned operand.
static void mv_row_terms(lgpu_multivec *mv, uint64_t n0, uint64_t n)
{
    const uint64_t n1 = n0 + n, *off = mv->h_offsets.data(), T0 = off[n0], T1 = off[n1];
    const uint32_t dim = mv->dim;
    const bool f16 = mv->f16;
    const uint64_t a = T0 < MV_TC_MIN_T ? 0 : T0;          // the first vector whose operand is taken
    const bool tc = mv_tc_shape(T1, n1, dim) && (a == 0 || mv->tc_ok);
    grow_keep(mv->ysqrt, T0 * 4, T1 * 4);
    if (tc) {
        if (a == 0) {                                      // the column gets there: operand of every vector
            mv->col_row.ensure(T1 * 4);
            if (!f16) mv->ops.open(mv->rows.on_host, T1 * dim * 2);
        } else {
            grow_keep(mv->col_row, a * 4, T1 * 4);
            if (!f16) mv->ops.grow(a * dim * 2, T1 * dim * 2);
        }
    }
    bool ok = true;
    DevBuf hs;
    mv->rows.visit(tc ? a : T0, T1, (size_t)dim * mv_elem_bytes(mv), [&](const RowChunk &ch) {
        const uint64_t m = ch.r1 - ch.r0;
        char *h = tc && !f16 ? mv->ops.data() + ch.r0 * dim * 2 : nullptr;   // the chunk's stored operand
        const bool copy = h && !ch.resident;
        if (copy) hs.ensure(m * dim * 2);
        const uint64_t skip = std::min(m, T0 > ch.r0 ? T0 - ch.r0 : 0);  // old vectors: their |v| is kept
        ok &= mv_vector_terms(ch.X, f16, m, dim, mv->ysqrt.as<float>() + ch.r0, skip, tc, copy ? hs.p : h);
        if (copy) LGPU_CUDA(cudaMemcpy(h, hs.p, m * dim * 2, cudaMemcpyDeviceToHost));
    });
    if (tc && T1 > a) {
        std::vector<uint32_t> cr(T1 - a);
        for (uint64_t r = a ? n0 : 0; r < n1; r++)
            for (uint64_t j = off[r]; j < off[r + 1]; j++) cr[j - a] = (uint32_t)r;
        LGPU_CUDA(cudaMemcpy(mv->col_row.as<uint32_t>() + a, cr.data(), (T1 - a) * 4, cudaMemcpyHostToDevice));
    }
    mv->tc_ok = tc && ok;
    for (uint64_t r = n0; r < n1; r++) mv->max_row = std::max(mv->max_row, off[r + 1] - off[r]);
    mv->total = T1;
}

// lgpu_multivec_open and lgpu_multivec_open_f16: vectors f32 or fp16 (f16), kept as given, in HBM when the row data --
// the vectors, and an f32 handle's operand when the column has the tensor-core shape -- fits there
// (LGPU_MULTIVEC_HBM_BYTES, rows_fit_hbm), else in pinned host memory the handle owns: an append of nrows rows to an
// empty store.  The rows and the operand are allocated exactly.
static int multivec_open(const void *values, bool f16, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                         const uint64_t *row_ids, int device, lgpu_multivec **out)
{
    lgpu_multivec *mv = nullptr;
    int rc = guarded([&] {
        LGPU_REQUIRE(out != nullptr && offsets != nullptr, "null argument");
        LGPU_REQUIRE(dim >= 1 && dim <= MV_MAX_DIM, "multivector dimension must be in [1, 65536]");
        const MvRows src{values, offsets};
        check_multivec_rows(src, nrows, 0);
        require_device(device);
        mv = new lgpu_multivec();
        mv->device = device; mv->nrows = nrows; mv->dim = dim; mv->f16 = f16;
        mv->h_offsets.assign(1, 0);
        const uint64_t T = offsets[nrows];
        const size_t xbytes = (size_t)T * dim * mv_elem_bytes(mv);
        const size_t hbytes = mv_tc_shape(T, nrows, dim) && !f16 ? (size_t)T * dim * 2 : 0;
        mv->rows.open(!rows_fit_hbm("LGPU_MULTIVEC_HBM_BYTES", xbytes + hbytes), xbytes);
        mv->ysqrt.ensure(std::max<size_t>((size_t)T * 4, 16));
        mv->offsets.ensure((size_t)(nrows + 1) * 8);
        mv_store_rows(mv, &src, 0, nrows);
        open_rows(mv, row_ids, nrows);
        mv_row_terms(mv, 0, nrows);
        LGPU_CUDA(cudaDeviceSynchronize());
        register_handle(mv);
        *out = mv;
    });
    if (rc != LGPU_OK && mv) delete mv;
    return rc;
}

int lgpu_multivec_open(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                       const uint64_t *row_ids, int device, lgpu_multivec **out)
{
    return multivec_open(values, false, offsets, nrows, dim, row_ids, device, out);
}

int lgpu_multivec_open_f16(const uint16_t *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                           const uint64_t *row_ids, int device, lgpu_multivec **out)
{
    return multivec_open(values, true, offsets, nrows, dim, row_ids, device, out);
}

// lgpu_multivec_append and lgpu_multivec_append_f16: the vectors must have the handle's row type (f16)
static int multivec_append(lgpu_multivec *mvh, const void *values, bool f16, const uint64_t *offsets, uint64_t n,
                           const uint64_t *row_ids)
{
    const MvRows src{values, offsets};
    return append_rows(mvh, &src, n, row_ids,
        [&](lgpu_multivec *mv) {
            LGPU_REQUIRE(mv->f16 == f16, mv->f16 ? "the handle holds fp16 vectors: append them with lgpu_multivec_append_f16"
                                                 : "the handle holds f32 vectors: append them with lgpu_multivec_append");
            check_multivec_rows(src, n, mv->total);
        },
        mv_store_rows, mv_row_terms);
}

int lgpu_multivec_append(lgpu_multivec *mvh, const float *values, const uint64_t *offsets, uint64_t n,
                         const uint64_t *row_ids)
{
    return multivec_append(mvh, values, false, offsets, n, row_ids);
}

int lgpu_multivec_append_f16(lgpu_multivec *mvh, const uint16_t *values, const uint64_t *offsets, uint64_t n,
                             const uint64_t *row_ids)
{
    return multivec_append(mvh, values, true, offsets, n, row_ids);
}

int lgpu_multivec_device_bytes(const lgpu_multivec *mv, uint64_t *bytes) { return rows_device_bytes(mv, bytes); }
int lgpu_multivec_host_bytes(const lgpu_multivec *mv, uint64_t *bytes, int *placement)
{
    return rows_host_bytes(mv, bytes, placement);
}

void lgpu_multivec_close(lgpu_multivec *mv) { close_handle(mv); }

// Host calls are never captured into a CUDA graph: the launch sequence depends on every query's vector count, not
// only on B.
static int multivec_call(lgpu_multivec *mvh, const Route &r, const float *q, const uint32_t *q_off, uint32_t B,
                         const lgpu_search_params *p, uint64_t *ids, float *dist, uint32_t *cnt)
{
    return search_call(mvh, r, q, B, p, ids, dist, cnt,
                       [&](lgpu_multivec *mv) {
                           check_call(p, B, q, ids, dist, cnt);
                           if (B == 0) return (size_t)0;
                           check_multivec_offsets(q_off, B);
                           mv_check_stage(mv);
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

// lgpu_debug_maxsim_gemm (f32 values: the F16MaxSim operand built as an f32 handle builds it) and
// lgpu_debug_maxsim_gemm_f16 (fp16 values: the F16RowMaxSim score on the values as they are, over |v| as an fp16 handle
// computes it)
static int debug_maxsim_gemm(const float *queries, uint32_t nqv, const void *values, bool f16, const uint64_t *offsets,
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
        const size_t es = f16 ? 2 : 4;
        DevBuf q, x, qh, xh, bad, cr, M, vn;
        q.ensure((size_t)nqv * dim * 4); x.ensure(std::max<size_t>((size_t)T * dim * es, 16));
        qh.ensure((size_t)nqv * dim * 2); xh.ensure(std::max<size_t>((size_t)T * dim * 2, 16));
        bad.ensure(std::max<size_t>(std::max<uint64_t>(T, nqv), 1) * 4); cr.ensure(std::max<size_t>(T, 1) * 4);
        M.ensure((size_t)nqv * nrows * 4); vn.ensure(std::max<size_t>(T, 1) * 4);
        std::vector<uint32_t> hcr(T);
        for (uint64_t r = 0; r < nrows; r++)
            for (uint64_t j = offsets[r]; j < offsets[r + 1]; j++) hcr[j] = (uint32_t)r;
        LGPU_CUDA(cudaMemcpy(q.p, queries, (size_t)nqv * dim * 4, cudaMemcpyHostToDevice));
        if (T) {
            LGPU_CUDA(cudaMemcpy(x.p, values, (size_t)T * dim * es, cudaMemcpyHostToDevice));
            LGPU_CUDA(cudaMemcpy(cr.p, hcr.data(), (size_t)T * 4, cudaMemcpyHostToDevice));
        }
        LGPU_CUDA(cudaMemset(M.p, 0, (size_t)nqv * nrows * 4));
        launch_mv_normalize_f16(q.as<float>(), nqv, dim, qh.p, bad.as<uint32_t>(), nullptr);
        if (f16) launch_row_norms(x.as<__half>(), T, dim, vn.as<float>(), nullptr);
        else launch_mv_normalize_f16(x.as<float>(), T, dim, xh.p, bad.as<uint32_t>(), nullptr);
        MaxSimOut mo{};
        mo.col_row = cr.as<uint32_t>(); mo.M = M.as<uint32_t>(); mo.ldM = nrows; mo.row_base = 0; mo.vnorm = vn.as<float>();
        launch_maxsim_gemm(qh.p, f16 ? x.p : xh.p, nqv, T, dim, mo, f16, prop.multiProcessorCount, nullptr);
        std::vector<uint32_t> keys((size_t)nqv * nrows);
        LGPU_CUDA(cudaMemcpy(keys.data(), M.p, keys.size() * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < keys.size(); i++) out[i] = keys[i] ? key_f32(keys[i]) : NAN;
    });
}

int lgpu_debug_maxsim_gemm(const float *queries, uint32_t nqv, const float *values, const uint64_t *offsets,
                           uint64_t nrows, uint32_t dim, int device, float *out)
{
    return debug_maxsim_gemm(queries, nqv, values, false, offsets, nrows, dim, device, out);
}

int lgpu_debug_maxsim_gemm_f16(const float *queries, uint32_t nqv, const uint16_t *values, const uint64_t *offsets,
                               uint64_t nrows, uint32_t dim, int device, float *out)
{
    return debug_maxsim_gemm(queries, nqv, values, true, offsets, nrows, dim, device, out);
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

// the sharded search's own bound on k: its merge (select mode 2 over world * k records) stays on the shared-memory
// selects, k <= SELECT_KMAX
static void check_sharded_call(lgpu_index *ix, const void *q, uint32_t B, const lgpu_search_params *p, const void *a,
                               const void *b, const void *c)
{
    check_ivf_call(ix, q, B, p, a, b, c);
    LGPU_REQUIRE(p->k <= SELECT_KMAX, "limit+offset above 2048 is not supported on the sharded path");
}

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
                      with_live(ws, st, RowFilter(), ix->live), deadline);
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
        HandleRef<lgpu_index> ix(ixh);
        HandleRef<lgpu_comm> c(ch);
        LGPU_REQUIRE(ix->kind == IvfKind::pq8, "sharded search serves 8-bit IVF_PQ indexes only");
        check_sharded_call(ix.h, queries, B, params, out_ids, out_dist, out_count);
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
        HandleRef<lgpu_index> ix(ixh);
        HandleRef<lgpu_comm> c(ch);
        LGPU_REQUIRE(ix->kind == IvfKind::pq8, "sharded search serves 8-bit IVF_PQ indexes only");
        check_sharded_call(ix.h, d_queries, B, params, d_out_ids, d_out_dist, d_out_count);
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
        HandleRef<lgpu_comm> c(ch);
        memcpy(times, c->last_ms, sizeof(c->last_ms));
    });
}

int lgpu_debug_coarse(lgpu_index *ixh, const float *queries, uint32_t B, uint32_t nprobes, uint32_t *out_parts,
                      float *out_dists)
{
    return guarded([&] {
        LGPU_REQUIRE(queries && out_parts && out_dists && B > 0 && nprobes > 0, "bad argument");
        HandleRef<lgpu_index> ix(ixh);
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
        const IvfQueries q{ivf_queries(ix.h, ws, st, ws->q.as<float>(), B), nullptr, nullptr, ix->dim};
        ivf_coarse(ix.h, ws, p, q, st, st, StageMarks{ws, false});
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
        HandleRef<lgpu_index> ix(ixh);
        LGPU_REQUIRE(ix->kind == IvfKind::pq8 || ix->kind == IvfKind::pq4,
                     "lgpu_debug_partition_distances serves IVF_PQ indexes only");
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
        HandleRef<lgpu_index> ix(ixh);
        LGPU_REQUIRE(ix->kind == IvfKind::pq8, "lgpu_debug_filter_bounds serves 8-bit IVF_PQ indexes only");
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
        ivf_coarse(ix.h, ws, p, IvfQueries{qs, nullptr, nullptr, ix->dim}, cs, st, StageMarks{ws, false});
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
    bool tc = gemm_shape_supported(dim) && k >= 256 && tc_enabled();
    float cmax = 0.f, cerr = 0.f;
    if (tc) {
        flags.ensure((size_t)CH * 4); gate.ensure(16);
        xb.ensure((size_t)CH * dim * 2); xn2.ensure((size_t)CH * 4); xerr.ensure((size_t)CH * 4);
        tc = prepare_tc_operand(d_cent, k, dim, cb, cn2, cmax, cerr, st);
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

// a training row holding a NaN or an infinity would be summed into the centre (or codeword) it lands in and poison it:
// an inf row has distance inf to every centre and goes to centre 0, a NaN row encodes to code 0 in every sub-space
static void require_finite_rows(const float *x, uint64_t n, uint32_t dim)
{
    for (uint64_t r = 0; r < n; r++)
        for (uint32_t t = 0; t < dim; t++)
            if (!std::isfinite(x[r * dim + t])) {
                set_error("training row " + std::to_string(r) + " holds a NaN or infinite value; training needs finite rows");
                throw Failure{LGPU_INVALID_INPUT};
            }
}

int lgpu_kmeans_train(const float *x, uint64_t n, uint32_t dim, float *centroids, uint32_t k, uint32_t iters, int device,
                      double *inertia_out)
{
    return guarded([&] {
        LGPU_REQUIRE(x && centroids && n > 0 && dim > 0 && k > 0, "null argument / empty shape");
        LGPU_REQUIRE(n < (1ull << 32), "too many training rows (sample them: sample_rate * num_partitions)");
        require_finite_rows(x, n, dim);
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
        require_finite_rows(x, n, dim);
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
