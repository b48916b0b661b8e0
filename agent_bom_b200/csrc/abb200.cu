// abb200.cu — C ABI of the H100 blast-radius engine: graph upload, walk dispatch,
// exposure-path rows, dependency reach.  See include/abb200.h for the contract.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cub/cub.cuh>
#include <nvtx3/nvToolsExt.h>      // header-only; ranges cost nothing unless a profiler is attached

#include "../../include/abb200.h"
#include "dedup.cuh"
#include "paths.cuh"
#include "context.cuh"
#include "histpack.cuh"
#include "reach.cuh"
#include "union.cuh"
#include "centrality.cuh"
#include "nxcentral.cuh"
#include "lateral.cuh"
#include "clusters.cuh"
#include "delta.cuh"
#include "walk.cuh"
#include "walkb.cuh"
#include "lookup.cuh"
#include "search.cuh"
#include "compliance.cuh"
#include "lifecycle.cuh"
#include "hops.cuh"

using namespace abb;

// ------------------------------------------------------------------ errors
static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

static int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_err = buf;
    return code;
}
#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess) return fail(ABB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

extern "C" const char *abb_last_error(void) { return g_err.c_str(); }
extern "C" int abb_version(void) { return ABB_VERSION; }
extern "C" int abb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
extern "C" int64_t abb_launch_count(void) { return g_launches.load(); }

// NVTX range around every host entry point and the stages inside a walk (Nsight Systems / ncu --nvtx show the C-ABI calls by name)
struct NvtxRange {
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

// ------------------------------------------------------------------ (a1) host CSR build
extern "C" int64_t abb_csr_entries(int64_t n_edges, const uint8_t *flags) {
    int64_t n = n_edges;
    for (int64_t i = 0; i < n_edges; i++) n += (flags[i] & ABB_EDGE_BIDIRECTIONAL) ? 1 : 0;
    return n;
}

extern "C" int abb_csr_build_host(int32_t n_nodes, int64_t n_edges, const int32_t *src, const int32_t *dst, const uint8_t *rel,
                                  const uint8_t *flags, uint32_t *fwd_off, int32_t *fwd_nbr, uint8_t *fwd_meta, uint32_t *fwd_eid,
                                  uint32_t *rev_off, int32_t *rev_nbr, uint8_t *rev_meta, uint32_t *rev_eid) {
    if (n_nodes < 0 || n_edges < 0) return fail(ABB_ERR_ARG, "negative sizes");
    if (n_edges >= (1ll << 31)) return fail(ABB_ERR_ARG, "edge index must fit 31 bits (eid2 is uint32)");
    std::vector<uint64_t> fc(static_cast<size_t>(n_nodes) + 1, 0), rc(static_cast<size_t>(n_nodes) + 1, 0);
    for (int64_t i = 0; i < n_edges; i++) {
        int32_t s = src[i], d = dst[i];
        if (s < 0 || s >= n_nodes || d < 0 || d >= n_nodes) return fail(ABB_ERR_ARG, "edge %lld endpoint out of range", (long long)i);
        fc[s]++; rc[d]++;
        if (flags[i] & ABB_EDGE_BIDIRECTIONAL) { fc[d]++; rc[s]++; }
    }
    uint64_t fa = 0, ra = 0;
    for (int32_t u = 0; u < n_nodes; u++) {
        uint64_t f = fc[u], r = rc[u];
        fwd_off[u] = static_cast<uint32_t>(fa); rev_off[u] = static_cast<uint32_t>(ra);
        fc[u] = fa; rc[u] = ra; fa += f; ra += r;
    }
    if (fa >= (1ull << 32)) return fail(ABB_ERR_ARG, "more than 2^32 adjacency entries");
    fwd_off[n_nodes] = static_cast<uint32_t>(fa); rev_off[n_nodes] = static_cast<uint32_t>(ra);
    // append in graph.edges order: adjacency[src] += e; reverse_adjacency[dst] += e;
    // bidirectional: adjacency[dst] += rev(e); reverse_adjacency[src] += rev(e)   (container.py:174-198)
    for (int64_t i = 0; i < n_edges; i++) {
        int32_t s = src[i], d = dst[i];
        uint8_t fl = flags[i];
        uint8_t m = static_cast<uint8_t>((rel[i] & ABB_META_REL_MASK) | ((fl & ABB_EDGE_TRAVERSABLE) ? ABB_META_TRAVERSABLE : 0));
        uint32_t e2 = static_cast<uint32_t>(i) * 2u;
        uint64_t p = fc[s]++; fwd_nbr[p] = d; fwd_meta[p] = m; fwd_eid[p] = e2;
        uint64_t r = rc[d]++; rev_nbr[r] = s; rev_meta[r] = m; rev_eid[r] = e2;
        if (fl & ABB_EDGE_BIDIRECTIONAL) {
            uint8_t mr = static_cast<uint8_t>(m | ABB_META_REVERSED_COPY);
            p = fc[d]++; fwd_nbr[p] = s; fwd_meta[p] = mr; fwd_eid[p] = e2 + 1;
            r = rc[s]++; rev_nbr[r] = d; rev_meta[r] = mr; rev_eid[r] = e2 + 1;
        }
    }
    // FIRST_PAIR: first entry of a row with a given neighbour (row-stamped scratch, O(E))
    std::vector<int32_t> stamp(static_cast<size_t>(n_nodes) + 1, -1);
    for (int pass = 0; pass < 2; pass++) {
        const uint32_t *off = pass ? rev_off : fwd_off; const int32_t *nb = pass ? rev_nbr : fwd_nbr; uint8_t *me = pass ? rev_meta : fwd_meta;
        std::fill(stamp.begin(), stamp.end(), -1);
        for (int32_t u = 0; u < n_nodes; u++)
            for (uint32_t p = off[u]; p < off[u + 1]; p++)
                if (stamp[nb[p]] != u) { stamp[nb[p]] = u; me[p] |= ABB_META_FIRST_PAIR; }
    }
    return ABB_OK;
}

constexpr int CTL_WORDS = 64;        // 5 tiers x 4 counters, twice (canonical walks at 0, individual walks at CTL_SET)
constexpr int CTL_SET = 32;
constexpr int CTL_FATAL = 4 * 4 + 2;  // last tier's fatal flag inside a set
constexpr int CTL_ROUTE = 24;         // {heavy hand-offs routed to the big block tier, to the warp tier} inside a set

// ------------------------------------------------------------------ device buffers
// The one owner of device memory: freed by its destructor, which must run while the buffer's device is current (scoped
// buffers are declared after the call's DeviceGuard; abb_graph_free deletes the graph under one).
struct DevBuf {
    void *p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept { if (this != &o) { release(); std::swap(p, o.p); std::swap(cap, o.cap); } return *this; }
    ~DevBuf() { release(); }
    // workspace reused across calls: grows with slack, old contents discarded
    int ensure(size_t bytes) {
        if (bytes <= cap) return ABB_OK;
        release();
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { e = cudaMalloc(&p, bytes); want = bytes; }
        if (e != cudaSuccess) return fail(ABB_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        cap = want;
        return ABB_OK;
    }
    // exact size: scratch that lives for one call (the ranking pass's R x 8 B keys leave no room for slack) and graph arrays
    int alloc(size_t bytes) {
        release();
        const size_t want = bytes ? bytes : 16;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) return fail(ABB_ERR_NOMEM, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
        cap = want;
        return ABB_OK;
    }
    // exact size (`bytes` plus `spare`), filled with `bytes` of host memory on `st`
    int upload(const void *src, size_t bytes, cudaStream_t st, size_t spare = 0) {
        if (int rc = alloc(bytes + spare)) return rc;
        if (bytes) CUDA_TRY(cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, st));
        return ABB_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

// grows workspace buffer `buf`; needs `int rc` in scope and keeps the first error in rc
#define ENS(buf, bytes) if (!rc) rc = (buf).ensure(static_cast<size_t>(bytes))

// One cub algorithm: `call(temp, bytes)` makes the cub call, once to size it and once to run it, so both share one argument list.
// `tmp` grows to exactly what cub asks for; each caller names its own (calls on different streams run at the same time).
template <class F>
static int cub_run(DevBuf &tmp, F &&call) {
    size_t bytes = 0;
    CUDA_TRY(call(nullptr, bytes));
    if (!tmp.p || bytes > tmp.cap) if (int rc = tmp.alloc(bytes)) return rc;
    CUDA_TRY(call(tmp.p, bytes));
    g_launches++;
    return ABB_OK;
}

// One kernel launch: enqueues `kern` with this configuration on `st`, counts it, and fails with ABB_ERR_CUDA under the caller's file and
// line when the launch is refused (bad configuration, too much shared memory, no image for the device).  The arguments convert to the
// kernel's parameter types as in a direct launch.  Call it as LAUNCH(kernel, grid, block, smem, stream, args...): C++17 has no
// std::source_location, so the macro supplies the call site.
template <class... P, class... A>
static int launch_at(const char *file, int line, void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A &&...args) {
    kern<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    g_launches++;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ABB_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(e), file, line);
    return ABB_OK;
}
#define LAUNCH(...) launch_at(__FILE__, __LINE__, __VA_ARGS__)

// exclusive prefix sum of n int64 values; `sync` waits for it
static int scan_i64(DevBuf &tmp, const int64_t *in, int64_t *out, int64_t n, cudaStream_t st, bool sync = false) {
    if (int rc = cub_run(tmp, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, in, out, static_cast<int>(n), st); })) return rc;
    if (sync) CUDA_TRY(cudaStreamSynchronize(st));
    return ABB_OK;
}

// positions k < n whose flag is set, in order, into pos; how many into *count (device memory)
template <class Pos, class Flag, class Count, class N>
static int select_flagged(DevBuf &tmp, Flag *flags, Pos *pos, Count *count, N n, cudaStream_t st) {
    cub::CountingInputIterator<Pos> iota(0);
    return cub_run(tmp, [&](void *t, size_t &b) { return cub::DeviceSelect::Flagged(t, b, iota, flags, pos, count, n, st); });
}

// blocks for `items` at `per_block` items each: at least one, and at most `per_sm` per SM when per_sm > 0
static unsigned grid_for(int64_t items, int64_t per_block, int sm_count = 0, int per_sm = 0) {
    int64_t b = (items + per_block - 1) / per_block;
    if (per_sm > 0) b = std::min<int64_t>(b, static_cast<int64_t>(per_sm) * sm_count);
    return static_cast<unsigned>(std::max<int64_t>(1, b));
}

static int ceil_log2_i64(int64_t n) { int b = 1; while ((1ll << b) < n) b++; return b; }

// pinned host blocks, recycled across results (cudaHostAlloc is milliseconds)
struct PinnedPool {
    std::mutex mu;
    std::vector<std::pair<void *, size_t>> free_blocks;
    void *get(size_t bytes, size_t *got) {
        if (bytes == 0) bytes = 16;
        {
            std::lock_guard<std::mutex> lk(mu);
            size_t best = SIZE_MAX, bi = SIZE_MAX;
            for (size_t i = 0; i < free_blocks.size(); i++)
                if (free_blocks[i].second >= bytes && free_blocks[i].second < best) { best = free_blocks[i].second; bi = i; }
            if (bi != SIZE_MAX && best <= bytes * 4 + (1 << 20)) {
                void *p = free_blocks[bi].first; *got = best;
                free_blocks.erase(free_blocks.begin() + bi);
                return p;
            }
        }
        size_t want = bytes + bytes / 8;
        void *p = nullptr;
        if (cudaHostAlloc(&p, want, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        *got = want;
        return p;
    }
    void put(void *p, size_t bytes) {
        if (!p) return;
        std::lock_guard<std::mutex> lk(mu);
        if (free_blocks.size() >= 64) { cudaFreeHost(p); return; }
        free_blocks.emplace_back(p, bytes);
    }
};
static PinnedPool g_pinned;

// a pinned block of g_pinned, returned to the pool by its destructor
struct HostBlock {
    void *p = nullptr; size_t bytes = 0;
    HostBlock() = default;
    HostBlock(HostBlock &&o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    HostBlock &operator=(HostBlock &&o) noexcept { if (this != &o) { release(); std::swap(p, o.p); std::swap(bytes, o.bytes); } return *this; }
    ~HostBlock() { release(); }
    bool alloc(size_t n) { release(); p = g_pinned.get(n, &bytes); return p != nullptr; }
    void release() { g_pinned.put(p, bytes); p = nullptr; bytes = 0; }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

// device-to-pinned-host copies on one stream: adds the bytes to *counted and keeps the first CUDA error
struct Readback {
    cudaStream_t st;
    int64_t *counted;
    cudaError_t err = cudaSuccess;
    void keep(cudaError_t e) { if (err == cudaSuccess) err = e; }
    void operator()(HostBlock &dst, const void *src, size_t bytes) {
        *counted += static_cast<int64_t>(bytes);
        if (err == cudaSuccess && bytes) err = cudaMemcpyAsync(dst.p, src, bytes, cudaMemcpyDeviceToHost, st);
    }
};

// ------------------------------------------------------------------ graph handle
struct ClusterTable;      // clusters_host.inl
struct DeltaTable;        // delta_host.inl
struct LookupState;       // lookup_host.inl
struct SearchState;       // search_host.inl
struct ComplianceTable;   // compliance_host.inl

// The one owner of a CUDA event, destroyed with it (the counterpart of DevBuf)
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(Event &&o) noexcept : e(o.e) { o.e = nullptr; }
    Event &operator=(Event &&o) noexcept { std::swap(e, o.e); return *this; }
    ~Event() { if (e) cudaEventDestroy(e); }
    int create(unsigned flags) { CUDA_TRY(cudaEventCreateWithFlags(&e, flags)); return ABB_OK; }
    operator cudaEvent_t() const { return e; }
};

// One global-bitmap walk tier: per-warp slots, each a visited bitmap over all nodes and a bounded queue with parents and depths.
// alloc: `n_slots` slots of `words` bitmap words and `queue_cap` queue entries each, bitmaps cleared.
struct GlobalSlots {
    DevBuf bitmap, queue, par, dep;
    int slots = 0; int64_t qcap = 0;
    int alloc(int n_slots, int64_t words, int64_t queue_cap) {
        slots = n_slots; qcap = queue_cap;
        const size_t sl = static_cast<size_t>(slots);
        int rc = ABB_OK;
        ENS(bitmap, sl * words * 4); ENS(queue, sl * qcap * 4); ENS(par, sl * qcap * 4); ENS(dep, sl * qcap * 4);
        if (rc) return rc;
        CUDA_TRY(cudaMemset(bitmap.p, 0, sl * words * 4));
        return ABB_OK;
    }
    void wire(WalkArgs &A, int64_t words) const {
        A.g_bitmap = bitmap.as<uint32_t>(); A.g_queue = queue.as<int32_t>(); A.g_par = par.as<int32_t>(); A.g_dep = dep.as<int32_t>();
        A.g_words = words; A.g_qcap = qcap;
    }
};

// Everything the storage tiers of a walk need (enqueue_tiers)
struct WalkTiers {
    // tier bookkeeping: CTL_WORDS counters; the hand-off lists of S1 (two-ended), the mid tier, the big tier and G1
    DevBuf ctl, ov[4];
    // block tiers (walkb.cuh): mid = 8 warps, queue + table in shared memory; big = 32 warps, 192 KB table, queue in a global scratch slot per block
    int block_tiers = 2;              // bit 0: mid tier (off by default: measured no faster than G1), bit 1: big tier (ABB_BLOCK_TIERS / abb_graph_set_option)
    int mid_slots = 8192, mid_qcap = 4096, big_slots = 49152, big_qcap = 36864;
    int big_grid = 0, mid_warps = 8;  // ABB_MID_WARPS=4: 4-warp mid blocks
    int64_t big_limit = 0;            // the big tier takes S1's heavy hand-offs when there are at most this many (default 24 per SM)
    DevBuf b_gq, b_gpar, b_gdep;
    // tier G1: many per-warp slots (bitmap over all nodes + a bounded queue); tier GX: a few slots that can hold a whole-graph walk
    GlobalSlots g1, gx; int64_t g_words = 0;
    int s1_minb = 5;
    int slice_align = 0;        // set while a host-mapped arena is the walk target
    bool align_direct = true;
};

// root-frontier de-duplication workspace
struct DedupWorkspace {
    DevBuf sig, ssig, q, sq, head, gid, hp, glen, goff, arena, memoff, memsrc, memstate, indiv, cnt, tmp;
    DevBuf gstart, gcount, gmaxd, gflags, ghist, lkey, lkey2, lgid, order;
    bool enabled = true;
    bool locality_order = true;   // walk the frontier groups in first-seed order (ABB_LOCALITY=0 disables)
    bool last_walk = false;       // the last walk was de-duplicated
};

// host-API staging of one walk
struct WalkStaging {
    DevBuf roots, root_off, targets, qstart, qcount, qmaxd, qflags, qestart, qecount, qhist;
    DevBuf nodes, parent, depth, edges, totals, hist_info_dev, hist_packed;
    unsigned long long hist_info[2] = {0, 0};   // column mask, largest count of the walk just staged
    bool hist_info_valid = false;
    bool hist_pack = true;      // host results carry only the non-zero histogram columns at the narrowest width (histpack.cuh)
    bool zero_copy = true;      // host-API walks write the node arena straight into pinned host memory when its size is known
    int64_t hint_nodes = 0, hint_edges = 0, hint_nq = 0, hint_last_nodes = 0;
    // size hint of the last PLAIN host walk (single roots, no parents / depths / edges), per spec: what the chunked path sizes its arenas from
    abb_walk_spec plain_spec{};
    int64_t plain_nq = -1, plain_nodes = 0;
    int64_t last_walk_queries = 0;
    Event ev_copy, ev_start, ev_end; bool timed = false;   // result copies wait for ev_copy; ev_start .. ev_end time the last walk
};

// chunked host walks (walk_host_chunked): a large plain batch is walked in `chunks` consecutive source ranges; each range's node arena
// is DMA-copied to the host while the next range is walked (two device arenas, ping-pong)
struct ChunkedWalk {
    int chunks = 8;                  // ABB_CHUNKS / option "chunks"; applies to batches of >= chunk_min queries (measured at L: 1 piece 43.9 ms, 4: 42.4, 8: 40.6)
    int64_t chunk_min = 2 << 20;
    DevBuf nodes_alt, roots, sig, key, key2, idx, order, counts, tmp, qstart, qcount, qmaxd, qflags, qhist;
    Event ev_walked, ev_copied[2];
    std::vector<int64_t> hint; int64_t hint_nq = -1;   // nodes each chunk produced last time (same batch size / chunk count)
    int last_host_chunks = 1;        // how many ranges the last host-buffer walk was split into (get_option "last_host_chunks")
};

// graph-constant tables of the exposure paths, built on first use (ensure_exposure_tables)
struct ExposureTables {
    // server tables: fan-out, and the principal rows each server contributes to a template
    DevBuf srv_cred, srv_tool, srv_roff, srv_row, srv_rel;
    // exposure tables: links of every finding node, templates of every vulnerable source, rows per finding node
    DevBuf vs, loff, link, rows, toff, trow, trel, overflow;
};

// exposure-path per-call workspace
struct PathsWorkspace {
    DevBuf findings, f_off, scan_tmp;
    // rows and links per finding; the host result's batch links and templates
    DevBuf f_cnt, f_link, f_lcnt, link_off, link_vs, link_rel, link_roff, link_toff, need, ulist, nu, t_cnt, t_off, t_off_node, t_row, t_rel;
    PathsArgs args{}; bool args_valid = false;   // the count pass's arguments, for the fill pass
    int replicate_grid = 0, rank_keys_grid = 0;   // grids of the row-parallel kernels (row_grid)
    Event ev_start, ev_end; bool timed = false;   // time the last count + fill
};

// finding-context workspace (context.cuh): per-finding bucket counts, totals, start offsets, source lists; the context kernels run on
// paths_stream next to the impact walk (staged: the findings are on the device), ev time the count and fill passes
struct ContextWorkspace {
    DevBuf bcnt, cnt, start, src;
    Event staged, ev[4];
};

struct abb_graph {
    int device = 0;
    GraphView v{};
    int64_t bytes = 0;
    int sm_count = 132;               // H100 SXM; set from the device in graph_finish_init
    mutable std::mutex mu;            // serialises use of the workspaces and of the snapshot tables
    cudaStream_t stream = nullptr;    // host-API stream
    cudaStream_t copy_stream = nullptr;   // result copies that may overlap later kernels of the same call
    cudaStream_t paths_stream = nullptr;  // exposure-path pipeline of abb_exposure_host, run next to the walk
    int64_t nx_batch = 0;             // cap on betweenness sources per batch and on path-search slots (0: sized from free memory)
    DevBuf identity_rank;
    // the walk's workspaces, then the path pipeline's and the finding context's (abb_exposure_host: who may use which, and when)
    WalkTiers tiers; DedupWorkspace dedup; WalkStaging staging; ChunkedWalk chunked;
    std::unique_ptr<ExposureTables> exposure;     // null: not built
    PathsWorkspace paths; ContextWorkspace context;
    // snapshot tables, one owner per feature, each type declared in its *_host.inl.  A null table is not built; a rebuild drops the old
    // table, builds a new one aside and installs it only once every step has succeeded.  Read and replaced under mu.
    std::unique_ptr<ClusterTable> clusters;
    std::unique_ptr<DeltaTable> delta;
    int64_t dl_union_limit = DL_UNION_LIMIT;
    std::unique_ptr<LookupState> lookup;
    std::unique_ptr<SearchState> search;
    std::unique_ptr<ComplianceTable> compliance;
    // graph arrays of an uploaded graph (an adopted graph's belong to the caller)
    std::vector<DevBuf> owned_arrays;

    ~abb_graph();   // defined after the *_host.inl files, where the snapshot-table types are complete
};

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int graph_finish_init(abb_graph *g) {
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, g->device));
    g->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g->copy_stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g->paths_stream, cudaStreamNonBlocking));
    for (Event *e : {&g->staging.ev_copy, &g->chunked.ev_walked, &g->chunked.ev_copied[0], &g->chunked.ev_copied[1], &g->context.staged})
        if (int rc = e->create(cudaEventDisableTiming)) return rc;
    for (Event *e : {&g->staging.ev_start, &g->staging.ev_end, &g->paths.ev_start, &g->paths.ev_end, &g->context.ev[0], &g->context.ev[1], &g->context.ev[2], &g->context.ev[3]})
        if (int rc = e->create(cudaEventDefault)) return rc;
    WalkTiers &wt = g->tiers;
    if (int rc = wt.ctl.ensure(CTL_WORDS * sizeof(unsigned long long))) return rc;
    const int64_t n = g->v.n;
    wt.g_words = (n + 31) / 32 + 1;
    // tier G1: 40 warps per SM (latency-bound pointer chasing wants every warp it can get), queue bounded at 64K entries
    int g1_slots = g->sm_count * 40;
    if (const char *e = getenv("ABB_G1_WARPS_PER_SM")) g1_slots = g->sm_count * std::max(4, std::min(48, atoi(e)));
    if (int rc = wt.g1.alloc(g1_slots, wt.g_words, std::min<int64_t>(n + 4096, 1 << 16))) return rc;
    // tier GX: 8 slots that can hold any walk (every node once + re-seeded roots)
    if (int rc = wt.gx.alloc(8, wt.g_words, n + 4096)) return rc;
    if (const char *e = getenv("ABB_DEDUP")) g->dedup.enabled = atoi(e) != 0;
    if (const char *e = getenv("ABB_BLOCK_TIERS")) wt.block_tiers = atoi(e) & 3;
    if (const char *e = getenv("ABB_LOCALITY")) g->dedup.locality_order = atoi(e) != 0;
    wt.big_grid = g->sm_count;
    wt.big_limit = 24ll * g->sm_count;
    if (const char *e = getenv("ABB_BIG_LIMIT")) wt.big_limit = atoll(e);
    if (const char *e = getenv("ABB_MID_WARPS")) wt.mid_warps = atoi(e) == 4 ? 4 : 8;
    if (const char *e = getenv("ABB_S1_MINB")) wt.s1_minb = atoi(e) == 4 ? 4 : 5;
    if (const char *e = getenv("ABB_ZEROCOPY")) g->staging.zero_copy = atoi(e) != 0;
    if (const char *e = getenv("ABB_HIST_PACK")) g->staging.hist_pack = atoi(e) != 0;
    if (const char *e = getenv("ABB_CHUNKS")) g->chunked.chunks = std::max(1, std::min(64, atoi(e)));
    if (const char *e = getenv("ABB_CHUNK_MIN")) g->chunked.chunk_min = std::max<int64_t>(2, atoll(e));
    if (const char *e = getenv("ABB_ALIGN_DIRECT")) wt.align_direct = atoi(e) != 0;
    if (!g->v.rank) {
        if (int rc = g->identity_rank.ensure(static_cast<size_t>(n + 1) * 4)) return rc;
        std::vector<int32_t> id(static_cast<size_t>(n));
        for (int64_t i = 0; i < n; i++) id[i] = static_cast<int32_t>(i);
        CUDA_TRY(cudaMemcpy(g->identity_rank.p, id.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice));
        g->v.rank = g->identity_rank.as<int32_t>();
    }
    return ABB_OK;
}

static int check_csr(const abb_csr *c) {
    if (!c) return fail(ABB_ERR_ARG, "null csr");
    if (c->n_nodes < 0 || c->n_entries < 0) return fail(ABB_ERR_ARG, "negative sizes");
    if (!c->fwd_off || !c->rev_off || !c->node_type) return fail(ABB_ERR_ARG, "missing csr arrays");
    if (c->n_entries > 0 && (!c->fwd_nbr || !c->fwd_meta || !c->fwd_eid || !c->rev_nbr || !c->rev_meta || !c->rev_eid))
        return fail(ABB_ERR_ARG, "missing csr entry arrays");
    return ABB_OK;
}

static void view_from_csr(GraphView &v, const abb_csr *c) {
    v.n = c->n_nodes; v.m = c->n_entries;
    v.foff = c->fwd_off; v.fnbr = c->fwd_nbr; v.fmeta = c->fwd_meta; v.feid = c->fwd_eid;
    v.roff = c->rev_off; v.rnbr = c->rev_nbr; v.rmeta = c->rev_meta; v.reid = c->rev_eid;
    v.ntype = c->node_type; v.rank = c->node_rank;
}

extern "C" int abb_graph_upload(int device, const abb_csr *host, abb_graph **out) {
    if (!out) return fail(ABB_ERR_ARG, "null out");
    if (int rc = check_csr(host)) return rc;
    if (abb_device_count() <= device || device < 0) return fail(ABB_ERR_CUDA, "no CUDA device %d (this library has no CPU fallback)", device);
    DeviceGuard dg(device);
    abb_graph *g = new abb_graph();
    g->device = device;
    abb_csr d = *host;
    const size_t n1 = static_cast<size_t>(host->n_nodes) + 1, m = static_cast<size_t>(host->n_entries);
    auto up = [&](const void *src, size_t bytes, const void **dstp) -> int {
        DevBuf &b = g->owned_arrays.emplace_back();
        if (int rc = b.alloc(bytes)) return rc;
        if (bytes) { cudaError_t e = cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice); if (e != cudaSuccess) return fail(ABB_ERR_CUDA, "H2D: %s", cudaGetErrorString(e)); }
        g->bytes += static_cast<int64_t>(bytes);
        *dstp = b.p;
        return ABB_OK;
    };
    int rc = ABB_OK;
#define UP(field, bytes) if (!rc) rc = up(host->field, (bytes), reinterpret_cast<const void **>(&d.field))
    UP(fwd_off, n1 * 4); UP(fwd_nbr, m * 4); UP(fwd_meta, m); UP(fwd_eid, m * 4);
    UP(rev_off, n1 * 4); UP(rev_nbr, m * 4); UP(rev_meta, m); UP(rev_eid, m * 4);
    UP(node_type, n1 - 1);
    if (host->node_rank) { UP(node_rank, (n1 - 1) * 4); }
#undef UP
    if (!rc) { view_from_csr(g->v, &d); rc = graph_finish_init(g); }
    if (rc) { abb_graph_free(g); return rc; }
    *out = g;
    return ABB_OK;
}

extern "C" int abb_graph_adopt(int device, const abb_csr *dev, abb_graph **out) {
    if (!out) return fail(ABB_ERR_ARG, "null out");
    if (int rc = check_csr(dev)) return rc;
    if (abb_device_count() <= device || device < 0) return fail(ABB_ERR_CUDA, "no CUDA device %d (this library has no CPU fallback)", device);
    DeviceGuard dg(device);
    abb_graph *g = new abb_graph();
    g->device = device;
    view_from_csr(g->v, dev);
    g->bytes = (static_cast<int64_t>(dev->n_nodes) + 1) * 8 + dev->n_entries * 18 + dev->n_nodes * 5;
    int rc = graph_finish_init(g);
    if (rc) { abb_graph_free(g); return rc; }
    *out = g;
    return ABB_OK;
}

extern "C" int abb_graph_view(const abb_graph *g, abb_csr *out) {
    if (!g || !out) return fail(ABB_ERR_ARG, "null argument");
    out->n_nodes = g->v.n; out->n_entries = g->v.m;
    out->fwd_off = g->v.foff; out->fwd_nbr = g->v.fnbr; out->fwd_meta = g->v.fmeta; out->fwd_eid = g->v.feid;
    out->rev_off = g->v.roff; out->rev_nbr = g->v.rnbr; out->rev_meta = g->v.rmeta; out->rev_eid = g->v.reid;
    out->node_type = g->v.ntype; out->node_rank = g->v.rank;
    return ABB_OK;
}
extern "C" int64_t abb_graph_bytes(const abb_graph *g) { return g ? g->bytes : 0; }
extern "C" int abb_graph_set_dedup(abb_graph *g, int enabled) {
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    std::lock_guard<std::mutex> lk(g->mu);
    g->dedup.enabled = enabled != 0;
    return ABB_OK;
}
extern "C" int abb_graph_device(const abb_graph *g) { return g ? g->device : -1; }

// The member behind one option, whatever its type: a flag stores value != 0, an int stores value & mask
struct OptionRef {
    bool *flag = nullptr; int *i32 = nullptr; int64_t *i64 = nullptr; int mask = -1;
    OptionRef(bool &m) : flag(&m) {}
    OptionRef(int &m, int mask_ = -1) : i32(&m), mask(mask_) {}
    OptionRef(int64_t &m) : i64(&m) {}
    int64_t get() const { return flag ? *flag : i32 ? *i32 : *i64; }
    void set(int64_t value) const { if (flag) *flag = value != 0; else if (i32) *i32 = static_cast<int>(value) & mask; else *i64 = value; }
};

// Tuning / test switches of a graph handle.  Results never depend on them (every tier is bit-identical; the GPU tests
// run the suite with the block tiers on, off and shrunk so that every hand-off between tiers is exercised).
// set_option accepts values in [lo, hi] and otherwise fails with `range`; a null `range` marks a read-only option.
static const struct GraphOption {
    const char *name; OptionRef (*member)(abb_graph &g); int64_t lo, hi; const char *range;
} g_options[] = {
    {"dedup", [](abb_graph &g) { return OptionRef(g.dedup.enabled); }, INT64_MIN, INT64_MAX, ""},
    {"block_tiers", [](abb_graph &g) { return OptionRef(g.tiers.block_tiers, 3); }, INT64_MIN, INT64_MAX, ""},
    {"mid_qcap", [](abb_graph &g) { return OptionRef(g.tiers.mid_qcap); }, 32, 4096, "mid_qcap must be in [32, 4096]"},
    {"big_qcap", [](abb_graph &g) { return OptionRef(g.tiers.big_qcap); }, 32, 36864, "big_qcap must be in [32, 36864]"},
    {"zero_copy", [](abb_graph &g) { return OptionRef(g.staging.zero_copy); }, INT64_MIN, INT64_MAX, ""},
    {"hist_pack", [](abb_graph &g) { return OptionRef(g.staging.hist_pack); }, INT64_MIN, INT64_MAX, ""},
    {"chunks", [](abb_graph &g) { return OptionRef(g.chunked.chunks); }, 1, 64, "chunks must be in [1, 64]"},
    {"chunk_min", [](abb_graph &g) { return OptionRef(g.chunked.chunk_min); }, 2, INT64_MAX, "chunk_min must be >= 2"},
    {"last_host_chunks", [](abb_graph &g) { return OptionRef(g.chunked.last_host_chunks); }, 0, 0, nullptr},
    {"big_limit", [](abb_graph &g) { return OptionRef(g.tiers.big_limit); }, 0, INT64_MAX, "big_limit must be >= 0"},
    {"nx_batch", [](abb_graph &g) { return OptionRef(g.nx_batch); }, 0, INT64_MAX, "nx_batch must be >= 0"},
    {"delta_union_limit", [](abb_graph &g) { return OptionRef(g.dl_union_limit); }, 0, DL_UNION_LIMIT, "delta_union_limit must be in [0, 2^27]"},
};

static const GraphOption *find_option(const char *name) {
    for (const GraphOption &o : g_options) if (strcmp(o.name, name) == 0) return &o;
    return nullptr;
}

extern "C" int abb_graph_set_option(abb_graph *g, const char *name, int64_t value) {
    if (!g || !name) return fail(ABB_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(g->mu);
    const GraphOption *o = find_option(name);
    if (!o || !o->range) return fail(ABB_ERR_ARG, "unknown option '%s'", name);
    if (value < o->lo || value > o->hi) return fail(ABB_ERR_ARG, "%s", o->range);
    o->member(*g).set(value);
    return ABB_OK;
}
extern "C" int64_t abb_graph_get_option(const abb_graph *g, const char *name) {
    if (!g || !name) return -1;
    std::lock_guard<std::mutex> lk(g->mu);
    const GraphOption *o = find_option(name);
    return o ? o->member(const_cast<abb_graph &>(*g)).get() : -1;   // only read
}

extern "C" void abb_graph_free(abb_graph *g) {
    if (!g) return;
    DeviceGuard dg(g->device);
    { std::lock_guard<std::mutex> lk(g->mu); }      // a host-API call still inside the library finishes before the teardown starts
    delete g;
}

// ------------------------------------------------------------------ walk specs (reference function -> spec)
static abb_walk_spec spec_base() {
    abb_walk_spec s; memset(&s, 0, sizeof s);
    s.direction = ABB_DIR_FORWARD; s.max_depth = 4; s.rel_mask = 0xFFFFFFFFu; s.max_nodes = -1; s.max_edges = -1; s.emit_types = 0xFFFFFFFFu;
    return s;
}
extern "C" abb_walk_spec abb_spec_impact_of(int32_t max_depth) {
    abb_walk_spec s = spec_base();
    s.direction = ABB_DIR_REVERSE; s.max_depth = max_depth < 0 ? 0 : max_depth;   // all relationships, traversable ignored
    s.flags = ABB_WALK_MARK_ROOTS | ABB_WALK_OMIT_ROOTS | ABB_WALK_HIST | ABB_WALK_REAL_ROOTS;
    return s;
}
extern "C" abb_walk_spec abb_spec_bfs(int32_t max_depth, int32_t traversable_only) {
    abb_walk_spec s = spec_base();
    // nodes at depth max_depth+1 are marked visited but never emitted (container.py:381-390): invisible, so walk to max_depth
    s.max_depth = max_depth < 0 ? 0 : max_depth;
    s.flags = ABB_WALK_MARK_ROOTS | ABB_WALK_OMIT_ROOTS | ABB_WALK_PARENTS | ABB_WALK_REAL_ROOTS | (traversable_only ? ABB_WALK_TRAVERSABLE_ONLY : 0);
    return s;
}
extern "C" abb_walk_spec abb_spec_reachable_from(int32_t max_depth, int32_t traversable_only) {
    abb_walk_spec s = spec_base();
    s.max_depth = max_depth < 0 ? 0 : max_depth;
    s.flags = ABB_WALK_MARK_ROOTS | ABB_WALK_OMIT_ROOTS | ABB_WALK_REAL_ROOTS | (traversable_only ? ABB_WALK_TRAVERSABLE_ONLY : 0);
    return s;
}
extern "C" abb_walk_spec abb_spec_shortest_path(void) {
    abb_walk_spec s = spec_base();
    s.max_depth = -1;
    s.flags = ABB_WALK_MARK_ROOTS | ABB_WALK_PARENTS | ABB_WALK_REAL_ROOTS | ABB_WALK_TARGET;
    return s;
}
extern "C" abb_walk_spec abb_spec_traverse_subgraph(int32_t direction, int32_t max_depth, int64_t max_nodes, int64_t max_edges, int32_t traversable_only,
                                                    uint32_t rel_mask, int32_t static_only, int32_t dynamic_only, int32_t include_roots) {
    abb_walk_spec s = spec_base();
    const uint32_t dyn = (1u << 26) | (1u << 27) | (1u << 28);   // invoked, accessed, delegated_to (container.py:777)
    s.direction = direction; s.max_depth = max_depth < 0 ? 0 : max_depth;
    s.max_nodes = max_nodes; s.max_edges = max_edges;
    uint32_t m = rel_mask ? rel_mask : 0xFFFFFFFFu;
    if (static_only) m &= ~dyn;
    if (dynamic_only) m &= dyn;
    s.rel_mask = m;
    s.flags = ABB_WALK_DEPTHS | ABB_WALK_EDGES | ABB_WALK_REAL_ROOTS | (include_roots ? ABB_WALK_MARK_ROOTS : 0) | (traversable_only ? ABB_WALK_TRAVERSABLE_ONLY : 0);
    return s;
}
extern "C" abb_walk_spec abb_spec_distances_along(uint32_t rel_mask, uint32_t emit_types) {
    abb_walk_spec s = spec_base();
    s.max_depth = -1; s.rel_mask = rel_mask;
    s.flags = ABB_WALK_MARK_ROOTS | ABB_WALK_OMIT_ROOTS | ABB_WALK_DEPTHS;
    s.emit_types = emit_types ? emit_types : 0xFFFFFFFFu;
    return s;
}

// ------------------------------------------------------------------ walk dispatch
constexpr int S1_H = 1024, S1_Q = 256, S1_WARPS = 8;      // 256 four-slot buckets, 256-entry queue per warp (5.4 KB): 40 warps per SM

template <int H, int Q, int WARPS, bool PAR, bool META, bool BUD, int MINB>
static int launch_smem(const abb_graph *g, const WalkArgs &A, int64_t max_items, cudaStream_t st) {
    auto kern = walk_smem_kernel<H, Q, PAR, META, BUD, WARPS, MINB>;
    constexpr int stride = (SmemStore<H, Q, PAR>::kBytes + 15) & ~15;
    const int smem = stride * WARPS;
    static thread_local int occ_cache = -1;  // per instantiation
    if (occ_cache < 0) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        int occ = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, WARPS * 32, smem));
        occ_cache = std::max(1, occ);
    }
    int64_t grid = static_cast<int64_t>(g->sm_count) * occ_cache;
    int64_t need = (max_items + static_cast<int64_t>(WARPS) * WORK_CHUNK - 1) / (static_cast<int64_t>(WARPS) * WORK_CHUNK);
    grid = std::max<int64_t>(1, std::min(grid, need));
    return LAUNCH(kern, static_cast<unsigned>(grid), WARPS * 32, smem, st, A);
}

template <int H, int Q, int WARPS>
static int launch_smem_variant(const abb_graph *g, const WalkArgs &A, int64_t max_items, bool par, bool meta, bool bud, cudaStream_t st) {
    // MINB: resident blocks the register allocation aims for — 5 (48 registers, 40 warps/SM) or 4 (64 registers, 32 warps/SM; ABB_S1_MINB=4)
#define V(P, M, B) if (par == P && meta == M && bud == B) return g->tiers.s1_minb == 4 ? launch_smem<H, Q, WARPS, P, M, B, 4>(g, A, max_items, st) : launch_smem<H, Q, WARPS, P, M, B, 5>(g, A, max_items, st)
    V(false, false, false); V(false, false, true); V(false, true, false); V(false, true, true);
    V(true, false, false); V(true, false, true); V(true, true, false); V(true, true, true);
#undef V
    return fail(ABB_ERR_ARG, "unreachable");
}

static int launch_global_variant(const WalkArgs &A, int slots, int sm_count, bool meta, bool bud, cudaStream_t st) {
    const int blocks = std::max(1, slots / 4);
    const bool dense = slots > sm_count * 40;      // more than 40 warps per SM: the 40-register build (12 blocks of 4 warps per SM)
    void (*kern)(WalkArgs);
    if (dense) {
        if (meta && bud) kern = walk_global_kernel<true, true, 12>;
        else if (meta) kern = walk_global_kernel<true, false, 12>;
        else if (bud) kern = walk_global_kernel<false, true, 12>;
        else kern = walk_global_kernel<false, false, 12>;
    } else if (meta && bud) kern = walk_global_kernel<true, true, 10>;
    else if (meta) kern = walk_global_kernel<true, false, 10>;
    else if (bud) kern = walk_global_kernel<false, true, 10>;
    else kern = walk_global_kernel<false, false, 10>;
    return LAUNCH(kern, blocks, 128, 0, st, A);
}

template <int W, bool QSM, bool PAR, bool META, int MINB>
static int launch_block(const abb_graph *g, const WalkArgs &A, const BlockTier &T, int grid_cap, cudaStream_t st) {
    auto kern = walk_block_kernel<W, QSM, PAR, META, MINB>;
    size_t smem = static_cast<size_t>(T.slots) * 4;
    if (QSM) smem += static_cast<size_t>(T.qcap) * (PAR ? 9 : 5);
    smem = (smem + 15) & ~static_cast<size_t>(15);
    static thread_local int occ_cache = -1;   // per instantiation
    static thread_local size_t smem_cache = 0;
    if (occ_cache < 0 || smem_cache != smem) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        int occ = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, W * 32, smem));
        occ_cache = std::max(1, occ); smem_cache = smem;
    }
    int grid = g->sm_count * occ_cache;
    if (grid_cap > 0) grid = std::min(grid, grid_cap);
    return LAUNCH(kern, static_cast<unsigned>(grid), W * 32, smem, st, A, T);
}

// Up to five tiers on one stream.  `A` carries spec/io and the first tier's work list (qlist/nq/nq_dev); every later
// tier reads its work list and count from device memory, so nothing here waits for the GPU.
//   S1  warp  + shared-memory bucketed hash/queue   (<= 256 queue entries)
//   B   block (32 warps) + 192 KB shared-memory hash, queue in global scratch (<= 36864)  — walkb.cuh, plain walks: takes S1's HEAVY hand-offs
//       (its own hand-offs form a second list the next tier reads after S1's)
//   M   block (4/8 warps) + shared-memory hash/queue (<= 2048/4096 entries)                — walkb.cuh, plain walks: S1's other hand-offs
//   G1  warp  + global bitmap, bounded queue slot   (<= 64K queue entries), 40 warps per SM (ABB_G1_WARPS_PER_SM)
//   GX  warp  + global bitmap, whole-graph slot     (anything)
// "plain" = no node/edge budget, no target stop, no recorded edges; the others go S1 -> G1 -> GX.
// S1 writes a TWO-ENDED hand-off list: queries a forecast calls heavy (roots or one level hold more candidates than the queue) from
// the front, the rest from the back.  Heavy ones go to the big block tier when it is on;
// otherwise G1 takes the front part first, so the long walks start at once instead of landing behind thousands of short ones.
// ctl: tier t uses ctl[4t .. 4t+3] = {work cursor, hand-off count (front), fatal flag, hand-off count (back)}; a skipped tier's stay zero.
static int enqueue_tiers(abb_graph *g, WalkArgs A, int64_t max_items, unsigned long long *ctl, cudaStream_t st) {
    NvtxRange nvtx_("walk: storage tiers");
    const uint32_t fl = A.spec.flags;
    const bool par = fl & ABB_WALK_PARENTS;
    const bool meta = A.spec.rel_mask != 0xFFFFFFFFu || (fl & ABB_WALK_TRAVERSABLE_ONLY);
    const bool bud = A.spec.max_nodes >= 0 || A.spec.max_edges >= 0;
    WalkTiers &wt = g->tiers;
    int32_t *ovs[4] = {wt.ov[0].as<int32_t>(), wt.ov[1].as<int32_t>(), wt.ov[2].as<int32_t>(), wt.ov[3].as<int32_t>()};
    A.list_cap = max_items;
    A.slice_align = wt.slice_align;
    // S1: two-ended hand-off list in ovs[0]
    A.ctl = ctl; A.overflow = ovs[0]; A.ov_cnt_front = ctl + 1; A.ov_cnt_back = ctl + 3;
    if (int rc = launch_smem_variant<S1_H, S1_Q, S1_WARPS>(g, A, max_items, par, meta, bud, st)) return rc;
    const int idb = ceil_log2_i64(std::max<int64_t>(g->v.n, 2));
    const bool plain = !bud && !(fl & (ABB_WALK_TARGET | ABB_WALK_EDGES));
    bool front_taken = false;                       // S1's heavy part routed (to the big tier when few, else first in line for the warp tier)
    unsigned long long *to_big = ctl + CTL_ROUTE, *to_warp = ctl + CTL_ROUTE + 1;
    if (plain && (wt.block_tiers & 2) && idb <= 26) {
        if (int rc = LAUNCH(route_heavy_kernel, 1, 1, 0, st, ctl + 1, to_big, to_warp, static_cast<unsigned long long>(wt.big_limit))) return rc;
        // big tier: the heavy (front) part of S1's list; what it cannot hold goes to a list of its own (ovs[2]) that the next tier
        // reads after S1's back part — NOT onto S1's list: front + back may already fill it
        A.qlist = ovs[0]; A.nq = 0; A.nq_dev = to_big; A.nq_back_dev = nullptr; A.ctl = ctl + 4 * 1;
        A.overflow = ovs[2]; A.ov_cnt_front = ctl + 4 * 1 + 1; A.ov_cnt_back = nullptr;
        const size_t words = static_cast<size_t>(wt.big_grid) * wt.big_qcap;
        if (int rc = wt.b_gq.ensure(words * 4)) return rc;
        if (par) if (int rc = wt.b_gpar.ensure(words * 4)) return rc;
        if (fl & ABB_WALK_DEPTHS) if (int rc = wt.b_gdep.ensure(words * 4)) return rc;
        BlockTier T{static_cast<uint32_t>(wt.big_slots), wt.big_qcap, idb, wt.b_gq.as<int32_t>(), wt.b_gpar.as<int32_t>(), wt.b_gdep.as<int32_t>()};
        int rc = meta ? launch_block<32, false, true, true, 1>(g, A, T, wt.big_grid, st) : launch_block<32, false, true, false, 1>(g, A, T, wt.big_grid, st);
        if (rc) return rc;
        front_taken = true;
    }
    // what the next tier reads: S1's list (its back part, or front then back), or the mid tier's plain list
    const unsigned long long *in_front = front_taken ? to_warp : ctl + 1, *in_back = ctl + 3;
    int32_t *in_list = ovs[0];
    const int32_t *in_list2 = front_taken ? ovs[2] : nullptr;
    const unsigned long long *in_cnt2 = front_taken ? ctl + 4 * 1 + 1 : nullptr;
    if (plain && (wt.block_tiers & 1) && idb <= 28) {
        A.qlist = in_list; A.nq = 0; A.nq_dev = in_front; A.nq_back_dev = in_back; A.qlist2 = in_list2; A.nq2_dev = in_cnt2; A.ctl = ctl + 4 * 2;
        A.overflow = ovs[1]; A.ov_cnt_front = ctl + 4 * 2 + 1; A.ov_cnt_back = nullptr;
        BlockTier T{static_cast<uint32_t>(wt.mid_slots), wt.mid_qcap, idb, nullptr, nullptr, nullptr};
        int rc;
        if (wt.mid_warps == 4) {               // 4-warp blocks: half the table / queue, twice the walks in flight per SM
            T.slots = static_cast<uint32_t>(std::min(wt.mid_slots, 4096)); T.qcap = std::min(wt.mid_qcap, 2048);
            if (par && meta) rc = launch_block<4, true, true, true, 6>(g, A, T, 0, st);
            else if (par) rc = launch_block<4, true, true, false, 6>(g, A, T, 0, st);
            else if (meta) rc = launch_block<4, true, false, true, 8>(g, A, T, 0, st);
            else rc = launch_block<4, true, false, false, 8>(g, A, T, 0, st);
        } else if (par && meta) rc = launch_block<8, true, true, true, 3>(g, A, T, 0, st);
        else if (par) rc = launch_block<8, true, true, false, 3>(g, A, T, 0, st);
        else if (meta) rc = launch_block<8, true, false, true, 4>(g, A, T, 0, st);
        else rc = launch_block<8, true, false, false, 4>(g, A, T, 0, st);
        if (rc) return rc;
        in_list = ovs[1]; in_front = ctl + 4 * 2 + 1; in_back = nullptr; in_list2 = nullptr; in_cnt2 = nullptr;
    }
    // G1
    A.qlist = in_list; A.nq = 0; A.nq_dev = in_front; A.nq_back_dev = in_back; A.qlist2 = in_list2; A.nq2_dev = in_cnt2; A.ctl = ctl + 4 * 3;
    A.overflow = ovs[3]; A.ov_cnt_front = ctl + 4 * 3 + 1; A.ov_cnt_back = nullptr;
    wt.g1.wire(A, wt.g_words);
    if (int rc = launch_global_variant(A, wt.g1.slots, g->sm_count, meta, bud, st)) return rc;
    // GX
    A.qlist = ovs[3]; A.nq_dev = ctl + 4 * 3 + 1; A.nq_back_dev = nullptr; A.qlist2 = nullptr; A.nq2_dev = nullptr; A.ctl = ctl + 4 * 4; A.overflow = nullptr; A.ov_cnt_front = A.ov_cnt_back = nullptr;
    wt.gx.wire(A, wt.g_words);
    return launch_global_variant(A, wt.gx.slots, g->sm_count, meta, bud, st);
}

static int check_walk_io(const abb_walk_spec *spec, const abb_walk_io *io) {
    if (!spec || !io) return fail(ABB_ERR_ARG, "null spec/io");
    if (io->n_queries < 0) return fail(ABB_ERR_ARG, "negative query count");
    if (!(spec->direction & 3)) return fail(ABB_ERR_ARG, "direction must be forward, reverse or both");
    if (io->n_queries >= (1ll << 31)) return fail(ABB_ERR_ARG, "too many queries in one batch");
    const uint32_t fl = spec->flags;
    if (!io->q_start || !io->q_count || !io->q_maxd || !io->q_flags || !io->totals || (!io->nodes && io->node_cap > 0))
        return fail(ABB_ERR_ARG, "missing walk outputs");
    if ((fl & ABB_WALK_PARENTS) && !io->parent) return fail(ABB_ERR_ARG, "PARENTS needs io.parent");
    if ((fl & ABB_WALK_DEPTHS) && !io->depth) return fail(ABB_ERR_ARG, "DEPTHS needs io.depth");
    if ((fl & ABB_WALK_EDGES) && (!io->q_estart || !io->q_ecount || (!io->edges && io->edge_cap > 0))) return fail(ABB_ERR_ARG, "EDGES needs edge outputs");
    if ((fl & ABB_WALK_HIST) && !io->q_hist) return fail(ABB_ERR_ARG, "HIST needs io.q_hist");
    if ((fl & ABB_WALK_TARGET) && !io->targets) return fail(ABB_ERR_ARG, "TARGET needs io.targets");
    return ABB_OK;
}

struct HeadToI64 { __host__ __device__ int64_t operator()(uint8_t v) const { return static_cast<int64_t>(v); } };

// Group single-source walks by their level-1 frontier, walk each group once, share the slice (dedup.cuh).
static int enqueue_dedup_walk(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, cudaStream_t st) {
    NvtxRange nvtx_("walk: root-frontier de-duplication + canonical / individual tiers");
    const int64_t nq = io->n_queries;
    const size_t q1 = static_cast<size_t>(nq) + 2;
    const uint32_t fl = spec->flags;
    int rc = ABB_OK;
    DedupWorkspace &D = g->dedup;
    ENS(D.sig, q1 * 8); ENS(D.ssig, q1 * 8); ENS(D.q, q1 * 4); ENS(D.sq, q1 * 4); ENS(D.head, q1); ENS(D.gid, q1 * 8); ENS(D.hp, q1 * 8);
    ENS(D.glen, q1 * 8); ENS(D.goff, q1 * 8); ENS(D.arena, q1 * 4 * L1_CAP); ENS(D.memoff, q1 * 8); ENS(D.memsrc, q1 * 4); ENS(D.memstate, q1 * 4);
    ENS(D.indiv, q1 * 4); ENS(D.cnt, 8 * sizeof(unsigned long long));
    ENS(D.lkey, q1 * 4); ENS(D.lkey2, q1 * 4); ENS(D.lgid, q1 * 4); ENS(D.order, q1 * 4);
    ENS(D.gstart, q1 * 8); ENS(D.gcount, q1 * 4); ENS(D.gmaxd, q1 * 4); ENS(D.gflags, q1 * 4);
    if (fl & ABB_WALK_HIST) { ENS(D.ghist, q1 * ABB_N_ENTITY_TYPES * 4); }
    if (rc) return rc;
    unsigned long long *cnt = D.cnt.as<unsigned long long>();
    unsigned long long *sig = D.sig.as<unsigned long long>(), *ssig = D.ssig.as<unsigned long long>();
    int32_t *qi = D.q.as<int32_t>(), *sq = D.sq.as<int32_t>(), *indiv = D.indiv.as<int32_t>();
    uint8_t *head = D.head.as<uint8_t>();
    int64_t *gid = D.gid.as<int64_t>(), *hp = D.hp.as<int64_t>(), *glen = D.glen.as<int64_t>(), *goff = D.goff.as<int64_t>();
    int64_t *memoff = D.memoff.as<int64_t>();
    const unsigned blocks = static_cast<unsigned>((nq + 255) / 256);
    CUDA_TRY(cudaMemsetAsync(cnt, 0, 8 * sizeof(unsigned long long), st));
    CUDA_TRY(cudaMemsetAsync(glen, 0, q1 * 8, st));
    if ((rc = LAUNCH(dedup_sig_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, nq, sig, qi))) return rc;
    if ((rc = cub_run(D.tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, sig, ssig, qi, sq, static_cast<int>(nq), 0, SIG_BITS, st); })))
        return rc;
    if ((rc = LAUNCH(dedup_heads_kernel, blocks, 256, 0, st, ssig, sq, nq, head, indiv, cnt))) return rc;
    cub::TransformInputIterator<int64_t, HeadToI64, const uint8_t *> head64(head, HeadToI64());
    if ((rc = cub_run(D.tmp, [&](void *t, size_t &b) { return cub::DeviceScan::InclusiveSum(t, b, head64, gid, static_cast<int>(nq), st); }))) return rc;
    if ((rc = select_flagged(D.tmp, head, hp, cnt, static_cast<int>(nq), st))) return rc;
    if ((rc = LAUNCH(dedup_groups_kernel, static_cast<unsigned>((nq + 1 + 255) / 256), 256, 0, st, g->v, *spec, io->roots, sq, hp, cnt, glen, memoff))) return rc;
    // glen is passed non-const here, unlike scan_i64's input: a different cub instantiation
    if ((rc = cub_run(D.tmp, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, glen, goff, static_cast<int>(nq + 1), st); }))) return rc;
    if ((rc = LAUNCH(dedup_roots_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, sq, hp, cnt, goff, D.arena.as<int32_t>()))) return rc;
    if ((rc = LAUNCH(dedup_members_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, sq, head, gid, goff, D.arena.as<int32_t>(), D.memsrc.as<int32_t>(),
                     D.memstate.as<int32_t>(), indiv, cnt)))
        return rc;
    unsigned long long *ctl = g->tiers.ctl.as<unsigned long long>();
    // canonical walks: one per group, seeded with the shared frontier, one level shallower, depths biased by one
    WalkArgs C{};
    C.g = g->v; C.spec = *spec; C.io = *io;
    C.spec.max_depth = spec->max_depth < 0 ? -1 : spec->max_depth - 1;
    C.spec.flags = (fl & ~(ABB_WALK_OMIT_ROOTS | ABB_WALK_REAL_ROOTS)) | ABB_WALK_MARK_ROOTS;
    C.io.roots = D.arena.as<int32_t>(); C.io.root_off = goff;
    C.io.q_start = D.gstart.as<int64_t>(); C.io.q_count = D.gcount.as<int32_t>(); C.io.q_maxd = D.gmaxd.as<int32_t>();
    C.io.q_flags = D.gflags.as<int32_t>(); C.io.q_hist = D.ghist.as<uint32_t>();
    C.qlist = nullptr; C.nq = 0; C.nq_dev = cnt;
    if (D.locality_order) {
        // walk order = first-seed order (a 2 M-key radix sort over the node-id bits, ~0.1 ms): neighbouring groups share rows in L2
        uint32_t *lkey = D.lkey.as<uint32_t>(), *lkey2 = D.lkey2.as<uint32_t>();
        int32_t *lgid = D.lgid.as<int32_t>(), *order = D.order.as<int32_t>();
        if ((rc = LAUNCH(dedup_locality_keys_kernel, blocks, 256, 0, st, cnt, goff, D.arena.as<int32_t>(), lkey, lgid, nq))) return rc;
        if ((rc = cub_run(D.tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, lkey, lkey2, lgid, order, static_cast<int>(nq), 0, 32, st); })))
            return rc;
        C.qlist = order;
    }
    C.depth_bias = 1; C.hist_roots = 1;
    C.mem_off = memoff; C.mem_src = D.memsrc.as<int32_t>(); C.mem_state = D.memstate.as<int32_t>();
    if ((rc = enqueue_tiers(g, C, nq, ctl, st))) return rc;
    if ((rc = LAUNCH(dedup_share_kernel, grid_for(nq, 256, g->sm_count, 8), 256, 0, st,
                     sq, gid, D.memstate.as<int32_t>(), cnt, C.io.q_start, C.io.q_count, C.io.q_maxd, C.io.q_flags, C.io.q_hist, io->q_start, io->q_count,
                     io->q_maxd, io->q_flags, (fl & ABB_WALK_HIST) ? io->q_hist : nullptr, indiv, cnt)))
        return rc;
    // individual walks: ineligible sources, signature collisions, sources reached by their own group's walk
    WalkArgs I{};
    I.g = g->v; I.spec = *spec; I.io = *io;
    I.qlist = indiv; I.nq = 0; I.nq_dev = cnt + 1;
    return enqueue_tiers(g, I, nq, ctl + CTL_SET, st);
}

static bool dedup_applies(const abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io) {
    const uint32_t fl = spec->flags;
    return g->dedup.enabled && !io->root_off && io->n_queries >= 256 && (fl & ABB_WALK_MARK_ROOTS) && (fl & ABB_WALK_OMIT_ROOTS) &&
           !(fl & (ABB_WALK_TARGET | ABB_WALK_EDGES | ABB_WALK_PARENTS)) && spec->max_nodes < 0 && spec->max_edges < 0 && spec->max_depth != 0;
}

static int enqueue_walk(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, cudaStream_t st) {
    if (int rc = check_walk_io(spec, io)) return rc;
    CUDA_TRY(cudaMemsetAsync(io->totals, 0, 2 * sizeof(unsigned long long), st));
    if (io->n_queries == 0) return ABB_OK;
    for (DevBuf &ov : g->tiers.ov) if (int rc = ov.ensure(static_cast<size_t>(io->n_queries) * 4)) return rc;
    CUDA_TRY(cudaMemsetAsync(g->tiers.ctl.p, 0, CTL_WORDS * sizeof(unsigned long long), st));
    g->staging.last_walk_queries = io->n_queries;
    g->dedup.last_walk = dedup_applies(g, spec, io);
    if (g->dedup.last_walk) return enqueue_dedup_walk(g, spec, io, st);
    WalkArgs A{};
    A.g = g->v; A.spec = *spec; A.io = *io;
    A.qlist = nullptr; A.nq = io->n_queries; A.nq_dev = nullptr;
    return enqueue_tiers(g, A, io->n_queries, g->tiers.ctl.as<unsigned long long>(), st);
}

extern "C" int abb_walk_launch(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, void *stream) {
    NvtxRange nvtx_("abb_walk_launch");
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaEventRecord(g->staging.ev_start, st));
    int rc = enqueue_walk(g, spec, io, st);
    if (rc) return rc;
    CUDA_TRY(cudaEventRecord(g->staging.ev_end, st));
    g->staging.timed = true;
    return ABB_OK;
}

extern "C" int abb_walk_signatures(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, int64_t n, unsigned long long *sig, void *stream) {
    if (!g || !spec || n < 0 || (n && (!roots || !sig))) return fail(ABB_ERR_ARG, "bad arguments");
    if (!n) return ABB_OK;
    DeviceGuard dg(g->device);
    return LAUNCH(dedup_sig_kernel, static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream), g->v, *spec, roots, n, sig, nullptr);
}

extern "C" float abb_last_walk_ms(abb_graph *g) {
    if (!g) return -1.f;
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);   // both events of one call: another thread's call records them under the lock
    if (!g->staging.timed) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(g->staging.ev_end) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, g->staging.ev_start, g->staging.ev_end) != cudaSuccess) return -1.f;
    return ms;
}
extern "C" int abb_last_walk_stats(abb_graph *g, int64_t *out4) {
    if (!g || !out4) return fail(ABB_ERR_ARG, "null argument");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    out4[0] = g->staging.last_walk_queries; out4[1] = out4[2] = out4[3] = 0;
    if (g->dedup.last_walk && g->dedup.cnt.p) {
        unsigned long long c[3] = {0, 0, 0};
        CUDA_TRY(cudaMemcpy(c, g->dedup.cnt.p, sizeof c, cudaMemcpyDeviceToHost));
        out4[1] = static_cast<int64_t>(c[0]); out4[2] = static_cast<int64_t>(c[1]); out4[3] = static_cast<int64_t>(c[2]);
    }
    return ABB_OK;
}

extern "C" int abb_last_walk_tier_counts(abb_graph *g, int64_t *out8) {
    if (!g || !out8) return fail(ABB_ERR_ARG, "null argument");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    unsigned long long c[CTL_WORDS];
    CUDA_TRY(cudaMemcpy(c, g->tiers.ctl.p, sizeof c, cudaMemcpyDeviceToHost));
    for (int set = 0; set < 2; set++) {
        const unsigned long long *k = c + set * CTL_SET;
        out8[set * 4 + 0] = static_cast<int64_t>(k[1] + k[3]);          // S1 hand-offs (heavy + other)
        out8[set * 4 + 1] = static_cast<int64_t>(k[1]);                 // of which heavy (to the big block tier, or first in line for G1)
        out8[set * 4 + 2] = static_cast<int64_t>(k[4 * 2 + 1]);         // mid block tier hand-offs
        out8[set * 4 + 3] = static_cast<int64_t>(k[4 * 3 + 1]);         // G1 hand-offs (to GX)
    }
    return ABB_OK;
}

extern "C" float abb_last_paths_ms(abb_graph *g) {
    if (!g) return -1.f;
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);   // both events of one call: another thread's call records them under the lock
    if (!g->paths.timed) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(g->paths.ev_end) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, g->paths.ev_start, g->paths.ev_end) != cudaSuccess) return -1.f;
    return ms;
}

// ------------------------------------------------------------------ walk, host-buffer form
struct abb_walk_result {
    int64_t nq = 0, total_nodes = 0, total_edges = 0, h2d = 0, d2h = 0;
    uint32_t flags = 0;
    HostBlock q_start, q_count, q_maxd, q_flags, q_estart, q_ecount, q_hist, nodes, parent, depth, edges;
    // histograms as shipped: k non-zero columns (bit set in hist_mask) of hist_width bytes per count; q_hist is rebuilt from it on demand
    HostBlock q_hist_packed;
    bool hist_is_packed = false, hist_expanded = false;
    uint32_t hist_mask = 0; int hist_k = 0, hist_width = 0;
    std::mutex mu;
};

extern "C" void abb_walk_result_free(abb_walk_result *r) { delete r; }
extern "C" int64_t abb_walk_result_queries(const abb_walk_result *r) { return r->nq; }
extern "C" int64_t abb_walk_result_total_nodes(const abb_walk_result *r) { return r->total_nodes; }
extern "C" int64_t abb_walk_result_total_edges(const abb_walk_result *r) { return r->total_edges; }
extern "C" const int64_t *abb_walk_result_start(const abb_walk_result *r) { return r->q_start.as<int64_t>(); }
extern "C" const int32_t *abb_walk_result_count(const abb_walk_result *r) { return r->q_count.as<int32_t>(); }
extern "C" const int32_t *abb_walk_result_maxd(const abb_walk_result *r) { return r->q_maxd.as<int32_t>(); }
extern "C" const int32_t *abb_walk_result_flags(const abb_walk_result *r) { return r->q_flags.as<int32_t>(); }
extern "C" const int64_t *abb_walk_result_estart(const abb_walk_result *r) { return r->q_estart.as<int64_t>(); }
extern "C" const int64_t *abb_walk_result_ecount(const abb_walk_result *r) { return r->q_ecount.as<int64_t>(); }
// packed columns -> the dense [nq x ABB_N_ENTITY_TYPES] uint32 table, once, threads over query ranges
static bool hist_expand(abb_walk_result *r) {
    std::lock_guard<std::mutex> lk(r->mu);
    if (!r->hist_is_packed || r->hist_expanded) return true;
    const size_t q = static_cast<size_t>(r->nq);
    if (!r->q_hist.alloc(q * ABB_N_ENTITY_TYPES * 4 + 4)) return false;
    uint32_t *dense = r->q_hist.as<uint32_t>();
    int col[ABB_N_ENTITY_TYPES]; int k = 0;
    for (int t = 0; t < ABB_N_ENTITY_TYPES; t++) if (r->hist_mask >> t & 1u) col[k++] = t;
    const void *packed = r->q_hist_packed.p;
    const int width = r->hist_width;
    auto work = [&](size_t a, size_t b) {
        memset(dense + a * ABB_N_ENTITY_TYPES, 0, (b - a) * ABB_N_ENTITY_TYPES * 4);
        if (width == 2) {
            const uint16_t *src = static_cast<const uint16_t *>(packed);
            for (size_t i = a; i < b; i++) for (int j = 0; j < k; j++) dense[i * ABB_N_ENTITY_TYPES + col[j]] = src[i * k + j];
        } else {
            const uint32_t *src = static_cast<const uint32_t *>(packed);
            for (size_t i = a; i < b; i++) for (int j = 0; j < k; j++) dense[i * ABB_N_ENTITY_TYPES + col[j]] = src[i * k + j];
        }
    };
    const size_t nthreads = std::max<size_t>(1, std::min<size_t>(16, q / (1 << 17)));
    if (nthreads <= 1) work(0, q);
    else {
        std::vector<std::thread> th;
        for (size_t t = 0; t < nthreads; t++) th.emplace_back(work, q * t / nthreads, q * (t + 1) / nthreads);
        for (auto &x : th) x.join();
    }
    r->hist_expanded = true;
    return true;
}
extern "C" const uint32_t *abb_walk_result_hist(const abb_walk_result *r) {
    if (!(r->flags & ABB_WALK_HIST)) return nullptr;
    return hist_expand(const_cast<abb_walk_result *>(r)) ? r->q_hist.as<uint32_t>() : nullptr;
}
extern "C" const void *abb_walk_result_hist_packed(const abb_walk_result *r, uint32_t *columns_mask, int32_t *bytes_per_count) {
    if (!r || !r->hist_is_packed) return nullptr;
    if (columns_mask) *columns_mask = r->hist_mask;
    if (bytes_per_count) *bytes_per_count = r->hist_width;
    return r->q_hist_packed.p ? r->q_hist_packed.p : static_cast<const void *>(r->q_start.p);   // k == 0: nothing to read, but not NULL
}
extern "C" const int32_t *abb_walk_result_nodes(const abb_walk_result *r) { return r->nodes.as<int32_t>(); }
extern "C" const int32_t *abb_walk_result_parent(const abb_walk_result *r) { return r->parent.as<int32_t>(); }
extern "C" const int32_t *abb_walk_result_depth(const abb_walk_result *r) { return r->depth.as<int32_t>(); }
extern "C" const uint32_t *abb_walk_result_edges(const abb_walk_result *r) { return r->edges.as<uint32_t>(); }
extern "C" int64_t abb_walk_result_h2d_bytes(const abb_walk_result *r) { return r->h2d; }
extern "C" int64_t abb_walk_result_d2h_bytes(const abb_walk_result *r) { return r->d2h; }

// ------------------------------------------------------------------ steps shared by the host walks
// fails when a walk of either set (canonical, individual) outgrew the last storage tier; the walk's stream must be idle
static int check_tier_fatal(abb_graph *g) {
    unsigned long long fatal = 0, fatal2 = 0;
    CUDA_TRY(cudaMemcpy(&fatal, g->tiers.ctl.as<unsigned long long>() + CTL_FATAL, sizeof fatal, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&fatal2, g->tiers.ctl.as<unsigned long long>() + CTL_SET + CTL_FATAL, sizeof fatal2, cudaMemcpyDeviceToHost));
    if (fatal || fatal2) return fail(ABB_ERR_CAPACITY, "a traversal outgrew the global scratch tier (more than n_nodes+4096 queue entries)");
    return ABB_OK;
}

// the non-zero histogram columns and the largest count of nq rows, into g->staging.hist_info once st has been synchronised
static int scan_hist_columns(abb_graph *g, const uint32_t *q_hist, int64_t nq, cudaStream_t st) {
    if (int rc = g->staging.hist_info_dev.ensure(2 * sizeof(unsigned long long))) return rc;
    CUDA_TRY(cudaMemsetAsync(g->staging.hist_info_dev.p, 0, 2 * sizeof(unsigned long long), st));
    if (int rc = LAUNCH(hist_columns_kernel, static_cast<unsigned>(g->sm_count) * 8, 256, 0, st, q_hist, nq * ABB_N_ENTITY_TYPES,
                        g->staging.hist_info_dev.as<unsigned long long>()))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(g->staging.hist_info, g->staging.hist_info_dev.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    return ABB_OK;
}

// r's packed-histogram layout from g->staging.hist_info: the non-zero columns, at 2 bytes per count when every count fits
static HistCols hist_layout(const abb_graph *g, abb_walk_result *r) {
    HistCols hc{};
    r->hist_is_packed = true;
    r->hist_mask = static_cast<uint32_t>(g->staging.hist_info[0]);
    for (int t = 0; t < ABB_N_ENTITY_TYPES; t++) if (r->hist_mask >> t & 1u) hc.col[hc.k++] = static_cast<uint8_t>(t);
    r->hist_k = hc.k;
    r->hist_width = g->staging.hist_info[1] < 65536ull ? 2 : 4;
    return hc;
}

// size hints for the next host walk: the largest node arena so far and the last batch; for a plain walk (one root per query, no
// parents / depths / edges / targets) also what the chunked path sizes its pieces from
static void note_walk_size(abb_graph *g, const abb_walk_spec *spec, int64_t nq, int64_t nodes, bool plain) {
    g->staging.hint_nodes = std::max(g->staging.hint_nodes, nodes);
    g->staging.hint_nq = nq; g->staging.hint_last_nodes = nodes;
    if (!plain) return;
    if (g->staging.plain_nq != nq || memcmp(&g->staging.plain_spec, spec, sizeof *spec) != 0) g->chunked.hint_nq = -1;
    g->staging.plain_spec = *spec; g->staging.plain_nq = nq; g->staging.plain_nodes = nodes;
}

// stage inputs, run (re-run once if the arenas were too small), leave results on the device
// `direct_nodes`: when the result size is known from the previous call, the walk kernels write the node arena
// straight into that pinned host block (UVA), so the PCIe transfer of the largest output overlaps the traversal
// instead of following it; if the estimate turns out too small the walk is re-run into a device arena.
// `roots_staged`: the caller has already copied the single roots into g->staging.roots on g->stream (sized for nq + 1).
static int walk_device_stage(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, const int64_t *root_off, const int32_t *targets,
                             int64_t nq, abb_walk_io *io_out, unsigned long long (&totals)[3], int64_t *h2d, HostBlock *direct_nodes = nullptr,
                             bool roots_staged = false) {
    cudaStream_t st = g->stream;
    WalkStaging &S = g->staging;
    const uint32_t fl = spec->flags;
    S.hist_info_valid = false;
    const int64_t n_roots = root_off ? root_off[nq] : nq;
    if (n_roots < 0) return fail(ABB_ERR_ARG, "bad root_off");
    const size_t q1 = static_cast<size_t>(nq) + 1;
    int rc = ABB_OK;
    ENS(S.roots, (n_roots + 1) * 4);
    if (root_off) ENS(S.root_off, q1 * 8);
    if (fl & ABB_WALK_TARGET) ENS(S.targets, q1 * 4);
    ENS(S.qstart, q1 * 8); ENS(S.qcount, q1 * 4); ENS(S.qmaxd, q1 * 4); ENS(S.qflags, q1 * 4);
    if (fl & ABB_WALK_EDGES) { ENS(S.qestart, q1 * 8); ENS(S.qecount, q1 * 8); }
    if (fl & ABB_WALK_HIST) ENS(S.qhist, q1 * ABB_N_ENTITY_TYPES * 4);
    ENS(S.totals, 3 * sizeof(unsigned long long));
    if (rc) return rc;
    *h2d = 0;
    if (n_roots && !roots_staged) { CUDA_TRY(cudaMemcpyAsync(S.roots.p, roots, static_cast<size_t>(n_roots) * 4, cudaMemcpyHostToDevice, st)); *h2d += n_roots * 4; }
    if (root_off) { CUDA_TRY(cudaMemcpyAsync(S.root_off.p, root_off, q1 * 8, cudaMemcpyHostToDevice, st)); *h2d += static_cast<int64_t>(q1) * 8; }
    if (fl & ABB_WALK_TARGET) { CUDA_TRY(cudaMemcpyAsync(S.targets.p, targets, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, st)); *h2d += nq * 4; }

    int64_t node_cap = std::max<int64_t>({S.hint_nodes, nq * 8, 1 << 16});
    int64_t edge_cap = (fl & ABB_WALK_EDGES) ? std::max<int64_t>({S.hint_edges, nq * 16, 1 << 16}) : 0;
    bool direct = direct_nodes && S.zero_copy && S.hint_nodes > 0 && !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES));
    if (direct) {
        // same batch size as last time: its exact need plus a little; otherwise scale the last per-query average generously, but
        // to no more than twice the largest arena any call has needed (a small batch of heavy sources, scaled to millions of
        // sources, would ask for more than the device holds; an estimate that is too small only costs a re-run into a device arena)
        node_cap = (nq == S.hint_nq) ? S.hint_last_nodes + S.hint_last_nodes / 64 + 4096 + (g->tiers.align_direct ? 32 * nq : 0)
                                      : std::min(static_cast<int64_t>(1.5 * static_cast<double>(S.hint_last_nodes) / std::max<int64_t>(S.hint_nq, 1) * nq) + 4096,
                                                 2 * node_cap);
        direct = direct_nodes->alloc(static_cast<size_t>(node_cap) * 4);
    }
    for (int attempt = 0; attempt < 3; attempt++) {
        if (!direct) ENS(S.nodes, node_cap * 4);
        if (fl & ABB_WALK_PARENTS) ENS(S.parent, node_cap * 4);
        if (fl & ABB_WALK_DEPTHS) ENS(S.depth, node_cap * 4);
        if (fl & ABB_WALK_EDGES) ENS(S.edges, edge_cap * 4);
        if (rc) return rc;
        abb_walk_io io{};
        io.n_queries = nq; io.roots = S.roots.as<int32_t>(); io.root_off = root_off ? S.root_off.as<int64_t>() : nullptr;
        io.targets = (fl & ABB_WALK_TARGET) ? S.targets.as<int32_t>() : nullptr;
        io.q_start = S.qstart.as<int64_t>(); io.q_count = S.qcount.as<int32_t>(); io.q_maxd = S.qmaxd.as<int32_t>(); io.q_flags = S.qflags.as<int32_t>();
        io.q_estart = S.qestart.as<int64_t>(); io.q_ecount = S.qecount.as<int64_t>(); io.q_hist = S.qhist.as<uint32_t>();
        io.nodes = direct ? direct_nodes->as<int32_t>() : S.nodes.as<int32_t>();
        io.parent = S.parent.as<int32_t>(); io.depth = S.depth.as<int32_t>(); io.node_cap = node_cap;
        io.edges = S.edges.as<uint32_t>(); io.edge_cap = edge_cap; io.totals = S.totals.as<unsigned long long>();
        CUDA_TRY(cudaEventRecord(S.ev_start, st));
        g->tiers.slice_align = (direct && g->tiers.align_direct) ? 32 : 0;
        CUDA_TRY(cudaMemsetAsync(S.totals.as<unsigned long long>() + 2, 0, sizeof(unsigned long long), st));
        int erc = enqueue_walk(g, spec, &io, st);
        g->tiers.slice_align = 0;
        if (erc) return erc;
        CUDA_TRY(cudaEventRecord(S.ev_end, st));
        S.timed = true;
        const bool scan_hist = (fl & ABB_WALK_HIST) && S.hist_pack && nq >= 1024;
        if (scan_hist) if ((rc = scan_hist_columns(g, io.q_hist, nq, st))) return rc;
        CUDA_TRY(cudaMemcpyAsync(totals, S.totals.p, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        S.hist_info_valid = scan_hist;
        if ((rc = check_tier_fatal(g))) return rc;
        *io_out = io;
        const bool fits = static_cast<int64_t>(totals[0]) <= node_cap && (!(fl & ABB_WALK_EDGES) || static_cast<int64_t>(totals[1]) <= edge_cap);
        const bool plain = !root_off && !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES | ABB_WALK_TARGET));
        note_walk_size(g, spec, nq, static_cast<int64_t>(totals[0]), fits && plain);
        S.hint_edges = std::max<int64_t>(S.hint_edges, static_cast<int64_t>(totals[1]));
        if (fits) return ABB_OK;
        if (direct) { direct_nodes->release(); direct = false; }     // estimate too small: fall back to a device arena
        node_cap = std::max<int64_t>(node_cap, static_cast<int64_t>(totals[0]));
        edge_cap = std::max<int64_t>(edge_cap, static_cast<int64_t>(totals[1]));
    }
    return fail(ABB_ERR_CAPACITY, "walk arenas still too small after resize");
}

// sync == false: the copies go to the graph's copy stream (ordered after everything enqueued so far on the main stream)
// so that kernels enqueued next on the main stream overlap them; the caller synchronises the copy stream.
// with_slices == false: only the per-query count / maxd / flags and histograms cross; q_start and the node arena stay on the device.
static int walk_collect(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io &io, const unsigned long long totals[3], int64_t h2d,
                        abb_walk_result **out, bool sync, HostBlock *direct_nodes = nullptr, bool with_slices = true) {
    cudaStream_t st = g->stream;
    if (!sync) {
        CUDA_TRY(cudaEventRecord(g->staging.ev_copy, g->stream));
        CUDA_TRY(cudaStreamWaitEvent(g->copy_stream, g->staging.ev_copy, 0));
        st = g->copy_stream;
    }
    const uint32_t fl = spec->flags;
    const int64_t nq = io.n_queries;
    std::unique_ptr<abb_walk_result> r(new abb_walk_result());
    r->nq = nq; r->flags = fl; r->total_nodes = with_slices ? static_cast<int64_t>(totals[0]) : 0; r->total_edges = (fl & ABB_WALK_EDGES) ? static_cast<int64_t>(totals[1]) : 0;
    r->h2d = h2d;
    const size_t q = static_cast<size_t>(nq), tn = static_cast<size_t>(r->total_nodes), te = static_cast<size_t>(r->total_edges);
    const bool have_nodes = direct_nodes && direct_nodes->p != nullptr;     // already written by the kernels over PCIe
    if (have_nodes) r->nodes = std::move(*direct_nodes);
    bool ok = (!with_slices || r->q_start.alloc(q * 8)) && r->q_count.alloc(q * 4) && r->q_maxd.alloc(q * 4) && r->q_flags.alloc(q * 4) &&
              (have_nodes || !with_slices || r->nodes.alloc(tn * 4));
    if (fl & ABB_WALK_EDGES) ok = ok && r->q_estart.alloc(q * 8) && r->q_ecount.alloc(q * 8) && r->edges.alloc(te * 4);
    const bool pack = (fl & ABB_WALK_HIST) && g->staging.hist_info_valid;
    g->staging.hist_info_valid = false;
    const HistCols hc = pack ? hist_layout(g, r.get()) : HistCols{};
    if (pack) ok = ok && (hc.k == 0 || r->q_hist_packed.alloc(q * hc.k * r->hist_width));
    else if (fl & ABB_WALK_HIST) ok = ok && r->q_hist.alloc(q * ABB_N_ENTITY_TYPES * 4);
    if (fl & ABB_WALK_PARENTS) ok = ok && r->parent.alloc(tn * 4);
    if (fl & ABB_WALK_DEPTHS) ok = ok && r->depth.alloc(tn * 4);
    if (!ok) return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    Readback d2h{st, &r->d2h};
    if (with_slices) d2h(r->q_start, io.q_start, q * 8);
    d2h(r->q_count, io.q_count, q * 4); d2h(r->q_maxd, io.q_maxd, q * 4); d2h(r->q_flags, io.q_flags, q * 4);
    if (have_nodes) r->d2h += static_cast<int64_t>((totals[2] ? totals[2] : static_cast<unsigned long long>(tn)) * 4); else if (with_slices) d2h(r->nodes, io.nodes, tn * 4);
    if (fl & ABB_WALK_EDGES) { d2h(r->q_estart, io.q_estart, q * 8); d2h(r->q_ecount, io.q_ecount, q * 8); d2h(r->edges, io.edges, te * 4); }
    if (pack) {
        if (hc.k) {
            const size_t pbytes = q * hc.k * r->hist_width;
            if (int rc = g->staging.hist_packed.ensure(pbytes)) return rc;
            const unsigned grid = static_cast<unsigned>(g->sm_count) * 8;
            const int rc = r->hist_width == 2 ? LAUNCH(hist_pack_kernel<uint16_t>, grid, 256, 0, st, io.q_hist, nq, hc, g->staging.hist_packed.as<uint16_t>())
                                              : LAUNCH(hist_pack_kernel<uint32_t>, grid, 256, 0, st, io.q_hist, nq, hc, g->staging.hist_packed.as<uint32_t>());
            if (rc) return rc;
            d2h.keep(cudaGetLastError());
            d2h(r->q_hist_packed, g->staging.hist_packed.p, pbytes);
        }
    } else if (fl & ABB_WALK_HIST) d2h(r->q_hist, io.q_hist, q * ABB_N_ENTITY_TYPES * 4);
    if (fl & ABB_WALK_PARENTS) d2h(r->parent, io.parent, tn * 4);
    if (fl & ABB_WALK_DEPTHS) d2h(r->depth, io.depth, tn * 4);
    if (sync && d2h.err == cudaSuccess) d2h.err = cudaStreamSynchronize(st);
    if (d2h.err != cudaSuccess) return fail(ABB_ERR_CUDA, "D2H failed: %s", cudaGetErrorString(d2h.err));
    *out = r.release();
    return ABB_OK;
}

// ------------------------------------------------------------------ chunked host walk
// A large plain batch (one root per query, no parents / depths / edges) whose result size is known from the previous call is walked
// in `chunks` pieces.  Piece k's node arena is copied to the host by the DMA engine (copy stream) while piece k+1 is walked, so the
// PCIe transfer runs at DMA speed behind the traversal instead of at the speed of SM stores (zero-copy) or after it.  Sources are
// assigned to pieces by frontier signature (signature mod chunks: a frontier group is never split, so nothing is walked or stored
// twice); each piece is a complete walk of its own.  Per-query arrays stay on the device for the whole batch, are put back into
// caller order by one scatter pass and cross once at the end.
constexpr int ABB_RETRY_UNCHUNKED = 1 << 20;   // internal: the caller falls back to the one-piece path

__global__ void add_base_kernel(int64_t *q_start, int64_t n, int64_t base) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) q_start[i] += base;
}

static bool chunked_applies(const abb_graph *g, const abb_walk_spec *spec, const int64_t *root_off, const int32_t *targets, int64_t nq) {
    const uint32_t fl = spec->flags;
    return g->chunked.chunks > 1 && nq >= g->chunked.chunk_min && nq >= 2 * g->chunked.chunks && !root_off && !targets &&
           !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES | ABB_WALK_TARGET)) && g->staging.plain_nq == nq && g->staging.plain_nodes > 0 &&
           memcmp(&g->staging.plain_spec, spec, sizeof *spec) == 0;
}

static int walk_host_chunked(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, int64_t nq, abb_walk_result **out) {
    NvtxRange nvtx_("walk_host_chunked");
    cudaStream_t st = g->stream, cst = g->copy_stream;
    WalkStaging &S = g->staging;
    ChunkedWalk &C = g->chunked;
    const uint32_t fl = spec->flags;
    const int K = C.chunks;
    const size_t q = static_cast<size_t>(nq), q1 = q + 1;
    const bool hist = (fl & ABB_WALK_HIST) != 0;
    int rc = ABB_OK;
    ENS(S.roots, q1 * 4); ENS(S.qstart, q1 * 8); ENS(S.qcount, q1 * 4); ENS(S.qmaxd, q1 * 4); ENS(S.qflags, q1 * 4);
    if (hist) ENS(S.qhist, q1 * ABB_N_ENTITY_TYPES * 4);
    ENS(S.totals, 3 * sizeof(unsigned long long));
    ENS(C.roots, q1 * 4); ENS(C.sig, q1 * 8); ENS(C.key, q1 * 4); ENS(C.key2, q1 * 4); ENS(C.idx, q1 * 4); ENS(C.order, q1 * 4); ENS(C.counts, 64 * 8);
    ENS(C.qstart, q1 * 8); ENS(C.qcount, q1 * 4); ENS(C.qmaxd, q1 * 4); ENS(C.qflags, q1 * 4);
    if (rc) return rc;
    const bool have_hint = C.hint_nq == nq && static_cast<int>(C.hint.size()) == K;
    // host arena: last total plus slack (the one-piece zero-copy pass pads slices, so its total is an upper bound already)
    const int64_t host_cap = S.plain_nodes + S.plain_nodes / (have_hint ? 64 : 8) + 4096ll * K;
    std::unique_ptr<abb_walk_result> r(new abb_walk_result());
    r->nq = nq; r->flags = fl;
    if (!(r->q_start.alloc(q * 8) && r->q_count.alloc(q * 4) && r->q_maxd.alloc(q * 4) && r->q_flags.alloc(q * 4) && r->nodes.alloc(static_cast<size_t>(host_cap) * 4)))
        return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    auto drain = [&]() { cudaStreamSynchronize(st); cudaStreamSynchronize(cst); };
    const unsigned qblocks = static_cast<unsigned>((nq + 255) / 256);
    CUDA_TRY(cudaMemcpyAsync(S.roots.p, roots, q * 4, cudaMemcpyHostToDevice, st));
    r->h2d = nq * 4;
    CUDA_TRY(cudaEventRecord(S.ev_start, st));
    // partition: chunk = frontier signature mod K when the walk de-duplicates (a frontier group is never split), contiguous ranges otherwise
    abb_walk_io probe{}; probe.n_queries = nq;
    const bool by_sig = dedup_applies(g, spec, &probe);
    unsigned long long *sig = nullptr;
    if (by_sig) {
        sig = C.sig.as<unsigned long long>();
        if ((rc = LAUNCH(dedup_sig_kernel, qblocks, 256, 0, st, g->v, *spec, S.roots.as<int32_t>(), nq, sig, nullptr))) { drain(); return rc; }
    }
    CUDA_TRY(cudaMemsetAsync(C.counts.p, 0, 64 * 8, st));
    if ((rc = LAUNCH(chunk_key_kernel, qblocks, 256, 0, st, sig, nq, K, C.key.as<uint32_t>(), C.idx.as<int32_t>(), C.counts.as<unsigned long long>()))) {
        drain(); return rc;
    }
    if ((rc = cub_run(C.tmp, [&](void *t, size_t &b) {
             return cub::DeviceRadixSort::SortPairs(t, b, C.key.as<uint32_t>(), C.key2.as<uint32_t>(), C.idx.as<int32_t>(), C.order.as<int32_t>(),
                                                    static_cast<int>(nq), 0, 6, st);
         }))) { drain(); return rc; }
    const int32_t *order = C.order.as<int32_t>();      // order[i] = caller index of the i-th query in chunk order
    if ((rc = LAUNCH(gather_i32_kernel, qblocks, 256, 0, st, S.roots.as<int32_t>(), order, C.roots.as<int32_t>(), nq))) { drain(); return rc; }
    unsigned long long counts[64] = {0};
    CUDA_TRY(cudaMemcpyAsync(counts, C.counts.p, 64 * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<int64_t> produced(static_cast<size_t>(K), 0);
    int64_t node_base = 0, b0 = 0;
    bool copied[2] = {false, false};
    for (int k = 0; k < K; k++) {
        const int64_t nk = static_cast<int64_t>(counts[k]);
        const int set = k & 1;
        if (!nk) continue;
        DevBuf &arena = set ? C.nodes_alt : S.nodes;
        int64_t cap = have_hint ? C.hint[static_cast<size_t>(k)] + C.hint[static_cast<size_t>(k)] / 64 + 4096
                                : 2 * (S.plain_nodes / K) + 65536;
        cap = std::max<int64_t>(cap, nk * 8);
        unsigned long long totals[3] = {0, 0, 0};
        bool done = false;
        for (int attempt = 0; attempt < 3 && !done; attempt++) {
            if (static_cast<size_t>(cap) * 4 > arena.cap && copied[set]) CUDA_TRY(cudaEventSynchronize(C.ev_copied[set]));   // about to reallocate it
            if ((rc = arena.ensure(static_cast<size_t>(cap) * 4))) { drain(); return rc; }
            if (copied[set]) CUDA_TRY(cudaStreamWaitEvent(st, C.ev_copied[set], 0));       // the arena's previous contents have left
            abb_walk_io io{};
            io.n_queries = nk; io.roots = C.roots.as<int32_t>() + b0;
            io.q_start = S.qstart.as<int64_t>() + b0; io.q_count = S.qcount.as<int32_t>() + b0; io.q_maxd = S.qmaxd.as<int32_t>() + b0;
            io.q_flags = S.qflags.as<int32_t>() + b0;
            io.q_hist = hist ? S.qhist.as<uint32_t>() + b0 * ABB_N_ENTITY_TYPES : nullptr;
            io.nodes = arena.as<int32_t>(); io.node_cap = cap; io.totals = S.totals.as<unsigned long long>();
            CUDA_TRY(cudaMemsetAsync(S.totals.as<unsigned long long>() + 2, 0, sizeof(unsigned long long), st));
            if (int erc = enqueue_walk(g, spec, &io, st)) { drain(); return erc; }
            CUDA_TRY(cudaMemcpyAsync(totals, S.totals.p, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            if ((rc = check_tier_fatal(g))) { drain(); return rc; }
            if (static_cast<int64_t>(totals[0]) <= cap) done = true; else cap = static_cast<int64_t>(totals[0]) + 4096;
        }
        if (!done) { drain(); return fail(ABB_ERR_CAPACITY, "walk arenas still too small after resize"); }
        const int64_t tot = static_cast<int64_t>(totals[0]);
        produced[static_cast<size_t>(k)] = tot;
        if (node_base + tot > host_cap) {          // the host arena guess was too small: let the one-piece path redo the batch
            drain();
            C.hint_nq = -1;
            return ABB_RETRY_UNCHUNKED;
        }
        if (node_base)
            if ((rc = LAUNCH(add_base_kernel, static_cast<unsigned>((nk + 255) / 256), 256, 0, st, S.qstart.as<int64_t>() + b0, nk, node_base))) { drain(); return rc; }
        CUDA_TRY(cudaEventRecord(C.ev_walked, st));
        CUDA_TRY(cudaStreamWaitEvent(cst, C.ev_walked, 0));
        if (tot) CUDA_TRY(cudaMemcpyAsync(r->nodes.as<int32_t>() + node_base, arena.p, static_cast<size_t>(tot) * 4, cudaMemcpyDeviceToHost, cst));
        CUDA_TRY(cudaEventRecord(C.ev_copied[set], cst));
        copied[set] = true;
        node_base += tot;
        b0 += nk;
    }
    if (b0 != nq) { drain(); return fail(ABB_ERR_CUDA, "chunk partition lost queries (%lld of %lld)", static_cast<long long>(b0), static_cast<long long>(nq)); }
    CUDA_TRY(cudaEventRecord(S.ev_end, st));
    S.timed = true;
    r->total_nodes = node_base;
    r->d2h += node_base * 4;
    // per-query results back into caller order, then to the host (the node copies of the last chunks are still in flight on the copy stream)
    const unsigned sgrid = static_cast<unsigned>(g->sm_count) * 8;
    if ((rc = LAUNCH(scatter_rows_kernel<int64_t>, sgrid, 256, 0, st, S.qstart.as<int64_t>(), order, C.qstart.as<int64_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, S.qcount.as<int32_t>(), order, C.qcount.as<int32_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, S.qmaxd.as<int32_t>(), order, C.qmaxd.as<int32_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, S.qflags.as<int32_t>(), order, C.qflags.as<int32_t>(), nq, 1))) {
        drain(); return rc;
    }
    const bool scan_hist = hist && S.hist_pack && nq >= 1024;
    if (scan_hist) {
        if ((rc = scan_hist_columns(g, S.qhist.as<uint32_t>(), nq, st))) { drain(); return rc; }
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    Readback d2h{st, &r->d2h, cudaGetLastError()};
    d2h(r->q_start, C.qstart.p, q * 8); d2h(r->q_count, C.qcount.p, q * 4); d2h(r->q_maxd, C.qmaxd.p, q * 4); d2h(r->q_flags, C.qflags.p, q * 4);
    if (scan_hist) {
        const HistCols hc = hist_layout(g, r.get());
        if (hc.k) {
            const size_t pbytes = q * hc.k * r->hist_width;
            if (!r->q_hist_packed.alloc(pbytes)) { drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed"); }
            if ((rc = S.hist_packed.ensure(pbytes))) { drain(); return rc; }
            rc = r->hist_width == 2
                     ? LAUNCH(hist_pack_scatter_kernel<uint16_t>, sgrid, 256, 0, st, S.qhist.as<uint32_t>(), order, nq, hc, S.hist_packed.as<uint16_t>())
                     : LAUNCH(hist_pack_scatter_kernel<uint32_t>, sgrid, 256, 0, st, S.qhist.as<uint32_t>(), order, nq, hc, S.hist_packed.as<uint32_t>());
            if (rc) { drain(); return rc; }
            d2h(r->q_hist_packed, S.hist_packed.p, pbytes);
        }
    } else if (hist) {
        if (!r->q_hist.alloc(q * ABB_N_ENTITY_TYPES * 4)) { drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed"); }
        if ((rc = C.qhist.ensure(q1 * ABB_N_ENTITY_TYPES * 4))) { drain(); return rc; }
        if ((rc = LAUNCH(scatter_rows_kernel<uint32_t>, sgrid, 256, 0, st, S.qhist.as<uint32_t>(), order, C.qhist.as<uint32_t>(), nq, ABB_N_ENTITY_TYPES))) {
            drain(); return rc;
        }
        d2h(r->q_hist, C.qhist.p, q * ABB_N_ENTITY_TYPES * 4);
    }
    cudaError_t &e = d2h.err;
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cst);
    if (e != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "chunked walk failed: %s", cudaGetErrorString(e)); }
    S.hist_info_valid = false;
    note_walk_size(g, spec, nq, node_base, true);
    C.hint = produced; C.hint_nq = nq;
    C.last_host_chunks = K;
    *out = r.release();
    return ABB_OK;
}

extern "C" int abb_walk_host(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, const int64_t *root_off, const int32_t *targets,
                             int64_t n_queries, abb_walk_result **out) {
    NvtxRange nvtx_("abb_walk_host");
    if (!g || !spec || !out || n_queries < 0 || (n_queries > 0 && !roots)) return fail(ABB_ERR_ARG, "bad arguments");
    if ((spec->flags & ABB_WALK_TARGET) && !targets) return fail(ABB_ERR_ARG, "TARGET needs targets");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    if (chunked_applies(g, spec, root_off, targets, n_queries)) {
        const int crc = walk_host_chunked(g, spec, roots, n_queries, out);
        if (crc != ABB_RETRY_UNCHUNKED) return crc;
    }
    g->chunked.last_host_chunks = 1;
    abb_walk_io io{}; unsigned long long totals[3] = {0, 0, 0}; int64_t h2d = 0;
    HostBlock direct;
    if (int rc = walk_device_stage(g, spec, roots, root_off, targets, n_queries, &io, totals, &h2d, &direct)) return rc;
    return walk_collect(g, spec, io, totals, h2d, out, true, &direct);
}

// ------------------------------------------------------------------ exposure-path rows
static unsigned warp_grid(const abb_graph *g, int64_t warps) {
    return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((warps + 7) / 8, static_cast<int64_t>(g->sm_count) * 8)));
}

// for_each_row gives each block an equal contiguous run of row tiles, so the grid is a whole number of waves of resident blocks
// (a partial last wave would add a block's whole run to the time).  Four waves rather than one, so that blocks still start
// promptly when another stream's kernels hold part of the GPU.
template <class K>
static unsigned row_grid(const abb_graph *g, K kernel, int &cached) {
    if (!cached) {
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, ROW_THREADS, 0);
        cached = 4 * g->sm_count * std::max(1, per_sm);
    }
    return static_cast<unsigned>(cached);
}

// the graph's parts of the exposure-path arguments: server tables and exposure tables
static PathsArgs paths_base(const GraphView &v, const ExposureTables &X) {
    PathsArgs A{};
    A.g = v; A.srv_cred = X.srv_cred.as<int32_t>(); A.srv_tool = X.srv_tool.as<int32_t>();
    A.srv_roff = X.srv_roff.as<int64_t>(); A.srv_row = X.srv_row.as<int4>(); A.srv_rel = X.srv_rel.as<int8_t>();
    A.x_vs = X.vs.as<uint8_t>(); A.x_loff = X.loff.as<int64_t>(); A.x_link = X.link.as<LinkRec>(); A.x_rows = X.rows.as<int32_t>();
    A.x_toff = X.toff.as<int64_t>(); A.t_row = X.trow.as<int4>(); A.t_rel = X.trel.as<int8_t>(); A.x_overflow = X.overflow.as<unsigned>();
    return A;
}

// Graph-constant exposure tables (paths.cuh), built once per graph and freed with it: the server tables (fan-out, and the principal
// rows every server contributes to a template), then the links of every finding node, the template of every vulnerable source and
// the rows of every finding node (count -> scan in place -> fill).  Built aside and installed only once complete: a failed build
// leaves nothing behind.  Synchronises the stream to size the row, link and template arrays, and once more at the end: later calls
// may come on other streams.
static int ensure_exposure_tables(abb_graph *g, cudaStream_t st) {
    if (g->exposure) return ABB_OK;
    NvtxRange nvtx_("paths: graph-constant exposure tables");
    std::unique_ptr<ExposureTables> X(new ExposureTables());
    DevBuf &scan_tmp = g->paths.scan_tmp;
    const int64_t n = g->v.n;
    const size_t n1 = static_cast<size_t>(n) + 1;
    if (int rc = X->srv_cred.ensure(n1 * 4)) return rc;
    if (int rc = X->srv_tool.ensure(n1 * 4)) return rc;
    const unsigned sgrid = grid_for(n, 256, g->sm_count, 16);
    if (int rc = LAUNCH(server_table_kernel, sgrid, 256, 0, st, g->v, X->srv_cred.as<int32_t>(), X->srv_tool.as<int32_t>())) return rc;
    // principal rows of every server (paths.cuh server_rows_kernel): count, scan in place, fill
    if (int rc = X->srv_roff.ensure(n1 * 8)) return rc;
    int64_t *roff = X->srv_roff.as<int64_t>();
    CUDA_TRY(cudaMemsetAsync(roff, 0, n1 * 8, st));
    if (int rc = LAUNCH(server_rows_kernel<false>, sgrid, 256, 0, st, g->v, X->srv_cred.as<int32_t>(), X->srv_tool.as<int32_t>(), roff, nullptr, nullptr))
        return rc;
    if (int rc = scan_i64(scan_tmp, roff, roff, static_cast<int64_t>(n1), st)) return rc;
    int64_t total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, roff + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (int rc = X->srv_row.ensure(static_cast<size_t>(total + 1) * 16)) return rc;
    if (int rc = X->srv_rel.ensure(static_cast<size_t>(total) + 16)) return rc;
    if (int rc = LAUNCH(server_rows_kernel<true>, sgrid, 256, 0, st, g->v, X->srv_cred.as<int32_t>(), X->srv_tool.as<int32_t>(), roff, X->srv_row.as<int4>(),
                        X->srv_rel.as<int8_t>()))
        return rc;
    int rc = X->vs.alloc(n1);
    if (!rc) rc = X->loff.alloc(n1 * 8);
    if (!rc) rc = X->toff.alloc(n1 * 8);
    if (!rc) rc = X->rows.alloc(n1 * 4);
    if (!rc) rc = X->overflow.alloc(4);
    if (rc) return rc;
    PathsArgs A = paths_base(g->v, *X);
    CUDA_TRY(cudaMemsetAsync(A.x_vs, 0, n1, st));
    CUDA_TRY(cudaMemsetAsync(A.x_loff, 0, n1 * 8, st));
    CUDA_TRY(cudaMemsetAsync(A.x_toff, 0, n1 * 8, st));
    CUDA_TRY(cudaMemsetAsync(A.x_overflow, 0, 4, st));
    const unsigned grid = warp_grid(g, (n + 31) / 32);
    if ((rc = LAUNCH(node_links_kernel<false>, grid, 256, 0, st, A))) return rc;
    if ((rc = scan_i64(scan_tmp, A.x_loff, A.x_loff, n + 1, st))) return rc;
    if ((rc = LAUNCH(template_kernel<false>, grid, 256, 0, st, A))) return rc;
    if ((rc = scan_i64(scan_tmp, A.x_toff, A.x_toff, n + 1, st))) return rc;
    int64_t NL = 0, TR = 0;
    CUDA_TRY(cudaMemcpyAsync(&NL, A.x_loff + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&TR, A.x_toff + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    // link records hold link and template offsets as int32
    if (NL >= (1ll << 31) - 1 || TR >= (1ll << 31) - 1) return fail(ABB_ERR_CAPACITY, "exposure tables: %lld links, %lld template rows (int32 offsets)", (long long)NL, (long long)TR);
    if (!rc) rc = X->link.alloc(static_cast<size_t>(NL) * 16);
    if (!rc) rc = X->trow.alloc(static_cast<size_t>(TR) * 16);
    if (!rc) rc = X->trel.alloc(static_cast<size_t>(TR) * 2);
    if (rc) return rc;
    A = paths_base(g->v, *X);
    if ((rc = LAUNCH(template_kernel<true>, grid, 256, 0, st, A)) || (rc = LAUNCH(node_links_kernel<true>, grid, 256, 0, st, A))) return rc;
    unsigned overflow = 0;
    CUDA_TRY(cudaMemcpyAsync(&overflow, A.x_overflow, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (overflow) return fail(ABB_ERR_CAPACITY, "exposure tables: a finding has 2^31 or more exposure-path rows");
    g->exposure = std::move(X);
    return ABB_OK;
}

// Count pass of the exposure-path pipeline (paths.cuh): each finding's row count and links gathered from the exposure tables, then
// one exclusive scan into io.f_off.  Once the tables exist this neither synchronises nor, for a batch no larger than an earlier
// one, allocates.  `link_counts` also writes each finding's link count (f_lcnt) for the host result.
static int enqueue_paths_count(abb_graph *g, const abb_paths_io *io, cudaStream_t st, bool link_counts = false) {
    NvtxRange nvtx_("paths: rows per finding");
    if (!io || io->n_findings < 0 || !io->f_off || (io->n_findings && !io->findings)) return fail(ABB_ERR_ARG, "bad paths io");
    if (io->n_findings >= (1ll << 31) - 2) return fail(ABB_ERR_ARG, "too many findings in one batch");
    if (int rc = ensure_exposure_tables(g, st)) return rc;
    g->paths.args_valid = false;
    const int64_t nf = io->n_findings;
    int rc = g->paths.f_cnt.ensure(static_cast<size_t>(nf + 1) * 8);
    if (!rc) rc = g->paths.f_link.ensure(static_cast<size_t>(nf + 1) * 8);
    if (!rc && link_counts) rc = g->paths.f_lcnt.ensure(static_cast<size_t>(nf + 1) * 8);
    if (rc) return rc;
    PathsArgs A = paths_base(g->v, *g->exposure);
    A.io = *io; A.f_cnt = g->paths.f_cnt.as<int64_t>(); A.f_link = g->paths.f_link.as<int2>(); A.f_lcnt = link_counts ? g->paths.f_lcnt.as<int64_t>() : nullptr;
    if ((rc = LAUNCH(finding_rows_kernel, static_cast<unsigned>((nf + 1 + 255) / 256), 256, 0, st, A))) return rc;
    if ((rc = scan_i64(g->paths.scan_tmp, A.f_cnt, io->f_off, nf + 1, st))) return rc;
    g->paths.args = A;
    g->paths.args_valid = true;
    return ABB_OK;
}

static int enqueue_paths_fill(abb_graph *g, const abb_paths_io *io, cudaStream_t st) {
    if (!io || !io->f_off || !io->hops || !io->rels || !io->ncred || !io->ntool) return fail(ABB_ERR_ARG, "bad paths io");
    if (!io->n_findings) return ABB_OK;
    if (!g->paths.args_valid || g->paths.args.io.findings != io->findings || g->paths.args.io.n_findings != io->n_findings || g->paths.args.io.f_off != io->f_off)
        return fail(ABB_ERR_ARG, "abb_paths_fill_launch must follow abb_paths_count_launch for the same findings / f_off");
    if ((reinterpret_cast<uintptr_t>(io->hops) & 15) != 0 || (reinterpret_cast<uintptr_t>(io->rels) & 3) != 0) return fail(ABB_ERR_ARG, "io.hops must be 16-byte and io.rels 4-byte aligned");
    PathsArgs A = g->paths.args;
    A.io = *io;
    return LAUNCH(replicate_kernel, row_grid(g, replicate_kernel, g->paths.replicate_grid), ROW_THREADS, 0, st, A);
}

extern "C" int abb_paths_count_launch(abb_graph *g, const abb_paths_io *io, void *stream) {
    NvtxRange nvtx_("abb_paths_count_launch");
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaEventRecord(g->paths.ev_start, st));
    return enqueue_paths_count(g, io, st);
}
extern "C" int abb_paths_fill_launch(abb_graph *g, const abb_paths_io *io, void *stream) {
    NvtxRange nvtx_("abb_paths_fill_launch");
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = enqueue_paths_fill(g, io, st);
    if (rc) return rc;
    CUDA_TRY(cudaEventRecord(g->paths.ev_end, st));
    g->paths.timed = true;
    return ABB_OK;
}

// Host result of the exposure-path pipeline.  What crosses PCIe is the FACTORISED form — per finding its links
// (vulnerable source + relationship), per link the template slice of that source — which determines every row;
// the flat row arrays of the ABI are expanded from it on the host, on first access.
struct abb_paths_result {
    int64_t nf = 0, rows = 0, n_links = 0, n_trows = 0, h2d = 0, d2h = 0;
    HostBlock off, link_off, link_vs, link_rel, link_roff, link_toff, t_row, t_rel, findings;
    std::mutex mu;
    bool expanded = false;
    HostBlock hops, rels, ncred, ntool;
};
extern "C" void abb_paths_result_free(abb_paths_result *r) { delete r; }

// links x templates -> flat rows (same layout the device's replicate kernel writes), threads over link ranges
static bool paths_expand(abb_paths_result *r) {
    std::lock_guard<std::mutex> lk(r->mu);
    if (r->expanded) return true;
    const size_t rows = static_cast<size_t>(r->rows);
    if (!(r->hops.alloc(rows * 16) && r->rels.alloc(rows * 4) && r->ncred.alloc(rows * 4) && r->ntool.alloc(rows * 4))) return false;
    const int64_t *loff = r->link_off.as<int64_t>(), *lroff = r->link_roff.as<int64_t>(), *ltoff = r->link_toff.as<int64_t>();
    const int32_t *lvs = r->link_vs.as<int32_t>(), *fnd = r->findings.as<int32_t>(), *trow = r->t_row.as<int32_t>();
    const int8_t *lrel = r->link_rel.as<int8_t>(), *trel = r->t_rel.as<int8_t>();
    int32_t *hops = r->hops.as<int32_t>(), *ncred = r->ncred.as<int32_t>(), *ntool = r->ntool.as<int32_t>();
    int8_t *rels = r->rels.as<int8_t>();
    auto work = [&](int64_t f0, int64_t f1) {
        for (int64_t fi = f0; fi < f1; fi++) {
            const int32_t f = fnd[fi];
            for (int64_t l = loff[fi]; l < loff[fi + 1]; l++) {
                const int32_t vs = lvs[l]; const int8_t rvf = lrel[l];
                const int64_t o0 = lroff[l], n = lroff[l + 1] - o0, t0 = ltoff[l];
                for (int64_t k = 0; k < n; k++) {
                    const int32_t *tr = trow + (t0 + k) * 4;
                    const int32_t srv = tr[1];
                    int32_t *h = hops + (o0 + k) * 4;
                    h[0] = tr[0]; h[1] = srv; h[2] = (vs != srv) ? vs : -1; h[3] = f;
                    int8_t *rr = rels + (o0 + k) * 4;
                    const int8_t ras = trel[(t0 + k) * 2], rsv = trel[(t0 + k) * 2 + 1];
                    if (vs != srv) { rr[0] = ras; rr[1] = rsv; rr[2] = rvf; rr[3] = -2; } else { rr[0] = ras; rr[1] = rvf; rr[2] = -2; rr[3] = -2; }
                    ncred[o0 + k] = tr[2]; ntool[o0 + k] = tr[3];
                }
            }
        }
    };
    const int nthreads = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(16, r->rows / (1 << 20))));
    if (nthreads <= 1) work(0, r->nf);
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < nthreads; t++) th.emplace_back(work, r->nf * t / nthreads, r->nf * (t + 1) / nthreads);
        for (auto &x : th) x.join();
    }
    r->expanded = true;
    return true;
}
extern "C" int64_t abb_paths_result_rows(const abb_paths_result *r) { return r->rows; }
extern "C" const int64_t *abb_paths_result_off(const abb_paths_result *r) { return r->off.as<int64_t>(); }
extern "C" const int32_t *abb_paths_result_hops(const abb_paths_result *r) { return paths_expand(const_cast<abb_paths_result *>(r)) ? r->hops.as<int32_t>() : nullptr; }
extern "C" const int8_t *abb_paths_result_rels(const abb_paths_result *r) { return paths_expand(const_cast<abb_paths_result *>(r)) ? r->rels.as<int8_t>() : nullptr; }
extern "C" const int32_t *abb_paths_result_ncred(const abb_paths_result *r) { return paths_expand(const_cast<abb_paths_result *>(r)) ? r->ncred.as<int32_t>() : nullptr; }
extern "C" const int32_t *abb_paths_result_ntool(const abb_paths_result *r) { return paths_expand(const_cast<abb_paths_result *>(r)) ? r->ntool.as<int32_t>() : nullptr; }
extern "C" int64_t abb_paths_result_links(const abb_paths_result *r) { return r->n_links; }
extern "C" int64_t abb_paths_result_template_rows(const abb_paths_result *r) { return r->n_trows; }
extern "C" const int64_t *abb_paths_result_link_off(const abb_paths_result *r) { return r->link_off.as<int64_t>(); }
extern "C" const int32_t *abb_paths_result_link_source(const abb_paths_result *r) { return r->link_vs.as<int32_t>(); }
extern "C" const int8_t *abb_paths_result_link_rel(const abb_paths_result *r) { return r->link_rel.as<int8_t>(); }
extern "C" const int64_t *abb_paths_result_link_row_off(const abb_paths_result *r) { return r->link_roff.as<int64_t>(); }
extern "C" const int64_t *abb_paths_result_link_template(const abb_paths_result *r) { return r->link_toff.as<int64_t>(); }
extern "C" const int32_t *abb_paths_result_template(const abb_paths_result *r) { return r->t_row.as<int32_t>(); }
extern "C" const int8_t *abb_paths_result_template_rel(const abb_paths_result *r) { return r->t_rel.as<int8_t>(); }
extern "C" int64_t abb_paths_result_h2d_bytes(const abb_paths_result *r) { return r->h2d; }
extern "C" int64_t abb_paths_result_d2h_bytes(const abb_paths_result *r) { return r->d2h; }

// findings already on the device (d_findings) or staged from the host
static int paths_run(abb_graph *g, const int32_t *h_findings, const int32_t *d_findings, int64_t nf, abb_paths_result **out, cudaStream_t st = nullptr) {
    if (!st) st = g->stream;
    PathsWorkspace &P = g->paths;
    std::unique_ptr<abb_paths_result> r(new abb_paths_result());
    r->nf = nf;
    if (!r->findings.alloc(static_cast<size_t>(nf + 1) * 4)) return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    if (nf) memcpy(r->findings.p, h_findings, static_cast<size_t>(nf) * 4);
    if (!d_findings) {
        if (int rc = P.findings.ensure(static_cast<size_t>(nf + 1) * 4)) return rc;
        if (nf) { CUDA_TRY(cudaMemcpyAsync(P.findings.p, h_findings, static_cast<size_t>(nf) * 4, cudaMemcpyHostToDevice, st)); r->h2d += nf * 4; }
        d_findings = P.findings.as<int32_t>();
    }
    if (int rc = P.f_off.ensure(static_cast<size_t>(nf + 1) * 8)) return rc;
    abb_paths_io io{};
    io.n_findings = nf; io.findings = d_findings; io.f_off = P.f_off.as<int64_t>();
    CUDA_TRY(cudaEventRecord(P.ev_start, st));
    if (int rc = enqueue_paths_count(g, &io, st, true)) return rc;
    // the batch's share of the exposure tables: its links (link counts scanned into link_off) and the templates of its distinct
    // vulnerable sources, in node order
    const PathsArgs A = P.args;
    const int64_t n = g->v.n;
    int rc = P.link_off.ensure(static_cast<size_t>(nf + 1) * 8);
    if (rc) return rc;
    int64_t *link_off = P.link_off.as<int64_t>();
    if ((rc = scan_i64(P.scan_tmp, A.f_lcnt, link_off, nf + 1, st))) return rc;
    int64_t NL = 0;
    CUDA_TRY(cudaMemcpyAsync(&NL, link_off + nf, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const int64_t nu_max = std::min<int64_t>(NL, n);
    ENS(P.link_vs, (NL + 2) * 4); ENS(P.link_rel, NL + 16); ENS(P.link_roff, (NL + 2) * 8); ENS(P.link_toff, (NL + 2) * 8); ENS(P.need, n + 16); ENS(P.ulist, (n + 2) * 4);
    ENS(P.nu, 16); ENS(P.t_cnt, (nu_max + 2) * 8); ENS(P.t_off, (nu_max + 2) * 8); ENS(P.t_off_node, (n + 2) * 8);
    if (rc) return rc;
    int32_t *link_vs = P.link_vs.as<int32_t>(), *ulist = P.ulist.as<int32_t>();
    int8_t *link_rel = P.link_rel.as<int8_t>();
    int64_t *link_roff = P.link_roff.as<int64_t>(), *link_toff = P.link_toff.as<int64_t>(), *t_cnt = P.t_cnt.as<int64_t>(), *t_off = P.t_off.as<int64_t>();
    uint8_t *need = P.need.as<uint8_t>();
    unsigned long long *nu = P.nu.as<unsigned long long>();
    CUDA_TRY(cudaMemsetAsync(need, 0, static_cast<size_t>(n) + 16, st));
    if ((rc = LAUNCH(batch_links_kernel, static_cast<unsigned>((nf + 1 + 255) / 256), 256, 0, st, A, link_off, link_vs, link_rel, link_roff, need))) return rc;
    if ((rc = select_flagged(P.scan_tmp, need, ulist, nu, static_cast<int>(n), st))) return rc;
    CUDA_TRY(cudaMemsetAsync(t_cnt, 0, static_cast<size_t>(nu_max + 2) * 8, st));
    if (nu_max) if ((rc = LAUNCH(batch_template_counts_kernel, static_cast<unsigned>((nu_max + 255) / 256), 256, 0, st, A, ulist, nu, t_cnt))) return rc;
    if ((rc = scan_i64(P.scan_tmp, t_cnt, t_off, nu_max + 1, st))) return rc;
    int64_t TR = 0;
    CUDA_TRY(cudaMemcpyAsync(&TR, t_off + nu_max, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ENS(P.t_row, (TR + 2) * 16); ENS(P.t_rel, (TR + 2) * 2);
    if (rc) return rc;
    int64_t *t_off_node = P.t_off_node.as<int64_t>();
    if (nu_max)
        if ((rc = LAUNCH(batch_templates_kernel, warp_grid(g, nu_max), 256, 0, st, A, ulist, nu, t_off, t_off_node, P.t_row.as<int4>(), P.t_rel.as<int8_t>())))
            return rc;
    if (NL) if ((rc = LAUNCH(batch_link_toff_kernel, static_cast<unsigned>((NL + 255) / 256), 256, 0, st, NL, link_vs, t_off_node, link_toff))) return rc;
    CUDA_TRY(cudaEventRecord(P.ev_end, st));
    P.timed = true;
    const size_t n1 = static_cast<size_t>(nf) + 1;
    r->n_links = NL; r->n_trows = TR;
    bool ok = r->off.alloc(n1 * 8) && r->link_off.alloc(n1 * 8) && r->link_vs.alloc(NL * 4) && r->link_rel.alloc(NL) && r->link_roff.alloc((NL + 1) * 8) &&
              r->link_toff.alloc(NL * 8) && r->t_row.alloc(TR * 16) && r->t_rel.alloc(TR * 2);
    if (!ok) return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    Readback d2h{st, &r->d2h};
    d2h(r->off, io.f_off, n1 * 8); d2h(r->link_off, link_off, n1 * 8); d2h(r->link_vs, link_vs, NL * 4); d2h(r->link_rel, link_rel, NL);
    d2h(r->link_roff, link_roff, (NL + 1) * 8); d2h(r->link_toff, link_toff, NL * 8); d2h(r->t_row, P.t_row.p, TR * 16); d2h(r->t_rel, P.t_rel.p, TR * 2);
    if (d2h.err == cudaSuccess) d2h.err = cudaStreamSynchronize(st);
    if (d2h.err != cudaSuccess) return fail(ABB_ERR_CUDA, "paths D2H failed: %s", cudaGetErrorString(d2h.err));
    r->rows = r->off.as<int64_t>()[nf];
    *out = r.release();
    return ABB_OK;
}

extern "C" int abb_paths_host(abb_graph *g, const int32_t *findings, int64_t n_findings, abb_paths_result **out) {
    NvtxRange nvtx_("abb_paths_host");
    if (!g || !out || n_findings < 0 || (n_findings && !findings)) return fail(ABB_ERR_ARG, "bad arguments");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    return paths_run(g, findings, nullptr, n_findings, out);
}

// ------------------------------------------------------------------ ranked page of exposure-path rows
struct abb_rank_result {
    int64_t total = 0, matched = 0, count = 0;
    std::vector<int32_t> hops, ncred, ntool;
    std::vector<int8_t> rels;
    std::vector<uint32_t> risk_rank;
    std::vector<int64_t> row;
};
extern "C" void abb_rank_result_free(abb_rank_result *r) { delete r; }
extern "C" int64_t abb_rank_result_total(const abb_rank_result *r) { return r->total; }
extern "C" int64_t abb_rank_result_count(const abb_rank_result *r) { return r->count; }
extern "C" int64_t abb_rank_result_matched(const abb_rank_result *r) { return r->matched; }
extern "C" const int32_t *abb_rank_result_hops(const abb_rank_result *r) { return r->hops.data(); }
extern "C" const int8_t *abb_rank_result_rels(const abb_rank_result *r) { return r->rels.data(); }
extern "C" const int32_t *abb_rank_result_ncred(const abb_rank_result *r) { return r->ncred.data(); }
extern "C" const int32_t *abb_rank_result_ntool(const abb_rank_result *r) { return r->ntool.data(); }
extern "C" const uint32_t *abb_rank_result_risk_rank(const abb_rank_result *r) { return r->risk_rank.data(); }
extern "C" const int64_t *abb_rank_result_row(const abb_rank_result *r) { return r->row.data(); }

// One ranking path: node_focus == nullptr ranks every row (abb_paths_rank_host); otherwise the rows that miss the focus are
// compacted away (cub::DeviceSelect keeps their order) and only the matched rows are sorted.
static int paths_rank(abb_graph *g, const int32_t *findings, int64_t n_findings, const int32_t *base_id, const uint32_t *risk_rank, int64_t n_base,
                      const int32_t *ncu, const int32_t *ntu, const uint8_t *node_focus, uint32_t need, int64_t offset, int64_t limit,
                      abb_rank_result **out) {
    if (!g || !out || n_findings < 0 || offset < 0 || limit < 0 || n_base <= 0 || !risk_rank || !ncu || !ntu || (n_findings && (!findings || !base_id)))
        return fail(ABB_ERR_ARG, "bad arguments");
    if (node_focus && (need & ~(ABB_FOCUS_CVE | ABB_FOCUS_PACKAGE | ABB_FOCUS_AGENT))) return fail(ABB_ERR_ARG, "need: unknown focus category 0x%x", need);
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = g->stream;
    const int64_t nf = n_findings, n = g->v.n;
    const bool focused = node_focus != nullptr;
    if (int rc = g->paths.findings.ensure(static_cast<size_t>(nf + 1) * 4)) return rc;
    if (int rc = g->paths.f_off.ensure(static_cast<size_t>(nf + 1) * 8)) return rc;
    DevBuf d_base, d_tab, d_ncu, d_ntu, d_focus;
    if (nf) CUDA_TRY(cudaMemcpyAsync(g->paths.findings.p, findings, static_cast<size_t>(nf) * 4, cudaMemcpyHostToDevice, st));
    if (int rc = d_base.upload(base_id, static_cast<size_t>(nf) * 4, st, 4)) return rc;
    if (int rc = d_tab.upload(risk_rank, static_cast<size_t>(n_base) * 75 * 4, st)) return rc;
    if (int rc = d_ncu.upload(ncu, static_cast<size_t>(n) * 4, st, 4)) return rc;
    if (int rc = d_ntu.upload(ntu, static_cast<size_t>(n) * 4, st, 4)) return rc;
    if (focused) { if (int rc = d_focus.upload(node_focus, static_cast<size_t>(n), st, 1)) return rc; }
    abb_paths_io io{};
    io.n_findings = nf; io.findings = g->paths.findings.as<int32_t>(); io.f_off = g->paths.f_off.as<int64_t>();
    if (int rc = enqueue_paths_count(g, &io, st)) return rc;
    int64_t R = 0;
    CUDA_TRY(cudaMemcpyAsync(&R, io.f_off + nf, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (R >= (1ll << 32) - 1) return fail(ABB_ERR_CAPACITY, "more than 2^32 exposure-path rows in one ranking batch");
    std::unique_ptr<abb_rank_result> r(new abb_rank_result());
    r->total = R;
    r->matched = R;
    // unfocused, the page is known before any kernel runs; focused, the matched count is needed first
    if (R == 0 || (!focused && std::min(limit, R - std::min(offset, R)) == 0)) { r->matched = focused ? 0 : R; *out = r.release(); return ABB_OK; }
    DevBuf k1, k2, v1, v2, tmp, d_sel;
    int rc = k1.alloc(static_cast<size_t>(R) * 8);
    if (!rc) rc = k2.alloc(static_cast<size_t>(R) * 8);
    if (!rc) rc = v1.alloc(static_cast<size_t>(R) * 4);
    if (!rc) rc = v2.alloc(static_cast<size_t>(R) * 4);
    if (rc) return rc;
    PathsArgs A = g->paths.args;
    RankArgs RA{d_base.as<int32_t>(), d_tab.as<uint32_t>(), d_ncu.as<int32_t>(), d_ntu.as<int32_t>(), k1.as<unsigned long long>(), v1.as<uint32_t>(),
                d_focus.as<uint8_t>(), need};
    if ((rc = LAUNCH(rank_keys_kernel, row_grid(g, rank_keys_kernel, g->paths.rank_keys_grid), ROW_THREADS, 0, st, A, RA))) return rc;
    // sort input: every row (k1, v1), or the matched rows compacted into (k2, v2); the sorted pairs land in the other pair
    unsigned long long *key_in = k1.as<unsigned long long>(), *key_out = k2.as<unsigned long long>();
    uint32_t *row_in = v1.as<uint32_t>(), *row_out = v2.as<uint32_t>();
    if (focused) {
        if ((rc = d_sel.alloc(8))) return rc;
        if ((rc = cub_run(tmp, [&](void *t, size_t &b) {
                 return cub::DeviceSelect::If(t, b, v1.as<uint32_t>(), v2.as<uint32_t>(), d_sel.as<int64_t>(), static_cast<int>(R), RowMatched{}, st);
             }))) return rc;
        int64_t M = 0;
        CUDA_TRY(cudaMemcpyAsync(&M, d_sel.p, 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        r->matched = M;
        if (M == 0 || std::min(limit, M - std::min(offset, M)) == 0) { *out = r.release(); return ABB_OK; }
        if ((rc = LAUNCH(gather_keys_kernel, static_cast<unsigned>((M + 255) / 256), 256, 0, st, k1.as<unsigned long long>(), v2.as<uint32_t>(), M,
                         k2.as<unsigned long long>())))
            return rc;
        std::swap(key_in, key_out); std::swap(row_in, row_out);
    }
    const int64_t M = r->matched;
    const int64_t first = std::min(offset, M), count = std::min(limit, M - first);
    r->count = count;
    if ((rc = cub_run(tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, key_in, key_out, row_in, row_out, static_cast<int>(M), 0, 64, st); })))
        return rc;
    DevBuf o_hops, o_rels, o_nc, o_nt, o_rank, o_row;
    rc = o_hops.alloc(static_cast<size_t>(count) * 16);
    if (!rc) rc = o_rels.alloc(static_cast<size_t>(count) * 4);
    if (!rc) rc = o_nc.alloc(static_cast<size_t>(count) * 4);
    if (!rc) rc = o_nt.alloc(static_cast<size_t>(count) * 4);
    if (!rc) rc = o_rank.alloc(static_cast<size_t>(count) * 4);
    if (!rc) rc = o_row.alloc(static_cast<size_t>(count) * 8);
    if (rc) return rc;
    A.io.hops = o_hops.as<int32_t>(); A.io.rels = o_rels.as<int8_t>(); A.io.ncred = o_nc.as<int32_t>(); A.io.ntool = o_nt.as<int32_t>(); A.io.row_cap = count;
    if ((rc = LAUNCH(rank_gather_kernel, static_cast<unsigned>((count + 255) / 256), 256, 0, st, A, RA, row_out, first, count, o_rank.as<uint32_t>(),
                     o_row.as<int64_t>())))
        return rc;
    r->hops.resize(static_cast<size_t>(count) * 4); r->rels.resize(static_cast<size_t>(count) * 4); r->ncred.resize(count); r->ntool.resize(count);
    r->risk_rank.resize(count); r->row.resize(count);
    cudaError_t ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->hops.data(), o_hops.p, static_cast<size_t>(count) * 16, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->rels.data(), o_rels.p, static_cast<size_t>(count) * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->ncred.data(), o_nc.p, static_cast<size_t>(count) * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->ntool.data(), o_nt.p, static_cast<size_t>(count) * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->risk_rank.data(), o_rank.p, static_cast<size_t>(count) * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->row.data(), o_row.p, static_cast<size_t>(count) * 8, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) return fail(ABB_ERR_CUDA, "ranking failed: %s", cudaGetErrorString(ce));
    *out = r.release();
    return ABB_OK;
}

extern "C" int abb_paths_rank_host(abb_graph *g, const int32_t *findings, int64_t n_findings, const int32_t *base_id, const uint32_t *risk_rank, int64_t n_base,
                                   const int32_t *ncu, const int32_t *ntu, int64_t offset, int64_t limit, abb_rank_result **out) {
    NvtxRange nvtx_("abb_paths_rank_host");
    return paths_rank(g, findings, n_findings, base_id, risk_rank, n_base, ncu, ntu, nullptr, 0, offset, limit, out);
}

extern "C" int abb_paths_rank_focus_host(abb_graph *g, const int32_t *findings, int64_t n_findings, const int32_t *base_id, const uint32_t *risk_rank,
                                         int64_t n_base, const int32_t *ncu, const int32_t *ntu, const uint8_t *node_focus, uint32_t need, int64_t offset,
                                         int64_t limit, abb_rank_result **out) {
    NvtxRange nvtx_("abb_paths_rank_focus_host");
    return paths_rank(g, findings, n_findings, base_id, risk_rank, n_base, ncu, ntu, node_focus, need, offset, limit, out);
}

extern "C" int abb_exposure_host(abb_graph *g, const int32_t *findings, int64_t n_findings, int32_t max_depth, abb_walk_result **impact_out,
                                 abb_paths_result **paths_out) {
    NvtxRange nvtx_("abb_exposure_host");
    if (!g || !impact_out || !paths_out || n_findings < 0 || (n_findings && !findings)) return fail(ABB_ERR_ARG, "bad arguments");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    const bool trace = getenv("ABB_TRACE") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = now();
    // The exposure-path pipeline does not depend on the walk: it runs on its own stream, driven by a helper thread (sizing its
    // factorised result synchronises that stream twice), while this thread stages and runs the walk.  The walk's node arena streams to the host over PCIe
    // as it is produced (zero-copy); the path pipeline's kernels and its factorised result copy fit inside that window.
    // Both threads use g under the one lock held here, so the two halves must touch disjoint state.  The path half (paths_run and
    // what it calls) uses only g->v, g->sm_count, g->device, g->paths_stream, g->paths and g->exposure; the walk half uses the walk's
    // workspaces (g->tiers, g->dedup, g->staging, g->chunked) and never g->paths, g->exposure or g->context.
    abb_paths_result *pr = nullptr;
    int prc = ABB_OK;
    std::string perr;
    std::thread helper([&] {
        DeviceGuard hdg(g->device);
        prc = paths_run(g, findings, nullptr, n_findings, &pr, g->paths_stream);
        if (prc) perr = g_err;
    });
    abb_walk_spec spec = abb_spec_impact_of(max_depth);
    abb_walk_io io{}; unsigned long long totals[3] = {0, 0, 0}; int64_t h2d = 0;
    HostBlock direct;
    abb_walk_result *wr = nullptr;
    int rc = chunked_applies(g, &spec, nullptr, nullptr, n_findings) ? walk_host_chunked(g, &spec, findings, n_findings, &wr) : ABB_RETRY_UNCHUNKED;
    auto t1 = now();
    if (rc == ABB_RETRY_UNCHUNKED) {
        g->chunked.last_host_chunks = 1;
        rc = walk_device_stage(g, &spec, findings, nullptr, nullptr, n_findings, &io, totals, &h2d, &direct);
        t1 = now();
        if (!rc) rc = walk_collect(g, &spec, io, totals, h2d, &wr, true, &direct);
    }
    const auto t2 = now();
    helper.join();
    const auto t3 = now();
    if (rc || prc) {
        delete wr;
        delete pr;
        if (!rc) { g_err = perr; return prc; }
        return rc;
    }
    if (trace) fprintf(stderr, "[abb] exposure_host: stage+walk %.2f ms, result copies %.2f ms, wait for the path pipeline %.2f ms\n", ms(t0, t1), ms(t1, t2), ms(t2, t3));
    *impact_out = wr; *paths_out = pr;
    return ABB_OK;
}

// ------------------------------------------------------------------ finding context (context.cuh)
struct abb_finding_context_result {
    int64_t nq = 0, total = 0, h2d = 0, d2h = 0;
    float walk_ms = -1.f, context_ms = -1.f;
    std::unique_ptr<abb_walk_result> walk;   // count / maxd / flags / histogram of the impact walk; no slices
    HostBlock start, bcnt, src;
};
extern "C" void abb_finding_context_result_free(abb_finding_context_result *r) { delete r; }
extern "C" int64_t abb_finding_context_result_queries(const abb_finding_context_result *r) { return r->nq; }
extern "C" const int32_t *abb_finding_context_result_count(const abb_finding_context_result *r) { return abb_walk_result_count(r->walk.get()); }
extern "C" const int32_t *abb_finding_context_result_maxd(const abb_finding_context_result *r) { return abb_walk_result_maxd(r->walk.get()); }
extern "C" const int32_t *abb_finding_context_result_flags(const abb_finding_context_result *r) { return abb_walk_result_flags(r->walk.get()); }
extern "C" const void *abb_finding_context_result_hist_packed(const abb_finding_context_result *r, uint32_t *columns_mask, int32_t *bytes_per_count) {
    return abb_walk_result_hist_packed(r->walk.get(), columns_mask, bytes_per_count);
}
extern "C" const uint32_t *abb_finding_context_result_hist(const abb_finding_context_result *r) { return abb_walk_result_hist(r->walk.get()); }
extern "C" const int64_t *abb_finding_context_result_start(const abb_finding_context_result *r) { return r->start.as<int64_t>(); }
extern "C" const int32_t *abb_finding_context_result_bucket_counts(const abb_finding_context_result *r) { return r->bcnt.as<int32_t>(); }
extern "C" int64_t abb_finding_context_result_total_sources(const abb_finding_context_result *r) { return r->total; }
extern "C" const int32_t *abb_finding_context_result_sources(const abb_finding_context_result *r) { return r->src.as<int32_t>(); }
extern "C" int64_t abb_finding_context_result_h2d_bytes(const abb_finding_context_result *r) { return r->h2d; }
extern "C" int64_t abb_finding_context_result_d2h_bytes(const abb_finding_context_result *r) { return r->d2h; }
extern "C" float abb_finding_context_result_walk_ms(const abb_finding_context_result *r) { return r->walk_ms; }
extern "C" float abb_finding_context_result_context_ms(const abb_finding_context_result *r) { return r->context_ms; }

// The findings are staged once.  The context count pass and its scan run on paths_stream while this thread runs the impact walk on the
// main stream into a device arena (walk_device_stage without a host block); then the fill pass runs on paths_stream while the walk's
// per-finding arrays (not its slices) are copied back on the main stream.
extern "C" int abb_finding_context_host(abb_graph *g, int32_t max_depth, const int32_t *findings, int64_t n_findings, abb_finding_context_result **out) {
    NvtxRange nvtx_("abb_finding_context_host");
    if (!g || !out || n_findings < 0 || (n_findings && !findings)) return fail(ABB_ERR_ARG, "bad arguments");
    if (n_findings >= (1ll << 31) - 2) return fail(ABB_ERR_ARG, "too many findings in one batch");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = g->stream, cs = g->paths_stream;
    ContextWorkspace &cx = g->context;
    DevBuf &scan_tmp = g->paths.scan_tmp;   // the path pipeline's scan scratch: it runs on paths_stream too, never during this call
    const int64_t nq = n_findings;
    const size_t q = static_cast<size_t>(nq), q1 = q + 1;
    auto drain = [&]() { cudaStreamSynchronize(st); cudaStreamSynchronize(cs); };
    int rc = ABB_OK;
    ENS(g->staging.roots, q1 * 4); ENS(cx.bcnt, q1 * CTX_BUCKETS * 4); ENS(cx.cnt, q1 * 8); ENS(cx.start, q1 * 8);
    if (rc) return rc;
    std::unique_ptr<abb_finding_context_result> r(new abb_finding_context_result());
    r->nq = nq;
    if (nq) CUDA_TRY(cudaMemcpyAsync(g->staging.roots.p, findings, q * 4, cudaMemcpyHostToDevice, st));
    r->h2d = nq * 4;
    CUDA_TRY(cudaEventRecord(cx.staged, st));
    CUDA_TRY(cudaStreamWaitEvent(cs, cx.staged, 0));
    // count pass + scan, next to the walk
    CtxArgs A{};
    A.g = g->v; A.findings = g->staging.roots.as<int32_t>(); A.n = nq;
    A.bcnt = cx.bcnt.as<int32_t>(); A.cnt = cx.cnt.as<int64_t>(); A.start = cx.start.as<int64_t>();
    const unsigned grid = warp_grid(g, (nq + 31) / 32);
    CUDA_TRY(cudaEventRecord(cx.ev[0], cs));
    CUDA_TRY(cudaMemsetAsync(A.cnt, 0, q1 * 8, cs));
    if (nq) if ((rc = LAUNCH(context_kernel<false>, grid, 256, 0, cs, A))) { drain(); return rc; }
    if ((rc = scan_i64(scan_tmp, A.cnt, cx.start.as<int64_t>(), nq + 1, cs))) { drain(); return rc; }
    CUDA_TRY(cudaEventRecord(cx.ev[1], cs));
    // the impact walk, unchanged, into the device arena
    const abb_walk_spec spec = abb_spec_impact_of(max_depth);
    abb_walk_io io{}; unsigned long long totals[3] = {0, 0, 0}; int64_t wh2d = 0;
    g->chunked.last_host_chunks = 1;
    if ((rc = walk_device_stage(g, &spec, findings, nullptr, nullptr, nq, &io, totals, &wh2d, nullptr, true))) { drain(); return rc; }
    int64_t total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, cx.start.as<int64_t>() + nq, 8, cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(cudaStreamSynchronize(cs));
    r->total = total;
    ENS(cx.src, (total + 1) * 4);
    if (rc) { drain(); return rc; }
    if (!(r->start.alloc(q * 8) && r->bcnt.alloc(q * CTX_BUCKETS * 4) && r->src.alloc(static_cast<size_t>(total) * 4))) {
        drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    }
    // fill pass and its copies on paths_stream, the walk's per-finding arrays on the main stream
    A.src = cx.src.as<int32_t>();
    CUDA_TRY(cudaEventRecord(cx.ev[2], cs));
    if (nq) if ((rc = LAUNCH(context_kernel<true>, grid, 256, 0, cs, A))) { drain(); return rc; }
    CUDA_TRY(cudaEventRecord(cx.ev[3], cs));
    Readback d2h{cs, &r->d2h, cudaGetLastError()};
    d2h(r->start, cx.start.p, q * 8); d2h(r->bcnt, cx.bcnt.p, q * CTX_BUCKETS * 4); d2h(r->src, cx.src.p, static_cast<size_t>(total) * 4);
    cudaError_t e = d2h.err;
    if (e != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "finding context failed: %s", cudaGetErrorString(e)); }
    abb_walk_result *walk = nullptr;
    if ((rc = walk_collect(g, &spec, io, totals, wh2d, &walk, true, nullptr, false))) { drain(); return rc; }
    r->walk.reset(walk);
    if ((e = cudaStreamSynchronize(cs)) != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "finding context failed: %s", cudaGetErrorString(e)); }
    r->d2h += r->walk->d2h;
    float a = 0.f, b = 0.f;
    if (cudaEventElapsedTime(&a, g->staging.ev_start, g->staging.ev_end) == cudaSuccess) r->walk_ms = a;
    if (cudaEventElapsedTime(&a, cx.ev[0], cx.ev[1]) == cudaSuccess && cudaEventElapsedTime(&b, cx.ev[2], cx.ev[3]) == cudaSuccess) r->context_ms = a + b;
    *out = r.release();
    return ABB_OK;
}

#include "reach_host.inl"
#include "union_host.inl"
#include "centrality_host.inl"
#include "nxcentral_host.inl"
#include "lateral_host.inl"
#include "clusters_host.inl"
#include "delta_host.inl"
#include "lookup_host.inl"
#include "search_host.inl"
#include "compliance_host.inl"
#include "lifecycle_host.inl"
#include "hops_host.inl"

// Runs with the graph's device current (abb_graph_free); the workspaces' events and buffers and the tables free themselves after it.
abb_graph::~abb_graph() {
    for (cudaStream_t s : {stream, copy_stream, paths_stream}) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
}
