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

// grows workspace buffer g->buf; needs `g` and `int rc` in scope and keeps the first error in rc
#define ENS(buf, bytes) if (!rc) rc = g->buf.ensure(static_cast<size_t>(bytes))

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

struct abb_graph {
    int device = 0;
    GraphView v{};
    int64_t bytes = 0;
    int sm_count = 132;               // H100 SXM; set from the device in graph_finish_init
    mutable std::mutex mu;            // serialises use of the shared workspace and of the snapshot tables
    cudaStream_t stream = nullptr;    // host-API stream
    cudaStream_t copy_stream = nullptr;   // result copies that may overlap later kernels of the same call
    cudaStream_t paths_stream = nullptr;  // exposure-path pipeline of abb_exposure_host, run next to the walk
    cudaEvent_t ev_copy = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool walk_timed = false, paths_timed = false;
    // tier bookkeeping
    DevBuf ctl, ov1, ov2, ov3, ov4;
    // block tiers (walkb.cuh): mid = 8 warps, queue + table in shared memory; big = 32 warps, 192 KB table, queue in a global scratch slot per block
    int block_tiers = 2;              // bit 0: mid tier (off by default: measured no faster than G1), bit 1: big tier (ABB_BLOCK_TIERS / abb_graph_set_option)
    int mid_slots = 8192, mid_qcap = 4096, big_slots = 49152, big_qcap = 36864;
    int big_grid = 0;
    int mid_warps = 8;                // ABB_MID_WARPS=4: 4-warp mid blocks
    int64_t big_limit = 0;            // the big tier takes S1's heavy hand-offs when there are at most this many (default 24 per SM)
    int64_t nx_batch = 0;             // cap on betweenness sources per batch and on path-search slots (0: sized from free memory)
    DevBuf b_gq, b_gpar, b_gdep;
    // tier G1: many per-warp slots (bitmap over all nodes + a bounded queue); tier GX: a few slots that can hold a whole-graph walk
    DevBuf g_bitmap, g_queue, g_par, g_dep;
    int g_slots = 0; int64_t g_words = 0, g_qcap = 0;
    DevBuf x_bitmap, x_queue, x_par, x_dep;
    int x_slots = 0; int64_t x_qcap = 0;
    // root-frontier de-duplication workspace
    DevBuf dd_sig, dd_ssig, dd_q, dd_sq, dd_head, dd_gid, dd_hp, dd_glen, dd_goff, dd_arena, dd_memoff, dd_memsrc, dd_memstate, dd_indiv, dd_cnt, dd_tmp;
    DevBuf dd_gstart, dd_gcount, dd_gmaxd, dd_gflags, dd_ghist, dd_lkey, dd_lkey2, dd_lgid, dd_order;
    bool locality_order = true;   // walk the frontier groups in first-seed order (ABB_LOCALITY=0 disables)
    bool dedup_enabled = true;
    int slice_align = 0;        // set while a host-mapped arena is the walk target
    bool align_direct = true;
    bool hist_pack = true;      // host results carry only the non-zero histogram columns at the narrowest width (histpack.cuh)
    DevBuf d_histinfo, d_hist_packed;
    unsigned long long hist_info[2] = {0, 0};   // column mask, largest count of the walk just staged
    bool hist_info_valid = false;
    // chunked host walks (walk_host_chunked): a large plain batch is walked in `chunks` consecutive source ranges; each range's node arena
    // is DMA-copied to the host while the next range is walked (two device arenas, ping-pong)
    int chunks = 8;                  // ABB_CHUNKS / option "chunks"; applies to batches of >= chunk_min queries (measured at L: 1 piece 43.9 ms, 4: 42.4, 8: 40.6)
    int64_t chunk_min = 2 << 20;
    DevBuf d_nodes_alt, ck_roots, ck_sig, ck_key, ck_key2, ck_idx, ck_order, ck_counts, ck_tmp, ck_qstart, ck_qcount, ck_qmaxd, ck_qflags, ck_qhist;
    cudaEvent_t ev_chunk_walked = nullptr, ev_chunk_copied[2] = {nullptr, nullptr};
    std::vector<int64_t> chunk_hint;   // nodes each chunk produced last time (same batch size / chunk count)
    int64_t chunk_hint_nq = -1;
    // size hint of the last PLAIN host walk (single roots, no parents / depths / edges), per spec: what the chunked path sizes its arenas from
    abb_walk_spec plain_spec{};
    int64_t plain_nq = -1, plain_nodes = 0;
    int last_host_chunks = 1;        // how many ranges the last host-buffer walk was split into (get_option "last_host_chunks")
    bool zero_copy = true;      // host-API walks write the node arena straight into pinned host memory when its size is known
    int64_t last_walk_queries = 0;
    bool last_walk_dedup = false;
    int s1_minb = 5;
    DevBuf identity_rank;
    // host-API staging
    DevBuf d_roots, d_root_off, d_targets, d_qstart, d_qcount, d_qmaxd, d_qflags, d_qestart, d_qecount, d_qhist;
    DevBuf d_nodes, d_parent, d_depth, d_edges, d_totals;
    int64_t hint_nodes = 0, hint_edges = 0, hint_nq = 0, hint_last_nodes = 0;
    // graph-constant server tables (built on first use): fan-out, and the principal rows each server contributes to a template
    DevBuf srv_cred, srv_tool, srv_roff, srv_row, srv_rel;
    bool srv_table_ready = false;
    // graph-constant exposure tables (built on first use, ensure_exposure_tables): links of every finding node, templates of every
    // vulnerable source, rows per finding node
    DevBuf x_vs, x_loff, x_link, x_rows, x_toff, x_trow, x_trel, x_overflow;
    bool x_tables_ready = false;
    // paths staging
    DevBuf p_findings, p_off, p_scan_tmp;
    // exposure-path per-call workspace: rows and links per finding; the host result's batch links and templates
    DevBuf pl_cnt, pl_link, pl_lcnt, pl_off, pl_vs, pl_rel, pl_roff, pl_toff, pl_need, pl_ulist, pl_nu, pt_cnt, pt_off, pt_off_node, pt_row, pt_rel;
    PathsArgs paths_args{};
    bool paths_args_valid = false;
    int replicate_grid = 0, rank_keys_grid = 0;   // grids of the row-parallel kernels (row_grid)
    int64_t hint_rows = 0;
    // finding-context workspace (context.cuh): per-finding bucket counts, totals, start offsets, source lists; the context kernels run on
    // paths_stream next to the impact walk (cx_staged: the findings are on the device), cx_ev time the count and fill passes
    DevBuf cx_bcnt, cx_cnt, cx_start, cx_src;
    cudaEvent_t cx_staged = nullptr;
    cudaEvent_t cx_ev[4] = {nullptr, nullptr, nullptr, nullptr};
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
    CUDA_TRY(cudaEventCreateWithFlags(&g->ev_copy, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&g->ev_chunk_walked, cudaEventDisableTiming));
    for (auto &e : g->ev_chunk_copied) CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (auto &e : g->ev) CUDA_TRY(cudaEventCreate(&e));
    CUDA_TRY(cudaEventCreateWithFlags(&g->cx_staged, cudaEventDisableTiming));
    for (auto &e : g->cx_ev) CUDA_TRY(cudaEventCreate(&e));
    if (int rc = g->ctl.ensure(CTL_WORDS * sizeof(unsigned long long))) return rc;
    const int64_t n = g->v.n;
    g->g_words = (n + 31) / 32 + 1;
    // tier G1: 40 warps per SM (latency-bound pointer chasing wants every warp it can get), queue bounded at 64K entries
    g->g_qcap = std::min<int64_t>(n + 4096, 1 << 16);
    g->g_slots = g->sm_count * 40;
    if (const char *e = getenv("ABB_G1_WARPS_PER_SM")) g->g_slots = g->sm_count * std::max(4, std::min(48, atoi(e)));
    {
        const size_t sl = static_cast<size_t>(g->g_slots);
        if (int rc = g->g_bitmap.ensure(sl * g->g_words * 4)) return rc;
        if (int rc = g->g_queue.ensure(sl * g->g_qcap * 4)) return rc;
        if (int rc = g->g_par.ensure(sl * g->g_qcap * 4)) return rc;
        if (int rc = g->g_dep.ensure(sl * g->g_qcap * 4)) return rc;
        CUDA_TRY(cudaMemset(g->g_bitmap.p, 0, sl * g->g_words * 4));
    }
    // tier GX: 8 slots that can hold any walk (every node once + re-seeded roots)
    g->x_qcap = n + 4096;
    g->x_slots = 8;
    {
        const size_t sl = static_cast<size_t>(g->x_slots);
        if (int rc = g->x_bitmap.ensure(sl * g->g_words * 4)) return rc;
        if (int rc = g->x_queue.ensure(sl * g->x_qcap * 4)) return rc;
        if (int rc = g->x_par.ensure(sl * g->x_qcap * 4)) return rc;
        if (int rc = g->x_dep.ensure(sl * g->x_qcap * 4)) return rc;
        CUDA_TRY(cudaMemset(g->x_bitmap.p, 0, sl * g->g_words * 4));
    }
    if (const char *e = getenv("ABB_DEDUP")) g->dedup_enabled = atoi(e) != 0;
    if (const char *e = getenv("ABB_BLOCK_TIERS")) g->block_tiers = atoi(e) & 3;
    if (const char *e = getenv("ABB_LOCALITY")) g->locality_order = atoi(e) != 0;
    g->big_grid = g->sm_count;
    g->big_limit = 24ll * g->sm_count;
    if (const char *e = getenv("ABB_BIG_LIMIT")) g->big_limit = atoll(e);
    if (const char *e = getenv("ABB_MID_WARPS")) g->mid_warps = atoi(e) == 4 ? 4 : 8;
    if (const char *e = getenv("ABB_S1_MINB")) g->s1_minb = atoi(e) == 4 ? 4 : 5;
    if (const char *e = getenv("ABB_ZEROCOPY")) g->zero_copy = atoi(e) != 0;
    if (const char *e = getenv("ABB_HIST_PACK")) g->hist_pack = atoi(e) != 0;
    if (const char *e = getenv("ABB_CHUNKS")) g->chunks = std::max(1, std::min(64, atoi(e)));
    if (const char *e = getenv("ABB_CHUNK_MIN")) g->chunk_min = std::max<int64_t>(2, atoll(e));
    if (const char *e = getenv("ABB_ALIGN_DIRECT")) g->align_direct = atoi(e) != 0;
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
    g->dedup_enabled = enabled != 0;
    return ABB_OK;
}
extern "C" int abb_graph_device(const abb_graph *g) { return g ? g->device : -1; }

// Tuning / test switches of a graph handle.  Results never depend on them (every tier is bit-identical; the GPU tests
// run the suite with the block tiers on, off and shrunk so that every hand-off between tiers is exercised).
extern "C" int abb_graph_set_option(abb_graph *g, const char *name, int64_t value) {
    if (!g || !name) return fail(ABB_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(g->mu);
    const std::string k(name);
    if (k == "dedup") g->dedup_enabled = value != 0;
    else if (k == "block_tiers") g->block_tiers = static_cast<int>(value) & 3;
    else if (k == "mid_qcap") {
        if (value < 32 || value > 4096) return fail(ABB_ERR_ARG, "mid_qcap must be in [32, 4096]");
        g->mid_qcap = static_cast<int>(value);
    } else if (k == "big_qcap") {
        if (value < 32 || value > 36864) return fail(ABB_ERR_ARG, "big_qcap must be in [32, 36864]");
        g->big_qcap = static_cast<int>(value);
    } else if (k == "zero_copy") g->zero_copy = value != 0;
    else if (k == "hist_pack") g->hist_pack = value != 0;
    else if (k == "chunks") {
        if (value < 1 || value > 64) return fail(ABB_ERR_ARG, "chunks must be in [1, 64]");
        g->chunks = static_cast<int>(value);
    } else if (k == "chunk_min") {
        if (value < 2) return fail(ABB_ERR_ARG, "chunk_min must be >= 2");
        g->chunk_min = value;
    }
    else if (k == "big_limit") {
        if (value < 0) return fail(ABB_ERR_ARG, "big_limit must be >= 0");
        g->big_limit = value;
    } else if (k == "nx_batch") {
        if (value < 0) return fail(ABB_ERR_ARG, "nx_batch must be >= 0");
        g->nx_batch = value;
    } else if (k == "delta_union_limit") {
        if (value < 0 || value > DL_UNION_LIMIT) return fail(ABB_ERR_ARG, "delta_union_limit must be in [0, 2^27]");
        g->dl_union_limit = value;
    } else return fail(ABB_ERR_ARG, "unknown option '%s'", name);
    return ABB_OK;
}
extern "C" int64_t abb_graph_get_option(const abb_graph *g, const char *name) {
    if (!g || !name) return -1;
    const std::string k(name);
    if (k == "dedup") return g->dedup_enabled;
    if (k == "block_tiers") return g->block_tiers;
    if (k == "mid_qcap") return g->mid_qcap;
    if (k == "big_qcap") return g->big_qcap;
    if (k == "zero_copy") return g->zero_copy;
    if (k == "hist_pack") return g->hist_pack;
    if (k == "chunks") return g->chunks;
    if (k == "chunk_min") return g->chunk_min;
    if (k == "last_host_chunks") return g->last_host_chunks;
    if (k == "big_limit") return g->big_limit;
    if (k == "nx_batch") return g->nx_batch;
    if (k == "delta_union_limit") return g->dl_union_limit;
    return -1;
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
#define V(P, M, B) if (par == P && meta == M && bud == B) return g->s1_minb == 4 ? launch_smem<H, Q, WARPS, P, M, B, 4>(g, A, max_items, st) : launch_smem<H, Q, WARPS, P, M, B, 5>(g, A, max_items, st)
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
    int32_t *ovs[4] = {g->ov1.as<int32_t>(), g->ov2.as<int32_t>(), g->ov3.as<int32_t>(), g->ov4.as<int32_t>()};
    A.list_cap = max_items;
    A.slice_align = g->slice_align;
    // S1: two-ended hand-off list in ovs[0]
    A.ctl = ctl; A.overflow = ovs[0]; A.ov_cnt_front = ctl + 1; A.ov_cnt_back = ctl + 3;
    if (int rc = launch_smem_variant<S1_H, S1_Q, S1_WARPS>(g, A, max_items, par, meta, bud, st)) return rc;
    const int idb = ceil_log2_i64(std::max<int64_t>(g->v.n, 2));
    const bool plain = !bud && !(fl & (ABB_WALK_TARGET | ABB_WALK_EDGES));
    bool front_taken = false;                       // S1's heavy part routed (to the big tier when few, else first in line for the warp tier)
    unsigned long long *to_big = ctl + CTL_ROUTE, *to_warp = ctl + CTL_ROUTE + 1;
    if (plain && (g->block_tiers & 2) && idb <= 26) {
        if (int rc = LAUNCH(route_heavy_kernel, 1, 1, 0, st, ctl + 1, to_big, to_warp, static_cast<unsigned long long>(g->big_limit))) return rc;
        // big tier: the heavy (front) part of S1's list; what it cannot hold goes to a list of its own (ovs[2]) that the next tier
        // reads after S1's back part — NOT onto S1's list: front + back may already fill it
        A.qlist = ovs[0]; A.nq = 0; A.nq_dev = to_big; A.nq_back_dev = nullptr; A.ctl = ctl + 4 * 1;
        A.overflow = ovs[2]; A.ov_cnt_front = ctl + 4 * 1 + 1; A.ov_cnt_back = nullptr;
        const size_t words = static_cast<size_t>(g->big_grid) * g->big_qcap;
        if (int rc = g->b_gq.ensure(words * 4)) return rc;
        if (par) if (int rc = g->b_gpar.ensure(words * 4)) return rc;
        if (fl & ABB_WALK_DEPTHS) if (int rc = g->b_gdep.ensure(words * 4)) return rc;
        BlockTier T{static_cast<uint32_t>(g->big_slots), g->big_qcap, idb, g->b_gq.as<int32_t>(), g->b_gpar.as<int32_t>(), g->b_gdep.as<int32_t>()};
        int rc = meta ? launch_block<32, false, true, true, 1>(g, A, T, g->big_grid, st) : launch_block<32, false, true, false, 1>(g, A, T, g->big_grid, st);
        if (rc) return rc;
        front_taken = true;
    }
    // what the next tier reads: S1's list (its back part, or front then back), or the mid tier's plain list
    const unsigned long long *in_front = front_taken ? to_warp : ctl + 1, *in_back = ctl + 3;
    int32_t *in_list = ovs[0];
    const int32_t *in_list2 = front_taken ? ovs[2] : nullptr;
    const unsigned long long *in_cnt2 = front_taken ? ctl + 4 * 1 + 1 : nullptr;
    if (plain && (g->block_tiers & 1) && idb <= 28) {
        A.qlist = in_list; A.nq = 0; A.nq_dev = in_front; A.nq_back_dev = in_back; A.qlist2 = in_list2; A.nq2_dev = in_cnt2; A.ctl = ctl + 4 * 2;
        A.overflow = ovs[1]; A.ov_cnt_front = ctl + 4 * 2 + 1; A.ov_cnt_back = nullptr;
        BlockTier T{static_cast<uint32_t>(g->mid_slots), g->mid_qcap, idb, nullptr, nullptr, nullptr};
        int rc;
        if (g->mid_warps == 4) {               // 4-warp blocks: half the table / queue, twice the walks in flight per SM
            T.slots = static_cast<uint32_t>(std::min(g->mid_slots, 4096)); T.qcap = std::min(g->mid_qcap, 2048);
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
    A.g_bitmap = g->g_bitmap.as<uint32_t>(); A.g_queue = g->g_queue.as<int32_t>(); A.g_par = g->g_par.as<int32_t>(); A.g_dep = g->g_dep.as<int32_t>();
    A.g_words = g->g_words; A.g_qcap = g->g_qcap;
    if (int rc = launch_global_variant(A, g->g_slots, g->sm_count, meta, bud, st)) return rc;
    // GX
    A.qlist = ovs[3]; A.nq_dev = ctl + 4 * 3 + 1; A.nq_back_dev = nullptr; A.qlist2 = nullptr; A.nq2_dev = nullptr; A.ctl = ctl + 4 * 4; A.overflow = nullptr; A.ov_cnt_front = A.ov_cnt_back = nullptr;
    A.g_bitmap = g->x_bitmap.as<uint32_t>(); A.g_queue = g->x_queue.as<int32_t>(); A.g_par = g->x_par.as<int32_t>(); A.g_dep = g->x_dep.as<int32_t>();
    A.g_qcap = g->x_qcap;
    return launch_global_variant(A, g->x_slots, g->sm_count, meta, bud, st);
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
    ENS(dd_sig, q1 * 8); ENS(dd_ssig, q1 * 8); ENS(dd_q, q1 * 4); ENS(dd_sq, q1 * 4); ENS(dd_head, q1); ENS(dd_gid, q1 * 8); ENS(dd_hp, q1 * 8);
    ENS(dd_glen, q1 * 8); ENS(dd_goff, q1 * 8); ENS(dd_arena, q1 * 4 * L1_CAP); ENS(dd_memoff, q1 * 8); ENS(dd_memsrc, q1 * 4); ENS(dd_memstate, q1 * 4);
    ENS(dd_indiv, q1 * 4); ENS(dd_cnt, 8 * sizeof(unsigned long long));
    ENS(dd_lkey, q1 * 4); ENS(dd_lkey2, q1 * 4); ENS(dd_lgid, q1 * 4); ENS(dd_order, q1 * 4);
    ENS(dd_gstart, q1 * 8); ENS(dd_gcount, q1 * 4); ENS(dd_gmaxd, q1 * 4); ENS(dd_gflags, q1 * 4);
    if (fl & ABB_WALK_HIST) { ENS(dd_ghist, q1 * ABB_N_ENTITY_TYPES * 4); }
    if (rc) return rc;
    unsigned long long *cnt = g->dd_cnt.as<unsigned long long>();
    unsigned long long *sig = g->dd_sig.as<unsigned long long>(), *ssig = g->dd_ssig.as<unsigned long long>();
    int32_t *qi = g->dd_q.as<int32_t>(), *sq = g->dd_sq.as<int32_t>(), *indiv = g->dd_indiv.as<int32_t>();
    uint8_t *head = g->dd_head.as<uint8_t>();
    int64_t *gid = g->dd_gid.as<int64_t>(), *hp = g->dd_hp.as<int64_t>(), *glen = g->dd_glen.as<int64_t>(), *goff = g->dd_goff.as<int64_t>();
    int64_t *memoff = g->dd_memoff.as<int64_t>();
    const unsigned blocks = static_cast<unsigned>((nq + 255) / 256);
    CUDA_TRY(cudaMemsetAsync(cnt, 0, 8 * sizeof(unsigned long long), st));
    CUDA_TRY(cudaMemsetAsync(glen, 0, q1 * 8, st));
    if ((rc = LAUNCH(dedup_sig_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, nq, sig, qi))) return rc;
    if ((rc = cub_run(g->dd_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, sig, ssig, qi, sq, static_cast<int>(nq), 0, SIG_BITS, st); })))
        return rc;
    if ((rc = LAUNCH(dedup_heads_kernel, blocks, 256, 0, st, ssig, sq, nq, head, indiv, cnt))) return rc;
    cub::TransformInputIterator<int64_t, HeadToI64, const uint8_t *> head64(head, HeadToI64());
    if ((rc = cub_run(g->dd_tmp, [&](void *t, size_t &b) { return cub::DeviceScan::InclusiveSum(t, b, head64, gid, static_cast<int>(nq), st); }))) return rc;
    if ((rc = select_flagged(g->dd_tmp, head, hp, cnt, static_cast<int>(nq), st))) return rc;
    if ((rc = LAUNCH(dedup_groups_kernel, static_cast<unsigned>((nq + 1 + 255) / 256), 256, 0, st, g->v, *spec, io->roots, sq, hp, cnt, glen, memoff))) return rc;
    // glen is passed non-const here, unlike scan_i64's input: a different cub instantiation
    if ((rc = cub_run(g->dd_tmp, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, glen, goff, static_cast<int>(nq + 1), st); }))) return rc;
    if ((rc = LAUNCH(dedup_roots_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, sq, hp, cnt, goff, g->dd_arena.as<int32_t>()))) return rc;
    if ((rc = LAUNCH(dedup_members_kernel, blocks, 256, 0, st, g->v, *spec, io->roots, sq, head, gid, goff, g->dd_arena.as<int32_t>(), g->dd_memsrc.as<int32_t>(),
                     g->dd_memstate.as<int32_t>(), indiv, cnt)))
        return rc;
    unsigned long long *ctl = g->ctl.as<unsigned long long>();
    // canonical walks: one per group, seeded with the shared frontier, one level shallower, depths biased by one
    WalkArgs C{};
    C.g = g->v; C.spec = *spec; C.io = *io;
    C.spec.max_depth = spec->max_depth < 0 ? -1 : spec->max_depth - 1;
    C.spec.flags = (fl & ~(ABB_WALK_OMIT_ROOTS | ABB_WALK_REAL_ROOTS)) | ABB_WALK_MARK_ROOTS;
    C.io.roots = g->dd_arena.as<int32_t>(); C.io.root_off = goff;
    C.io.q_start = g->dd_gstart.as<int64_t>(); C.io.q_count = g->dd_gcount.as<int32_t>(); C.io.q_maxd = g->dd_gmaxd.as<int32_t>();
    C.io.q_flags = g->dd_gflags.as<int32_t>(); C.io.q_hist = g->dd_ghist.as<uint32_t>();
    C.qlist = nullptr; C.nq = 0; C.nq_dev = cnt;
    if (g->locality_order) {
        // walk order = first-seed order (a 2 M-key radix sort over the node-id bits, ~0.1 ms): neighbouring groups share rows in L2
        uint32_t *lkey = g->dd_lkey.as<uint32_t>(), *lkey2 = g->dd_lkey2.as<uint32_t>();
        int32_t *lgid = g->dd_lgid.as<int32_t>(), *order = g->dd_order.as<int32_t>();
        if ((rc = LAUNCH(dedup_locality_keys_kernel, blocks, 256, 0, st, cnt, goff, g->dd_arena.as<int32_t>(), lkey, lgid, nq))) return rc;
        if ((rc = cub_run(g->dd_tmp, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, lkey, lkey2, lgid, order, static_cast<int>(nq), 0, 32, st); })))
            return rc;
        C.qlist = order;
    }
    C.depth_bias = 1; C.hist_roots = 1;
    C.mem_off = memoff; C.mem_src = g->dd_memsrc.as<int32_t>(); C.mem_state = g->dd_memstate.as<int32_t>();
    if ((rc = enqueue_tiers(g, C, nq, ctl, st))) return rc;
    if ((rc = LAUNCH(dedup_share_kernel, grid_for(nq, 256, g->sm_count, 8), 256, 0, st,
                     sq, gid, g->dd_memstate.as<int32_t>(), cnt, C.io.q_start, C.io.q_count, C.io.q_maxd, C.io.q_flags, C.io.q_hist, io->q_start, io->q_count,
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
    return g->dedup_enabled && !io->root_off && io->n_queries >= 256 && (fl & ABB_WALK_MARK_ROOTS) && (fl & ABB_WALK_OMIT_ROOTS) &&
           !(fl & (ABB_WALK_TARGET | ABB_WALK_EDGES | ABB_WALK_PARENTS)) && spec->max_nodes < 0 && spec->max_edges < 0 && spec->max_depth != 0;
}

static int enqueue_walk(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, cudaStream_t st) {
    if (int rc = check_walk_io(spec, io)) return rc;
    CUDA_TRY(cudaMemsetAsync(io->totals, 0, 2 * sizeof(unsigned long long), st));
    if (io->n_queries == 0) return ABB_OK;
    if (int rc = g->ov1.ensure(static_cast<size_t>(io->n_queries) * 4)) return rc;
    if (int rc = g->ov2.ensure(static_cast<size_t>(io->n_queries) * 4)) return rc;
    if (int rc = g->ov3.ensure(static_cast<size_t>(io->n_queries) * 4)) return rc;
    if (int rc = g->ov4.ensure(static_cast<size_t>(io->n_queries) * 4)) return rc;
    CUDA_TRY(cudaMemsetAsync(g->ctl.p, 0, CTL_WORDS * sizeof(unsigned long long), st));
    g->last_walk_queries = io->n_queries;
    g->last_walk_dedup = dedup_applies(g, spec, io);
    if (g->last_walk_dedup) return enqueue_dedup_walk(g, spec, io, st);
    WalkArgs A{};
    A.g = g->v; A.spec = *spec; A.io = *io;
    A.qlist = nullptr; A.nq = io->n_queries; A.nq_dev = nullptr;
    return enqueue_tiers(g, A, io->n_queries, g->ctl.as<unsigned long long>(), st);
}

extern "C" int abb_walk_launch(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, void *stream) {
    NvtxRange nvtx_("abb_walk_launch");
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaEventRecord(g->ev[0], st));
    int rc = enqueue_walk(g, spec, io, st);
    if (rc) return rc;
    CUDA_TRY(cudaEventRecord(g->ev[1], st));
    g->walk_timed = true;
    return ABB_OK;
}

extern "C" int abb_walk_signatures(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, int64_t n, unsigned long long *sig, void *stream) {
    if (!g || !spec || n < 0 || (n && (!roots || !sig))) return fail(ABB_ERR_ARG, "bad arguments");
    if (!n) return ABB_OK;
    DeviceGuard dg(g->device);
    return LAUNCH(dedup_sig_kernel, static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream), g->v, *spec, roots, n, sig, nullptr);
}

extern "C" float abb_last_walk_ms(abb_graph *g) {
    if (!g || !g->walk_timed) return -1.f;
    DeviceGuard dg(g->device);
    float ms = -1.f;
    if (cudaEventSynchronize(g->ev[1]) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, g->ev[0], g->ev[1]) != cudaSuccess) return -1.f;
    return ms;
}
extern "C" int abb_last_walk_stats(abb_graph *g, int64_t *out4) {
    if (!g || !out4) return fail(ABB_ERR_ARG, "null argument");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    out4[0] = g->last_walk_queries; out4[1] = out4[2] = out4[3] = 0;
    if (g->last_walk_dedup && g->dd_cnt.p) {
        unsigned long long c[3] = {0, 0, 0};
        CUDA_TRY(cudaMemcpy(c, g->dd_cnt.p, sizeof c, cudaMemcpyDeviceToHost));
        out4[1] = static_cast<int64_t>(c[0]); out4[2] = static_cast<int64_t>(c[1]); out4[3] = static_cast<int64_t>(c[2]);
    }
    return ABB_OK;
}

extern "C" int abb_last_walk_tier_counts(abb_graph *g, int64_t *out8) {
    if (!g || !out8) return fail(ABB_ERR_ARG, "null argument");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    unsigned long long c[CTL_WORDS];
    CUDA_TRY(cudaMemcpy(c, g->ctl.p, sizeof c, cudaMemcpyDeviceToHost));
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
    if (!g || !g->paths_timed) return -1.f;
    DeviceGuard dg(g->device);
    float ms = -1.f;
    if (cudaEventSynchronize(g->ev[3]) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, g->ev[2], g->ev[3]) != cudaSuccess) return -1.f;
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
    CUDA_TRY(cudaMemcpy(&fatal, g->ctl.as<unsigned long long>() + CTL_FATAL, sizeof fatal, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&fatal2, g->ctl.as<unsigned long long>() + CTL_SET + CTL_FATAL, sizeof fatal2, cudaMemcpyDeviceToHost));
    if (fatal || fatal2) return fail(ABB_ERR_CAPACITY, "a traversal outgrew the global scratch tier (more than n_nodes+4096 queue entries)");
    return ABB_OK;
}

// the non-zero histogram columns and the largest count of nq rows, into g->hist_info once st has been synchronised
static int scan_hist_columns(abb_graph *g, const uint32_t *q_hist, int64_t nq, cudaStream_t st) {
    if (int rc = g->d_histinfo.ensure(2 * sizeof(unsigned long long))) return rc;
    CUDA_TRY(cudaMemsetAsync(g->d_histinfo.p, 0, 2 * sizeof(unsigned long long), st));
    if (int rc = LAUNCH(hist_columns_kernel, static_cast<unsigned>(g->sm_count) * 8, 256, 0, st, q_hist, nq * ABB_N_ENTITY_TYPES,
                        g->d_histinfo.as<unsigned long long>()))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(g->hist_info, g->d_histinfo.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    return ABB_OK;
}

// r's packed-histogram layout from g->hist_info: the non-zero columns, at 2 bytes per count when every count fits
static HistCols hist_layout(const abb_graph *g, abb_walk_result *r) {
    HistCols hc{};
    r->hist_is_packed = true;
    r->hist_mask = static_cast<uint32_t>(g->hist_info[0]);
    for (int t = 0; t < ABB_N_ENTITY_TYPES; t++) if (r->hist_mask >> t & 1u) hc.col[hc.k++] = static_cast<uint8_t>(t);
    r->hist_k = hc.k;
    r->hist_width = g->hist_info[1] < 65536ull ? 2 : 4;
    return hc;
}

// size hints for the next host walk: the largest node arena so far and the last batch; for a plain walk (one root per query, no
// parents / depths / edges / targets) also what the chunked path sizes its pieces from
static void note_walk_size(abb_graph *g, const abb_walk_spec *spec, int64_t nq, int64_t nodes, bool plain) {
    g->hint_nodes = std::max(g->hint_nodes, nodes);
    g->hint_nq = nq; g->hint_last_nodes = nodes;
    if (!plain) return;
    if (g->plain_nq != nq || memcmp(&g->plain_spec, spec, sizeof *spec) != 0) g->chunk_hint_nq = -1;
    g->plain_spec = *spec; g->plain_nq = nq; g->plain_nodes = nodes;
}

// stage inputs, run (re-run once if the arenas were too small), leave results on the device
// `direct_nodes`: when the result size is known from the previous call, the walk kernels write the node arena
// straight into that pinned host block (UVA), so the PCIe transfer of the largest output overlaps the traversal
// instead of following it; if the estimate turns out too small the walk is re-run into a device arena.
// `roots_staged`: the caller has already copied the single roots into g->d_roots on g->stream (sized for nq + 1).
static int walk_device_stage(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, const int64_t *root_off, const int32_t *targets,
                             int64_t nq, abb_walk_io *io_out, unsigned long long (&totals)[3], int64_t *h2d, HostBlock *direct_nodes = nullptr,
                             bool roots_staged = false) {
    cudaStream_t st = g->stream;
    const uint32_t fl = spec->flags;
    g->hist_info_valid = false;
    const int64_t n_roots = root_off ? root_off[nq] : nq;
    if (n_roots < 0) return fail(ABB_ERR_ARG, "bad root_off");
    const size_t q1 = static_cast<size_t>(nq) + 1;
    int rc = ABB_OK;
    ENS(d_roots, (n_roots + 1) * 4);
    if (root_off) ENS(d_root_off, q1 * 8);
    if (fl & ABB_WALK_TARGET) ENS(d_targets, q1 * 4);
    ENS(d_qstart, q1 * 8); ENS(d_qcount, q1 * 4); ENS(d_qmaxd, q1 * 4); ENS(d_qflags, q1 * 4);
    if (fl & ABB_WALK_EDGES) { ENS(d_qestart, q1 * 8); ENS(d_qecount, q1 * 8); }
    if (fl & ABB_WALK_HIST) ENS(d_qhist, q1 * ABB_N_ENTITY_TYPES * 4);
    ENS(d_totals, 3 * sizeof(unsigned long long));
    if (rc) return rc;
    *h2d = 0;
    if (n_roots && !roots_staged) { CUDA_TRY(cudaMemcpyAsync(g->d_roots.p, roots, static_cast<size_t>(n_roots) * 4, cudaMemcpyHostToDevice, st)); *h2d += n_roots * 4; }
    if (root_off) { CUDA_TRY(cudaMemcpyAsync(g->d_root_off.p, root_off, q1 * 8, cudaMemcpyHostToDevice, st)); *h2d += static_cast<int64_t>(q1) * 8; }
    if (fl & ABB_WALK_TARGET) { CUDA_TRY(cudaMemcpyAsync(g->d_targets.p, targets, static_cast<size_t>(nq) * 4, cudaMemcpyHostToDevice, st)); *h2d += nq * 4; }

    int64_t node_cap = std::max<int64_t>({g->hint_nodes, nq * 8, 1 << 16});
    int64_t edge_cap = (fl & ABB_WALK_EDGES) ? std::max<int64_t>({g->hint_edges, nq * 16, 1 << 16}) : 0;
    bool direct = direct_nodes && g->zero_copy && g->hint_nodes > 0 && !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES));
    if (direct) {
        // same batch size as last time: its exact need plus a little; otherwise scale the last per-query average generously, but
        // to no more than twice the largest arena any call has needed (a small batch of heavy sources, scaled to millions of
        // sources, would ask for more than the device holds; an estimate that is too small only costs a re-run into a device arena)
        node_cap = (nq == g->hint_nq) ? g->hint_last_nodes + g->hint_last_nodes / 64 + 4096 + (g->align_direct ? 32 * nq : 0)
                                      : std::min(static_cast<int64_t>(1.5 * static_cast<double>(g->hint_last_nodes) / std::max<int64_t>(g->hint_nq, 1) * nq) + 4096,
                                                 2 * node_cap);
        direct = direct_nodes->alloc(static_cast<size_t>(node_cap) * 4);
    }
    for (int attempt = 0; attempt < 3; attempt++) {
        if (!direct) ENS(d_nodes, node_cap * 4);
        if (fl & ABB_WALK_PARENTS) ENS(d_parent, node_cap * 4);
        if (fl & ABB_WALK_DEPTHS) ENS(d_depth, node_cap * 4);
        if (fl & ABB_WALK_EDGES) ENS(d_edges, edge_cap * 4);
        if (rc) return rc;
        abb_walk_io io{};
        io.n_queries = nq; io.roots = g->d_roots.as<int32_t>(); io.root_off = root_off ? g->d_root_off.as<int64_t>() : nullptr;
        io.targets = (fl & ABB_WALK_TARGET) ? g->d_targets.as<int32_t>() : nullptr;
        io.q_start = g->d_qstart.as<int64_t>(); io.q_count = g->d_qcount.as<int32_t>(); io.q_maxd = g->d_qmaxd.as<int32_t>(); io.q_flags = g->d_qflags.as<int32_t>();
        io.q_estart = g->d_qestart.as<int64_t>(); io.q_ecount = g->d_qecount.as<int64_t>(); io.q_hist = g->d_qhist.as<uint32_t>();
        io.nodes = direct ? direct_nodes->as<int32_t>() : g->d_nodes.as<int32_t>();
        io.parent = g->d_parent.as<int32_t>(); io.depth = g->d_depth.as<int32_t>(); io.node_cap = node_cap;
        io.edges = g->d_edges.as<uint32_t>(); io.edge_cap = edge_cap; io.totals = g->d_totals.as<unsigned long long>();
        CUDA_TRY(cudaEventRecord(g->ev[0], st));
        g->slice_align = (direct && g->align_direct) ? 32 : 0;
        CUDA_TRY(cudaMemsetAsync(g->d_totals.as<unsigned long long>() + 2, 0, sizeof(unsigned long long), st));
        int erc = enqueue_walk(g, spec, &io, st);
        g->slice_align = 0;
        if (erc) return erc;
        CUDA_TRY(cudaEventRecord(g->ev[1], st));
        g->walk_timed = true;
        const bool scan_hist = (fl & ABB_WALK_HIST) && g->hist_pack && nq >= 1024;
        if (scan_hist) if ((rc = scan_hist_columns(g, io.q_hist, nq, st))) return rc;
        CUDA_TRY(cudaMemcpyAsync(totals, g->d_totals.p, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        g->hist_info_valid = scan_hist;
        if ((rc = check_tier_fatal(g))) return rc;
        *io_out = io;
        const bool fits = static_cast<int64_t>(totals[0]) <= node_cap && (!(fl & ABB_WALK_EDGES) || static_cast<int64_t>(totals[1]) <= edge_cap);
        const bool plain = !root_off && !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES | ABB_WALK_TARGET));
        note_walk_size(g, spec, nq, static_cast<int64_t>(totals[0]), fits && plain);
        g->hint_edges = std::max<int64_t>(g->hint_edges, static_cast<int64_t>(totals[1]));
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
        CUDA_TRY(cudaEventRecord(g->ev_copy, g->stream));
        CUDA_TRY(cudaStreamWaitEvent(g->copy_stream, g->ev_copy, 0));
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
    const bool pack = (fl & ABB_WALK_HIST) && g->hist_info_valid;
    g->hist_info_valid = false;
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
            if (int rc = g->d_hist_packed.ensure(pbytes)) return rc;
            const unsigned grid = static_cast<unsigned>(g->sm_count) * 8;
            const int rc = r->hist_width == 2 ? LAUNCH(hist_pack_kernel<uint16_t>, grid, 256, 0, st, io.q_hist, nq, hc, g->d_hist_packed.as<uint16_t>())
                                              : LAUNCH(hist_pack_kernel<uint32_t>, grid, 256, 0, st, io.q_hist, nq, hc, g->d_hist_packed.as<uint32_t>());
            if (rc) return rc;
            d2h.keep(cudaGetLastError());
            d2h(r->q_hist_packed, g->d_hist_packed.p, pbytes);
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
    return g->chunks > 1 && nq >= g->chunk_min && nq >= 2 * g->chunks && !root_off && !targets &&
           !(fl & (ABB_WALK_PARENTS | ABB_WALK_DEPTHS | ABB_WALK_EDGES | ABB_WALK_TARGET)) && g->plain_nq == nq && g->plain_nodes > 0 &&
           memcmp(&g->plain_spec, spec, sizeof *spec) == 0;
}

static int walk_host_chunked(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, int64_t nq, abb_walk_result **out) {
    NvtxRange nvtx_("walk_host_chunked");
    cudaStream_t st = g->stream, cst = g->copy_stream;
    const uint32_t fl = spec->flags;
    const int K = g->chunks;
    const size_t q = static_cast<size_t>(nq), q1 = q + 1;
    const bool hist = (fl & ABB_WALK_HIST) != 0;
    int rc = ABB_OK;
    ENS(d_roots, q1 * 4); ENS(d_qstart, q1 * 8); ENS(d_qcount, q1 * 4); ENS(d_qmaxd, q1 * 4); ENS(d_qflags, q1 * 4);
    if (hist) ENS(d_qhist, q1 * ABB_N_ENTITY_TYPES * 4);
    ENS(d_totals, 3 * sizeof(unsigned long long));
    ENS(ck_roots, q1 * 4); ENS(ck_sig, q1 * 8); ENS(ck_key, q1 * 4); ENS(ck_key2, q1 * 4); ENS(ck_idx, q1 * 4); ENS(ck_order, q1 * 4); ENS(ck_counts, 64 * 8);
    ENS(ck_qstart, q1 * 8); ENS(ck_qcount, q1 * 4); ENS(ck_qmaxd, q1 * 4); ENS(ck_qflags, q1 * 4);
    if (rc) return rc;
    const bool have_hint = g->chunk_hint_nq == nq && static_cast<int>(g->chunk_hint.size()) == K;
    // host arena: last total plus slack (the one-piece zero-copy pass pads slices, so its total is an upper bound already)
    const int64_t host_cap = g->plain_nodes + g->plain_nodes / (have_hint ? 64 : 8) + 4096ll * K;
    std::unique_ptr<abb_walk_result> r(new abb_walk_result());
    r->nq = nq; r->flags = fl;
    if (!(r->q_start.alloc(q * 8) && r->q_count.alloc(q * 4) && r->q_maxd.alloc(q * 4) && r->q_flags.alloc(q * 4) && r->nodes.alloc(static_cast<size_t>(host_cap) * 4)))
        return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    auto drain = [&]() { cudaStreamSynchronize(st); cudaStreamSynchronize(cst); };
    const unsigned qblocks = static_cast<unsigned>((nq + 255) / 256);
    CUDA_TRY(cudaMemcpyAsync(g->d_roots.p, roots, q * 4, cudaMemcpyHostToDevice, st));
    r->h2d = nq * 4;
    CUDA_TRY(cudaEventRecord(g->ev[0], st));
    // partition: chunk = frontier signature mod K when the walk de-duplicates (a frontier group is never split), contiguous ranges otherwise
    abb_walk_io probe{}; probe.n_queries = nq;
    const bool by_sig = dedup_applies(g, spec, &probe);
    unsigned long long *sig = nullptr;
    if (by_sig) {
        sig = g->ck_sig.as<unsigned long long>();
        if ((rc = LAUNCH(dedup_sig_kernel, qblocks, 256, 0, st, g->v, *spec, g->d_roots.as<int32_t>(), nq, sig, nullptr))) { drain(); return rc; }
    }
    CUDA_TRY(cudaMemsetAsync(g->ck_counts.p, 0, 64 * 8, st));
    if ((rc = LAUNCH(chunk_key_kernel, qblocks, 256, 0, st, sig, nq, K, g->ck_key.as<uint32_t>(), g->ck_idx.as<int32_t>(), g->ck_counts.as<unsigned long long>()))) {
        drain(); return rc;
    }
    if ((rc = cub_run(g->ck_tmp, [&](void *t, size_t &b) {
             return cub::DeviceRadixSort::SortPairs(t, b, g->ck_key.as<uint32_t>(), g->ck_key2.as<uint32_t>(), g->ck_idx.as<int32_t>(), g->ck_order.as<int32_t>(),
                                                    static_cast<int>(nq), 0, 6, st);
         }))) { drain(); return rc; }
    const int32_t *order = g->ck_order.as<int32_t>();      // order[i] = caller index of the i-th query in chunk order
    if ((rc = LAUNCH(gather_i32_kernel, qblocks, 256, 0, st, g->d_roots.as<int32_t>(), order, g->ck_roots.as<int32_t>(), nq))) { drain(); return rc; }
    unsigned long long counts[64] = {0};
    CUDA_TRY(cudaMemcpyAsync(counts, g->ck_counts.p, 64 * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<int64_t> produced(static_cast<size_t>(K), 0);
    int64_t node_base = 0, b0 = 0;
    bool copied[2] = {false, false};
    for (int k = 0; k < K; k++) {
        const int64_t nk = static_cast<int64_t>(counts[k]);
        const int set = k & 1;
        if (!nk) continue;
        DevBuf &arena = set ? g->d_nodes_alt : g->d_nodes;
        int64_t cap = have_hint ? g->chunk_hint[static_cast<size_t>(k)] + g->chunk_hint[static_cast<size_t>(k)] / 64 + 4096
                                : 2 * (g->plain_nodes / K) + 65536;
        cap = std::max<int64_t>(cap, nk * 8);
        unsigned long long totals[3] = {0, 0, 0};
        bool done = false;
        for (int attempt = 0; attempt < 3 && !done; attempt++) {
            if (static_cast<size_t>(cap) * 4 > arena.cap && copied[set]) CUDA_TRY(cudaEventSynchronize(g->ev_chunk_copied[set]));   // about to reallocate it
            if ((rc = arena.ensure(static_cast<size_t>(cap) * 4))) { drain(); return rc; }
            if (copied[set]) CUDA_TRY(cudaStreamWaitEvent(st, g->ev_chunk_copied[set], 0));       // the arena's previous contents have left
            abb_walk_io io{};
            io.n_queries = nk; io.roots = g->ck_roots.as<int32_t>() + b0;
            io.q_start = g->d_qstart.as<int64_t>() + b0; io.q_count = g->d_qcount.as<int32_t>() + b0; io.q_maxd = g->d_qmaxd.as<int32_t>() + b0;
            io.q_flags = g->d_qflags.as<int32_t>() + b0;
            io.q_hist = hist ? g->d_qhist.as<uint32_t>() + b0 * ABB_N_ENTITY_TYPES : nullptr;
            io.nodes = arena.as<int32_t>(); io.node_cap = cap; io.totals = g->d_totals.as<unsigned long long>();
            CUDA_TRY(cudaMemsetAsync(g->d_totals.as<unsigned long long>() + 2, 0, sizeof(unsigned long long), st));
            if (int erc = enqueue_walk(g, spec, &io, st)) { drain(); return erc; }
            CUDA_TRY(cudaMemcpyAsync(totals, g->d_totals.p, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            if ((rc = check_tier_fatal(g))) { drain(); return rc; }
            if (static_cast<int64_t>(totals[0]) <= cap) done = true; else cap = static_cast<int64_t>(totals[0]) + 4096;
        }
        if (!done) { drain(); return fail(ABB_ERR_CAPACITY, "walk arenas still too small after resize"); }
        const int64_t tot = static_cast<int64_t>(totals[0]);
        produced[static_cast<size_t>(k)] = tot;
        if (node_base + tot > host_cap) {          // the host arena guess was too small: let the one-piece path redo the batch
            drain();
            g->chunk_hint_nq = -1;
            return ABB_RETRY_UNCHUNKED;
        }
        if (node_base)
            if ((rc = LAUNCH(add_base_kernel, static_cast<unsigned>((nk + 255) / 256), 256, 0, st, g->d_qstart.as<int64_t>() + b0, nk, node_base))) { drain(); return rc; }
        CUDA_TRY(cudaEventRecord(g->ev_chunk_walked, st));
        CUDA_TRY(cudaStreamWaitEvent(cst, g->ev_chunk_walked, 0));
        if (tot) CUDA_TRY(cudaMemcpyAsync(r->nodes.as<int32_t>() + node_base, arena.p, static_cast<size_t>(tot) * 4, cudaMemcpyDeviceToHost, cst));
        CUDA_TRY(cudaEventRecord(g->ev_chunk_copied[set], cst));
        copied[set] = true;
        node_base += tot;
        b0 += nk;
    }
    if (b0 != nq) { drain(); return fail(ABB_ERR_CUDA, "chunk partition lost queries (%lld of %lld)", static_cast<long long>(b0), static_cast<long long>(nq)); }
    CUDA_TRY(cudaEventRecord(g->ev[1], st));
    g->walk_timed = true;
    r->total_nodes = node_base;
    r->d2h += node_base * 4;
    // per-query results back into caller order, then to the host (the node copies of the last chunks are still in flight on the copy stream)
    const unsigned sgrid = static_cast<unsigned>(g->sm_count) * 8;
    if ((rc = LAUNCH(scatter_rows_kernel<int64_t>, sgrid, 256, 0, st, g->d_qstart.as<int64_t>(), order, g->ck_qstart.as<int64_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, g->d_qcount.as<int32_t>(), order, g->ck_qcount.as<int32_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, g->d_qmaxd.as<int32_t>(), order, g->ck_qmaxd.as<int32_t>(), nq, 1)) ||
        (rc = LAUNCH(scatter_rows_kernel<int32_t>, sgrid, 256, 0, st, g->d_qflags.as<int32_t>(), order, g->ck_qflags.as<int32_t>(), nq, 1))) {
        drain(); return rc;
    }
    const bool scan_hist = hist && g->hist_pack && nq >= 1024;
    if (scan_hist) {
        if ((rc = scan_hist_columns(g, g->d_qhist.as<uint32_t>(), nq, st))) { drain(); return rc; }
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    Readback d2h{st, &r->d2h, cudaGetLastError()};
    d2h(r->q_start, g->ck_qstart.p, q * 8); d2h(r->q_count, g->ck_qcount.p, q * 4); d2h(r->q_maxd, g->ck_qmaxd.p, q * 4); d2h(r->q_flags, g->ck_qflags.p, q * 4);
    if (scan_hist) {
        const HistCols hc = hist_layout(g, r.get());
        if (hc.k) {
            const size_t pbytes = q * hc.k * r->hist_width;
            if (!r->q_hist_packed.alloc(pbytes)) { drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed"); }
            if ((rc = g->d_hist_packed.ensure(pbytes))) { drain(); return rc; }
            rc = r->hist_width == 2
                     ? LAUNCH(hist_pack_scatter_kernel<uint16_t>, sgrid, 256, 0, st, g->d_qhist.as<uint32_t>(), order, nq, hc, g->d_hist_packed.as<uint16_t>())
                     : LAUNCH(hist_pack_scatter_kernel<uint32_t>, sgrid, 256, 0, st, g->d_qhist.as<uint32_t>(), order, nq, hc, g->d_hist_packed.as<uint32_t>());
            if (rc) { drain(); return rc; }
            d2h(r->q_hist_packed, g->d_hist_packed.p, pbytes);
        }
    } else if (hist) {
        if (!r->q_hist.alloc(q * ABB_N_ENTITY_TYPES * 4)) { drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed"); }
        if ((rc = g->ck_qhist.ensure(q1 * ABB_N_ENTITY_TYPES * 4))) { drain(); return rc; }
        if ((rc = LAUNCH(scatter_rows_kernel<uint32_t>, sgrid, 256, 0, st, g->d_qhist.as<uint32_t>(), order, g->ck_qhist.as<uint32_t>(), nq, ABB_N_ENTITY_TYPES))) {
            drain(); return rc;
        }
        d2h(r->q_hist, g->ck_qhist.p, q * ABB_N_ENTITY_TYPES * 4);
    }
    cudaError_t &e = d2h.err;
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cst);
    if (e != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "chunked walk failed: %s", cudaGetErrorString(e)); }
    g->hist_info_valid = false;
    note_walk_size(g, spec, nq, node_base, true);
    g->chunk_hint = produced; g->chunk_hint_nq = nq;
    g->last_host_chunks = K;
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
    g->last_host_chunks = 1;
    abb_walk_io io{}; unsigned long long totals[3] = {0, 0, 0}; int64_t h2d = 0;
    HostBlock direct;
    if (int rc = walk_device_stage(g, spec, roots, root_off, targets, n_queries, &io, totals, &h2d, &direct)) return rc;
    return walk_collect(g, spec, io, totals, h2d, out, true, &direct);
}

// ------------------------------------------------------------------ exposure-path rows
static int ensure_server_table(abb_graph *g, cudaStream_t st) {
    if (g->srv_table_ready) return ABB_OK;
    const size_t n = static_cast<size_t>(g->v.n) + 1;
    if (int rc = g->srv_cred.ensure(n * 4)) return rc;
    if (int rc = g->srv_tool.ensure(n * 4)) return rc;
    const unsigned grid = grid_for(g->v.n, 256, g->sm_count, 16);
    if (int rc = LAUNCH(server_table_kernel, grid, 256, 0, st, g->v, g->srv_cred.as<int32_t>(), g->srv_tool.as<int32_t>())) return rc;
    // principal rows of every server (paths.cuh server_rows_kernel): count, scan in place, fill
    if (int rc = g->srv_roff.ensure(n * 8)) return rc;
    int64_t *roff = g->srv_roff.as<int64_t>();
    CUDA_TRY(cudaMemsetAsync(roff, 0, n * 8, st));
    if (int rc = LAUNCH(server_rows_kernel<false>, grid, 256, 0, st, g->v, g->srv_cred.as<int32_t>(), g->srv_tool.as<int32_t>(), roff, nullptr, nullptr))
        return rc;
    if (int rc = scan_i64(g->p_scan_tmp, roff, roff, static_cast<int64_t>(n), st)) return rc;
    int64_t total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, roff + g->v.n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (int rc = g->srv_row.ensure(static_cast<size_t>(total + 1) * 16)) return rc;
    if (int rc = g->srv_rel.ensure(static_cast<size_t>(total) + 16)) return rc;
    if (int rc = LAUNCH(server_rows_kernel<true>, grid, 256, 0, st, g->v, g->srv_cred.as<int32_t>(), g->srv_tool.as<int32_t>(), roff, g->srv_row.as<int4>(),
                        g->srv_rel.as<int8_t>()))
        return rc;
    CUDA_TRY(cudaStreamSynchronize(st));   // one-time: later launches may come on other streams
    g->srv_table_ready = true;
    return ABB_OK;
}

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

// the graph's parts of the exposure-path arguments: server table and exposure tables
static PathsArgs paths_base(abb_graph *g) {
    PathsArgs A{};
    A.g = g->v; A.srv_cred = g->srv_cred.as<int32_t>(); A.srv_tool = g->srv_tool.as<int32_t>();
    A.srv_roff = g->srv_roff.as<int64_t>(); A.srv_row = g->srv_row.as<int4>(); A.srv_rel = g->srv_rel.as<int8_t>();
    A.x_vs = g->x_vs.as<uint8_t>(); A.x_loff = g->x_loff.as<int64_t>(); A.x_link = g->x_link.as<LinkRec>(); A.x_rows = g->x_rows.as<int32_t>();
    A.x_toff = g->x_toff.as<int64_t>(); A.t_row = g->x_trow.as<int4>(); A.t_rel = g->x_trel.as<int8_t>(); A.x_overflow = g->x_overflow.as<unsigned>();
    return A;
}

// Graph-constant exposure tables (paths.cuh): the links of every finding node, the template of every vulnerable source and the
// rows of every finding node, built once per graph (count -> scan in place -> fill) and freed with it.  Synchronises the stream
// to size the link and template arrays, and once more at the end: later calls may come on other streams.
static int ensure_exposure_tables(abb_graph *g, cudaStream_t st) {
    if (g->x_tables_ready) return ABB_OK;
    NvtxRange nvtx_("paths: graph-constant exposure tables");
    if (int rc = ensure_server_table(g, st)) return rc;
    const int64_t n = g->v.n;
    const size_t n1 = static_cast<size_t>(n) + 1;
    int rc = ABB_OK;
    if (!rc) rc = g->x_vs.alloc(n1);
    if (!rc) rc = g->x_loff.alloc(n1 * 8);
    if (!rc) rc = g->x_toff.alloc(n1 * 8);
    if (!rc) rc = g->x_rows.alloc(n1 * 4);
    if (!rc) rc = g->x_overflow.alloc(4);
    if (rc) return rc;
    PathsArgs A = paths_base(g);
    CUDA_TRY(cudaMemsetAsync(A.x_vs, 0, n1, st));
    CUDA_TRY(cudaMemsetAsync(A.x_loff, 0, n1 * 8, st));
    CUDA_TRY(cudaMemsetAsync(A.x_toff, 0, n1 * 8, st));
    CUDA_TRY(cudaMemsetAsync(A.x_overflow, 0, 4, st));
    const unsigned grid = warp_grid(g, (n + 31) / 32);
    if ((rc = LAUNCH(node_links_kernel<false>, grid, 256, 0, st, A))) return rc;
    if ((rc = scan_i64(g->p_scan_tmp, A.x_loff, A.x_loff, n + 1, st))) return rc;
    if ((rc = LAUNCH(template_kernel<false>, grid, 256, 0, st, A))) return rc;
    if ((rc = scan_i64(g->p_scan_tmp, A.x_toff, A.x_toff, n + 1, st))) return rc;
    int64_t NL = 0, TR = 0;
    CUDA_TRY(cudaMemcpyAsync(&NL, A.x_loff + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&TR, A.x_toff + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    // link records hold link and template offsets as int32
    if (NL >= (1ll << 31) - 1 || TR >= (1ll << 31) - 1) return fail(ABB_ERR_CAPACITY, "exposure tables: %lld links, %lld template rows (int32 offsets)", (long long)NL, (long long)TR);
    if (!rc) rc = g->x_link.alloc(static_cast<size_t>(NL) * 16);
    if (!rc) rc = g->x_trow.alloc(static_cast<size_t>(TR) * 16);
    if (!rc) rc = g->x_trel.alloc(static_cast<size_t>(TR) * 2);
    if (rc) return rc;
    A = paths_base(g);
    if ((rc = LAUNCH(template_kernel<true>, grid, 256, 0, st, A)) || (rc = LAUNCH(node_links_kernel<true>, grid, 256, 0, st, A))) return rc;
    unsigned overflow = 0;
    CUDA_TRY(cudaMemcpyAsync(&overflow, A.x_overflow, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (overflow) return fail(ABB_ERR_CAPACITY, "exposure tables: a finding has 2^31 or more exposure-path rows");
    g->x_tables_ready = true;
    return ABB_OK;
}

// Count pass of the exposure-path pipeline (paths.cuh): each finding's row count and links gathered from the exposure tables, then
// one exclusive scan into io.f_off.  Once the tables exist this neither synchronises nor, for a batch no larger than an earlier
// one, allocates.  `link_counts` also writes each finding's link count (pl_lcnt) for the host result.
static int enqueue_paths_count(abb_graph *g, const abb_paths_io *io, cudaStream_t st, bool link_counts = false) {
    NvtxRange nvtx_("paths: rows per finding");
    if (!io || io->n_findings < 0 || !io->f_off || (io->n_findings && !io->findings)) return fail(ABB_ERR_ARG, "bad paths io");
    if (io->n_findings >= (1ll << 31) - 2) return fail(ABB_ERR_ARG, "too many findings in one batch");
    if (int rc = ensure_exposure_tables(g, st)) return rc;
    g->paths_args_valid = false;
    const int64_t nf = io->n_findings;
    int rc = g->pl_cnt.ensure(static_cast<size_t>(nf + 1) * 8);
    if (!rc) rc = g->pl_link.ensure(static_cast<size_t>(nf + 1) * 8);
    if (!rc && link_counts) rc = g->pl_lcnt.ensure(static_cast<size_t>(nf + 1) * 8);
    if (rc) return rc;
    PathsArgs A = paths_base(g);
    A.io = *io; A.f_cnt = g->pl_cnt.as<int64_t>(); A.f_link = g->pl_link.as<int2>(); A.f_lcnt = link_counts ? g->pl_lcnt.as<int64_t>() : nullptr;
    if ((rc = LAUNCH(finding_rows_kernel, static_cast<unsigned>((nf + 1 + 255) / 256), 256, 0, st, A))) return rc;
    if ((rc = scan_i64(g->p_scan_tmp, A.f_cnt, io->f_off, nf + 1, st))) return rc;
    g->paths_args = A;
    g->paths_args_valid = true;
    return ABB_OK;
}

static int enqueue_paths_fill(abb_graph *g, const abb_paths_io *io, cudaStream_t st) {
    if (!io || !io->f_off || !io->hops || !io->rels || !io->ncred || !io->ntool) return fail(ABB_ERR_ARG, "bad paths io");
    if (!io->n_findings) return ABB_OK;
    if (!g->paths_args_valid || g->paths_args.io.findings != io->findings || g->paths_args.io.n_findings != io->n_findings || g->paths_args.io.f_off != io->f_off)
        return fail(ABB_ERR_ARG, "abb_paths_fill_launch must follow abb_paths_count_launch for the same findings / f_off");
    if ((reinterpret_cast<uintptr_t>(io->hops) & 15) != 0 || (reinterpret_cast<uintptr_t>(io->rels) & 3) != 0) return fail(ABB_ERR_ARG, "io.hops must be 16-byte and io.rels 4-byte aligned");
    PathsArgs A = g->paths_args;
    A.io = *io;
    return LAUNCH(replicate_kernel, row_grid(g, replicate_kernel, g->replicate_grid), ROW_THREADS, 0, st, A);
}

extern "C" int abb_paths_count_launch(abb_graph *g, const abb_paths_io *io, void *stream) {
    NvtxRange nvtx_("abb_paths_count_launch");
    if (!g) return fail(ABB_ERR_ARG, "null graph");
    DeviceGuard dg(g->device);
    std::lock_guard<std::mutex> lk(g->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaEventRecord(g->ev[2], st));
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
    CUDA_TRY(cudaEventRecord(g->ev[3], st));
    g->paths_timed = true;
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
    std::unique_ptr<abb_paths_result> r(new abb_paths_result());
    r->nf = nf;
    if (!r->findings.alloc(static_cast<size_t>(nf + 1) * 4)) return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    if (nf) memcpy(r->findings.p, h_findings, static_cast<size_t>(nf) * 4);
    if (!d_findings) {
        if (int rc = g->p_findings.ensure(static_cast<size_t>(nf + 1) * 4)) return rc;
        if (nf) { CUDA_TRY(cudaMemcpyAsync(g->p_findings.p, h_findings, static_cast<size_t>(nf) * 4, cudaMemcpyHostToDevice, st)); r->h2d += nf * 4; }
        d_findings = g->p_findings.as<int32_t>();
    }
    if (int rc = g->p_off.ensure(static_cast<size_t>(nf + 1) * 8)) return rc;
    abb_paths_io io{};
    io.n_findings = nf; io.findings = d_findings; io.f_off = g->p_off.as<int64_t>();
    CUDA_TRY(cudaEventRecord(g->ev[2], st));
    if (int rc = enqueue_paths_count(g, &io, st, true)) return rc;
    // the batch's share of the exposure tables: its links (link counts scanned into link_off) and the templates of its distinct
    // vulnerable sources, in node order
    const PathsArgs A = g->paths_args;
    const int64_t n = g->v.n;
    int rc = g->pl_off.ensure(static_cast<size_t>(nf + 1) * 8);
    if (rc) return rc;
    int64_t *link_off = g->pl_off.as<int64_t>();
    if ((rc = scan_i64(g->p_scan_tmp, A.f_lcnt, link_off, nf + 1, st))) return rc;
    int64_t NL = 0;
    CUDA_TRY(cudaMemcpyAsync(&NL, link_off + nf, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const int64_t nu_max = std::min<int64_t>(NL, n);
    ENS(pl_vs, (NL + 2) * 4); ENS(pl_rel, NL + 16); ENS(pl_roff, (NL + 2) * 8); ENS(pl_toff, (NL + 2) * 8); ENS(pl_need, n + 16); ENS(pl_ulist, (n + 2) * 4);
    ENS(pl_nu, 16); ENS(pt_cnt, (nu_max + 2) * 8); ENS(pt_off, (nu_max + 2) * 8); ENS(pt_off_node, (n + 2) * 8);
    if (rc) return rc;
    int32_t *link_vs = g->pl_vs.as<int32_t>(), *ulist = g->pl_ulist.as<int32_t>();
    int8_t *link_rel = g->pl_rel.as<int8_t>();
    int64_t *link_roff = g->pl_roff.as<int64_t>(), *link_toff = g->pl_toff.as<int64_t>(), *t_cnt = g->pt_cnt.as<int64_t>(), *t_off = g->pt_off.as<int64_t>();
    uint8_t *need = g->pl_need.as<uint8_t>();
    unsigned long long *nu = g->pl_nu.as<unsigned long long>();
    CUDA_TRY(cudaMemsetAsync(need, 0, static_cast<size_t>(n) + 16, st));
    if ((rc = LAUNCH(batch_links_kernel, static_cast<unsigned>((nf + 1 + 255) / 256), 256, 0, st, A, link_off, link_vs, link_rel, link_roff, need))) return rc;
    if ((rc = select_flagged(g->p_scan_tmp, need, ulist, nu, static_cast<int>(n), st))) return rc;
    CUDA_TRY(cudaMemsetAsync(t_cnt, 0, static_cast<size_t>(nu_max + 2) * 8, st));
    if (nu_max) if ((rc = LAUNCH(batch_template_counts_kernel, static_cast<unsigned>((nu_max + 255) / 256), 256, 0, st, A, ulist, nu, t_cnt))) return rc;
    if ((rc = scan_i64(g->p_scan_tmp, t_cnt, t_off, nu_max + 1, st))) return rc;
    int64_t TR = 0;
    CUDA_TRY(cudaMemcpyAsync(&TR, t_off + nu_max, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ENS(pt_row, (TR + 2) * 16); ENS(pt_rel, (TR + 2) * 2);
    if (rc) return rc;
    int64_t *t_off_node = g->pt_off_node.as<int64_t>();
    if (nu_max)
        if ((rc = LAUNCH(batch_templates_kernel, warp_grid(g, nu_max), 256, 0, st, A, ulist, nu, t_off, t_off_node, g->pt_row.as<int4>(), g->pt_rel.as<int8_t>())))
            return rc;
    if (NL) if ((rc = LAUNCH(batch_link_toff_kernel, static_cast<unsigned>((NL + 255) / 256), 256, 0, st, NL, link_vs, t_off_node, link_toff))) return rc;
    CUDA_TRY(cudaEventRecord(g->ev[3], st));
    g->paths_timed = true;
    const size_t n1 = static_cast<size_t>(nf) + 1;
    r->n_links = NL; r->n_trows = TR;
    bool ok = r->off.alloc(n1 * 8) && r->link_off.alloc(n1 * 8) && r->link_vs.alloc(NL * 4) && r->link_rel.alloc(NL) && r->link_roff.alloc((NL + 1) * 8) &&
              r->link_toff.alloc(NL * 8) && r->t_row.alloc(TR * 16) && r->t_rel.alloc(TR * 2);
    if (!ok) return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    Readback d2h{st, &r->d2h};
    d2h(r->off, io.f_off, n1 * 8); d2h(r->link_off, link_off, n1 * 8); d2h(r->link_vs, link_vs, NL * 4); d2h(r->link_rel, link_rel, NL);
    d2h(r->link_roff, link_roff, (NL + 1) * 8); d2h(r->link_toff, link_toff, NL * 8); d2h(r->t_row, g->pt_row.p, TR * 16); d2h(r->t_rel, g->pt_rel.p, TR * 2);
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
    if (int rc = g->p_findings.ensure(static_cast<size_t>(nf + 1) * 4)) return rc;
    if (int rc = g->p_off.ensure(static_cast<size_t>(nf + 1) * 8)) return rc;
    DevBuf d_base, d_tab, d_ncu, d_ntu, d_focus;
    if (nf) CUDA_TRY(cudaMemcpyAsync(g->p_findings.p, findings, static_cast<size_t>(nf) * 4, cudaMemcpyHostToDevice, st));
    if (int rc = d_base.upload(base_id, static_cast<size_t>(nf) * 4, st, 4)) return rc;
    if (int rc = d_tab.upload(risk_rank, static_cast<size_t>(n_base) * 75 * 4, st)) return rc;
    if (int rc = d_ncu.upload(ncu, static_cast<size_t>(n) * 4, st, 4)) return rc;
    if (int rc = d_ntu.upload(ntu, static_cast<size_t>(n) * 4, st, 4)) return rc;
    if (focused) { if (int rc = d_focus.upload(node_focus, static_cast<size_t>(n), st, 1)) return rc; }
    abb_paths_io io{};
    io.n_findings = nf; io.findings = g->p_findings.as<int32_t>(); io.f_off = g->p_off.as<int64_t>();
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
    PathsArgs A = g->paths_args;
    RankArgs RA{d_base.as<int32_t>(), d_tab.as<uint32_t>(), d_ncu.as<int32_t>(), d_ntu.as<int32_t>(), k1.as<unsigned long long>(), v1.as<uint32_t>(),
                d_focus.as<uint8_t>(), need};
    if ((rc = LAUNCH(rank_keys_kernel, row_grid(g, rank_keys_kernel, g->rank_keys_grid), ROW_THREADS, 0, st, A, RA))) return rc;
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
        g->last_host_chunks = 1;
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
    const int64_t nq = n_findings;
    const size_t q = static_cast<size_t>(nq), q1 = q + 1;
    auto drain = [&]() { cudaStreamSynchronize(st); cudaStreamSynchronize(cs); };
    int rc = ABB_OK;
    ENS(d_roots, q1 * 4); ENS(cx_bcnt, q1 * CTX_BUCKETS * 4); ENS(cx_cnt, q1 * 8); ENS(cx_start, q1 * 8);
    if (rc) return rc;
    std::unique_ptr<abb_finding_context_result> r(new abb_finding_context_result());
    r->nq = nq;
    if (nq) CUDA_TRY(cudaMemcpyAsync(g->d_roots.p, findings, q * 4, cudaMemcpyHostToDevice, st));
    r->h2d = nq * 4;
    CUDA_TRY(cudaEventRecord(g->cx_staged, st));
    CUDA_TRY(cudaStreamWaitEvent(cs, g->cx_staged, 0));
    // count pass + scan, next to the walk
    CtxArgs A{};
    A.g = g->v; A.findings = g->d_roots.as<int32_t>(); A.n = nq;
    A.bcnt = g->cx_bcnt.as<int32_t>(); A.cnt = g->cx_cnt.as<int64_t>(); A.start = g->cx_start.as<int64_t>();
    const unsigned grid = warp_grid(g, (nq + 31) / 32);
    CUDA_TRY(cudaEventRecord(g->cx_ev[0], cs));
    CUDA_TRY(cudaMemsetAsync(A.cnt, 0, q1 * 8, cs));
    if (nq) if ((rc = LAUNCH(context_kernel<false>, grid, 256, 0, cs, A))) { drain(); return rc; }
    if ((rc = scan_i64(g->p_scan_tmp, A.cnt, g->cx_start.as<int64_t>(), nq + 1, cs))) { drain(); return rc; }
    CUDA_TRY(cudaEventRecord(g->cx_ev[1], cs));
    // the impact walk, unchanged, into the device arena
    const abb_walk_spec spec = abb_spec_impact_of(max_depth);
    abb_walk_io io{}; unsigned long long totals[3] = {0, 0, 0}; int64_t wh2d = 0;
    g->last_host_chunks = 1;
    if ((rc = walk_device_stage(g, &spec, findings, nullptr, nullptr, nq, &io, totals, &wh2d, nullptr, true))) { drain(); return rc; }
    int64_t total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, g->cx_start.as<int64_t>() + nq, 8, cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(cudaStreamSynchronize(cs));
    r->total = total;
    ENS(cx_src, (total + 1) * 4);
    if (rc) { drain(); return rc; }
    if (!(r->start.alloc(q * 8) && r->bcnt.alloc(q * CTX_BUCKETS * 4) && r->src.alloc(static_cast<size_t>(total) * 4))) {
        drain(); return fail(ABB_ERR_NOMEM, "pinned host allocation failed");
    }
    // fill pass and its copies on paths_stream, the walk's per-finding arrays on the main stream
    A.src = g->cx_src.as<int32_t>();
    CUDA_TRY(cudaEventRecord(g->cx_ev[2], cs));
    if (nq) if ((rc = LAUNCH(context_kernel<true>, grid, 256, 0, cs, A))) { drain(); return rc; }
    CUDA_TRY(cudaEventRecord(g->cx_ev[3], cs));
    Readback d2h{cs, &r->d2h, cudaGetLastError()};
    d2h(r->start, g->cx_start.p, q * 8); d2h(r->bcnt, g->cx_bcnt.p, q * CTX_BUCKETS * 4); d2h(r->src, g->cx_src.p, static_cast<size_t>(total) * 4);
    cudaError_t e = d2h.err;
    if (e != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "finding context failed: %s", cudaGetErrorString(e)); }
    abb_walk_result *walk = nullptr;
    if ((rc = walk_collect(g, &spec, io, totals, wh2d, &walk, true, nullptr, false))) { drain(); return rc; }
    r->walk.reset(walk);
    if ((e = cudaStreamSynchronize(cs)) != cudaSuccess) { drain(); return fail(ABB_ERR_CUDA, "finding context failed: %s", cudaGetErrorString(e)); }
    r->d2h += r->walk->d2h;
    float a = 0.f, b = 0.f;
    if (cudaEventElapsedTime(&a, g->ev[0], g->ev[1]) == cudaSuccess) r->walk_ms = a;
    if (cudaEventElapsedTime(&a, g->cx_ev[0], g->cx_ev[1]) == cudaSuccess && cudaEventElapsedTime(&b, g->cx_ev[2], g->cx_ev[3]) == cudaSuccess) r->context_ms = a + b;
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

// Runs with the graph's device current (abb_graph_free); the DevBuf members and the snapshot tables free themselves after it.
abb_graph::~abb_graph() {
    for (cudaStream_t s : {stream, copy_stream, paths_stream}) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (cudaEvent_t e : {ev_copy, ev_chunk_walked, ev_chunk_copied[0], ev_chunk_copied[1], ev[0], ev[1], ev[2], ev[3], cx_staged, cx_ev[0], cx_ev[1], cx_ev[2], cx_ev[3]})
        if (e) cudaEventDestroy(e);
}
