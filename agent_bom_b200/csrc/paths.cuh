// paths.cuh — per-finding typed exposure-path pattern walk (sm_90a).
//
// Device restatement of the topology part of the reference's
// _derived_attack_paths (api/routes/graph.py:686-760) and
// _edge_relationships_for_hops (:488-503):
//
//   finding f  <-VULNERABLE_TO- vs            (in-edges of f, graph.edges order, originals only)
//   servers = [vs] if vs is a SERVER else
//             [s for s -DEPENDS_ON-> vs if s is a SERVER]
//   per server: agents = sorted(set(a for a -USES-> server if a is agent/user/service_account)) or [server]
//               ncred / ntool = # EXPOSES_CRED / PROVIDES_TOOL out-edges whose target has a node record
//   row (agent, server, vs, f) + first relationship per hop pair.
//
// The rows are factorised: a finding's LINKS (one per vulnerable source vs) and,
// per distinct vs, a TEMPLATE (its (agent, server) rows), which every finding
// attached to vs shares.  The principals of a server depend only on the graph, so
// they sit in a graph-constant server row table built once per graph
// (server_rows_kernel); a template is the concatenation of its servers' table
// rows.  Links and templates depend only on the graph too: they are built once per
// graph for every finding node and every vulnerable source (ensure_exposure_tables)
// with one thread per node in two passes (count, then fill at the scanned offsets)
// so rows land in the reference's emission order; reverse rows longer than LONG_ROW
// are handed to the whole warp.  A call then only gathers each finding's row count
// and scans it (finding_rows_kernel), and writes the flat rows row-parallel
// (for_each_row).  "Originals only" = entries without ABB_META_REVERSED_COPY: the
// reference builds its incoming/outgoing maps from graph.edges, which never holds
// the reversed copies of bidirectional edges (:698-702).
//
// Pair relationships: by_pair.setdefault((a,b)) keeps the first edge between a
// and b.  Entries of adjacency[a] with neighbour b and entries of
// reverse_adjacency[b] with neighbour a correspond one-to-one in order, so the
// answer is the relationship of the first reverse-row entry of b whose
// neighbour is a — and every pair the pattern needs is reached THROUGH such an
// entry, whose ABB_META_FIRST_PAIR bit says whether it is that first one.
#pragma once
#include "walk.cuh"

namespace abb {

constexpr int REL_USES = 1, REL_DEPENDS_ON = 2, REL_PROVIDES_TOOL = 3, REL_EXPOSES_CRED = 4, REL_VULNERABLE_TO = 9;
constexpr int ET_AGENT = 0, ET_SERVER = 1, ET_VULN = 8, ET_MISCONF = 9, ET_USER = 13, ET_SERVICE_ACCOUNT = 17;
constexpr uint32_t LONG_ROW = 64;   // reverse rows longer than this are handled by the whole warp

// A link of a finding node: x = vulnerable source, y = relationship of the pair (vs, finding), z = the link's first row within the
// node's rows, w = first row of vs's template in t_row.
using LinkRec = int4;

struct PathsArgs {
    GraphView g;
    abb_paths_io io;
    const int32_t *srv_cred;    // [n_nodes] EXPOSES_CRED fan-out of server nodes (graph-constant table)
    const int32_t *srv_tool;    // [n_nodes] PROVIDES_TOOL fan-out
    // graph-constant server row table: the principal rows every server contributes to a template
    const int64_t *srv_roff;    // [n_nodes+1] first table row of each node (only servers own rows, at least one each)
    const int4 *srv_row;        // [n_server_rows] agent, server, ncred, ntool
    const int8_t *srv_rel;      // [n_server_rows] relationship of the pair (agent, server)
    // graph-constant exposure tables (ensure_exposure_tables): every finding node's links, every vulnerable source's template
    uint8_t *x_vs;              // [n_nodes] 1 on a vulnerable source (a non-ghost source of an original VULNERABLE_TO entry into a finding)
    int64_t *x_loff;            // [n_nodes+1] links of node u are x_link[x_loff[u] .. x_loff[u+1]) (counts, then scanned in place)
    LinkRec *x_link;            // [n_links] in reverse-row order
    int32_t *x_rows;            // [n_nodes] rows of node u (the sum of its links' template lengths; 0 for non-findings)
    int64_t *x_toff;            // [n_nodes+1] template of node u is t_row[x_toff[u] .. x_toff[u+1]) (counts, then scanned in place)
    int4 *t_row;                // [n_template_rows] agent, server, ncred, ntool
    int8_t *t_rel;              // [n_template_rows*2] (agent,server) and (server,vs) relationships
    unsigned *x_overflow;       // set when a node's rows do not fit the link record's int32
    // per call
    int64_t *f_cnt;             // [n_findings+1] rows of each finding, scanned into io.f_off
    int2 *f_link;               // [n_findings] first link and link count of each finding
    int64_t *f_lcnt;            // [n_findings+1] link counts (host-result path only, else nullptr)
};

// graph-constant table: credential / tool fan-out of every server (originals only, target must have a node record)
__global__ void server_table_kernel(GraphView g, int32_t *srv_cred, int32_t *srv_tool) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < g.n; base += nwarps * 32) {
        const int64_t u = base + lane;
        int nc = 0, nt = 0;
        if (u < g.n && __ldg(g.ntype + u) == ET_SERVER) {
            for (uint32_t p = __ldg(g.foff + u); p < __ldg(g.foff + u + 1); p++) {
                const uint32_t m = __ldg(g.fmeta + p);
                if (m & ABB_META_REVERSED_COPY) continue;
                const int rel = m & ABB_META_REL_MASK;
                if (rel != REL_EXPOSES_CRED && rel != REL_PROVIDES_TOOL) continue;
                if (__ldg(g.ntype + __ldg(g.fnbr + p)) == ABB_NODE_GHOST) continue;
                if (rel == REL_EXPOSES_CRED) nc++; else nt++;
            }
        }
        if (u < g.n) { srv_cred[u] = nc; srv_tool[u] = nt; }
    }
}

__device__ __forceinline__ bool is_principal(uint8_t t) { return t == ET_AGENT || t == ET_USER || t == ET_SERVICE_ACCOUNT; }

// relationship of the first reverse-row entry of b whose neighbour is a (lane-serial), -1 if none
__device__ __forceinline__ int first_rel_rev(const GraphView &g, int32_t a, int32_t b) {
    for (uint32_t p = __ldg(g.roff + b), e = __ldg(g.roff + b + 1); p < e; p++)
        if (__ldg(g.rnbr + p) == a) return __ldg(g.rmeta + p) & ABB_META_REL_MASK;
    return -1;
}

// next agent of server s in ascending id-string rank above `last` (lane-serial over the reverse row); false when exhausted
__device__ __forceinline__ bool next_agent_serial(const GraphView &g, int32_t s, int32_t &last, int32_t &agent, int &rel_as) {
    int32_t best = 0x7FFFFFFF; uint32_t bm = 0;
    for (uint32_t p = __ldg(g.roff + s), e = __ldg(g.roff + s + 1); p < e; p++) {
        const uint32_t m = __ldg(g.rmeta + p);
        if ((m & ABB_META_REVERSED_COPY) || (m & ABB_META_REL_MASK) != REL_USES) continue;
        const int32_t a = __ldg(g.rnbr + p);
        if (!is_principal(__ldg(g.ntype + a))) continue;
        const int32_t r = __ldg(g.rank + a);
        if (r > last && r < best) { best = r; agent = a; bm = m; }
    }
    if (best == 0x7FFFFFFF) return false;
    last = best;
    rel_as = (bm & ABB_META_FIRST_PAIR) ? REL_USES : first_rel_rev(g, agent, s);
    return true;
}

// same, whole warp over a long reverse row
__device__ __forceinline__ bool next_agent_warp(const GraphView &g, int32_t s, int32_t &last, int32_t &agent, int &rel_as, int lane) {
    int32_t best = 0x7FFFFFFF, bn = -1; uint32_t bm = 0;
    for (uint32_t p = __ldg(g.roff + s), e = __ldg(g.roff + s + 1); p < e; p += 32) {
        const uint32_t k = p + lane;
        if (k >= e) continue;
        const uint32_t m = __ldg(g.rmeta + k);
        if ((m & ABB_META_REVERSED_COPY) || (m & ABB_META_REL_MASK) != REL_USES) continue;
        const int32_t a = __ldg(g.rnbr + k);
        if (!is_principal(__ldg(g.ntype + a))) continue;
        const int32_t r = __ldg(g.rank + a);
        if (r > last && r < best) { best = r; bn = a; bm = m; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int32_t ob = __shfl_xor_sync(FULL, best, o), on = __shfl_xor_sync(FULL, bn, o);
        const uint32_t om = __shfl_xor_sync(FULL, bm, o);
        if (ob < best) { best = ob; bn = on; bm = om; }
    }
    if (bn < 0) return false;
    last = best; agent = bn;
    rel_as = (bm & ABB_META_FIRST_PAIR) ? REL_USES : first_rel_rev(g, agent, s);
    return true;
}

// ---- graph-constant server row table: for every server, its principals in ascending id-string rank with the relationship of
// the pair (agent, server), or the server itself (with the relationship of the pair (server, server)) when no principal uses it
// (:737-738).  Lane u owns node u; a server with a long reverse row is handed to the whole warp.  COUNT writes each server's
// row count to srv_roff[u] (scanned in place afterwards), FILL writes the rows from srv_roff[u].
template <bool FILL>
__global__ void __launch_bounds__(256) server_rows_kernel(const GraphView g, const int32_t *srv_cred, const int32_t *srv_tool, int64_t *srv_roff, int4 *srv_row,
                                                          int8_t *srv_rel) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    auto put = [&](int64_t k, int32_t a, int32_t s, int rel) {
        srv_row[k] = make_int4(a, s, __ldg(srv_cred + s), __ldg(srv_tool + s));
        srv_rel[k] = static_cast<int8_t>(rel);
    };
    for (int64_t base = warp * 32; base < g.n; base += nwarps * 32) {
        const int64_t u = base + lane;
        const int32_t s = (u < g.n && __ldg(g.ntype + u) == ET_SERVER) ? static_cast<int32_t>(u) : -1;
        const bool is_long = s >= 0 && __ldg(g.roff + s + 1) - __ldg(g.roff + s) > LONG_ROW;
        const int64_t row0 = (FILL && s >= 0) ? srv_roff[s] : 0;
        if (s >= 0 && !is_long) {
            int32_t last = -1, a; int r; int k = 0;
            while (next_agent_serial(g, s, last, a, r)) { if (FILL) put(row0 + k, a, s, r); k++; }
            if (k == 0) { if (FILL) put(row0, s, s, first_rel_rev(g, s, s)); k = 1; }
            if (!FILL) srv_roff[s] = k;
        }
        for (unsigned rem = __ballot_sync(FULL, is_long); rem; rem &= rem - 1) {
            const int src = __ffs(rem) - 1;
            const int32_t ls = __shfl_sync(FULL, s, src);
            const int64_t l0 = __shfl_sync(FULL, row0, src);
            int32_t last = -1, a; int r; int k = 0;
            while (next_agent_warp(g, ls, last, a, r, lane)) { if (FILL && lane == 0) put(l0 + k, a, ls, r); k++; }
            if (k == 0) { if (FILL && lane == 0) put(l0, ls, ls, first_rel_rev(g, ls, ls)); k = 1; }
            if (!FILL && lane == 0) srv_roff[ls] = k;
        }
    }
}

// ---- exposure tables, links: every finding node's links (VULNERABLE_TO originals whose source has a node record), in row order.
// The source behind reverse-row entry k of a finding, or -1; rvf = relationship of the pair (vs, finding), -3 = not the first
// entry of the pair (looked up in the fill pass).
__device__ __forceinline__ int32_t link_source(const GraphView &g, uint32_t k, int &rvf) {
    const uint32_t m = __ldg(g.rmeta + k);
    if ((m & ABB_META_REVERSED_COPY) || (m & ABB_META_REL_MASK) != REL_VULNERABLE_TO) return -1;
    const int32_t v = __ldg(g.rnbr + k);
    if (__ldg(g.ntype + v) == ABB_NODE_GHOST) return -1;
    rvf = (m & ABB_META_FIRST_PAIR) ? REL_VULNERABLE_TO : -3;
    return v;
}

__device__ __forceinline__ int64_t template_rows(const PathsArgs &A, int32_t vs) { return A.x_toff[vs + 1] - A.x_toff[vs]; }

// link record o of finding f: vs's template starts at x_toff[vs], the link's rows at `roff` within f's rows
__device__ __forceinline__ void put_link(const PathsArgs &A, int64_t o, int32_t vs, int32_t f, int rvf, int64_t roff) {
    if (rvf == -3) rvf = first_rel_rev(A.g, vs, f);
    A.x_link[o] = make_int4(vs, rvf, static_cast<int32_t>(roff), static_cast<int32_t>(A.x_toff[vs]));
}

// Lane u owns node u; a finding with a long reverse row is handed to the whole warp.  COUNT writes the node's link count to
// x_loff[u] (scanned in place afterwards) and flags its vulnerable sources in x_vs; FILL runs after the templates exist and writes
// the link records from x_loff[u] and the node's row count.
template <bool FILL>
__global__ void __launch_bounds__(256) node_links_kernel(const PathsArgs A) {
    const GraphView &g = A.g;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < g.n; base += nwarps * 32) {
        const int32_t u = static_cast<int32_t>(base + lane);
        uint32_t s0 = 0, e0 = 0;
        if (u < g.n) {
            const uint8_t t = __ldg(g.ntype + u);
            if (t == ET_VULN || t == ET_MISCONF) { s0 = __ldg(g.roff + u); e0 = __ldg(g.roff + u + 1); }
        }
        const bool is_long = e0 - s0 > LONG_ROW;
        const int64_t o0 = (FILL && u < g.n) ? A.x_loff[u] : 0;
        int64_t n = 0, rows = 0;
        if (!is_long) {
            for (uint32_t p = s0; p < e0; p++) {
                int rvf;
                const int32_t vs = link_source(g, p, rvf);
                if (vs < 0) continue;
                if (FILL) { put_link(A, o0 + n, vs, u, rvf, rows); rows += template_rows(A, vs); }
                else A.x_vs[vs] = 1;
                n++;
            }
        }
        for (unsigned rem = __ballot_sync(FULL, is_long); rem; rem &= rem - 1) {
            const int src = __ffs(rem) - 1;
            const int32_t lu = __shfl_sync(FULL, u, src);
            const uint32_t ls0 = __shfl_sync(FULL, s0, src), le0 = __shfl_sync(FULL, e0, src);
            const int64_t lo0 = __shfl_sync(FULL, o0, src);
            int64_t ln = 0, lrows = 0;
            for (uint32_t p = ls0; p < le0; p += 32) {
                const uint32_t k = p + lane;
                int rvf = -1;
                const int32_t vs = k < le0 ? link_source(g, k, rvf) : -1;
                const unsigned vm = __ballot_sync(FULL, vs >= 0);
                if (FILL) {
                    const int64_t c = vs >= 0 ? template_rows(A, vs) : 0;
                    int64_t inc = c;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) { const int64_t v = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += v; }
                    if (vs >= 0) put_link(A, lo0 + ln + __popc(vm & lanemask_lt(lane)), vs, lu, rvf, lrows + inc - c);
                    lrows += __shfl_sync(FULL, inc, 31);
                } else if (vs >= 0) {
                    A.x_vs[vs] = 1;
                }
                ln += __popc(vm);
            }
            if (lane == src) { n = ln; rows = lrows; }
        }
        if (u < g.n) {
            if (!FILL) A.x_loff[u] = n;
            else {
                if (rows > 0x7FFFFFFF) atomicOr(A.x_overflow, 1u);
                A.x_rows[u] = static_cast<int32_t>(rows);
            }
        }
    }
}

// ---- exposure tables, templates: the rows of every vulnerable source (count, then fill): the server table's rows of vs itself
// when it is a server, else of every server that DEPENDS_ON it, in reverse-row order.
// The server behind reverse-row entry k of a non-server vulnerable source, or -1; rsv as rvf above.
__device__ __forceinline__ int32_t dependent_server(const GraphView &g, uint32_t k, int &rsv) {
    const uint32_t m = __ldg(g.rmeta + k);
    if ((m & ABB_META_REVERSED_COPY) || (m & ABB_META_REL_MASK) != REL_DEPENDS_ON) return -1;
    const int32_t v = __ldg(g.rnbr + k);
    if (__ldg(g.ntype + v) != ET_SERVER) return -1;
    rsv = (m & ABB_META_FIRST_PAIR) ? REL_DEPENDS_ON : -3;
    return v;
}

__device__ __forceinline__ int64_t server_rows(const PathsArgs &A, int32_t s) { return __ldg(A.srv_roff + s + 1) - __ldg(A.srv_roff + s); }

// server s's table rows into the template from `row`; the template's relationships are the pairs (agent, server), (server, vs)
__device__ __forceinline__ void copy_server_rows(const PathsArgs &A, int64_t row, int32_t s, int32_t vs, int rsv) {
    if (rsv == -3) rsv = first_rel_rev(A.g, s, vs);
    for (int64_t k = __ldg(A.srv_roff + s), e = __ldg(A.srv_roff + s + 1); k < e; k++, row++) {
        A.t_row[row] = __ldg(A.srv_row + k);
        reinterpret_cast<uint16_t *>(A.t_rel)[row] = static_cast<uint16_t>(static_cast<uint8_t>(__ldg(A.srv_rel + k)) | ((rsv & 0xFF) << 8));
    }
}

// Lane u owns node u when it is a vulnerable source; one with a long reverse row is handed to the whole warp.  COUNT writes the
// template length to x_toff[u] (0 for other nodes; scanned in place afterwards), FILL writes the rows from x_toff[u].
template <bool FILL>
__global__ void __launch_bounds__(256) template_kernel(const PathsArgs A) {
    const GraphView &g = A.g;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < g.n; base += nwarps * 32) {
        const int64_t u = base + lane;
        int32_t vs = -1; uint32_t s2 = 0, e2 = 0; bool is_long = false;
        int64_t row = 0, n = 0;
        if (u < g.n && A.x_vs[u]) {
            vs = static_cast<int32_t>(u);
            if (FILL) row = A.x_toff[vs];
            if (__ldg(g.ntype + vs) == ET_SERVER) {
                n = server_rows(A, vs);
                if (FILL) copy_server_rows(A, row, vs, vs, -2);
            } else {
                s2 = __ldg(g.roff + vs); e2 = __ldg(g.roff + vs + 1);
                is_long = e2 - s2 > LONG_ROW;
                if (!is_long) {
                    for (uint32_t p = s2; p < e2; p++) {
                        int rsv;
                        const int32_t s = dependent_server(g, p, rsv);
                        if (s < 0) continue;
                        if (FILL) copy_server_rows(A, row + n, s, vs, rsv);
                        n += server_rows(A, s);
                    }
                }
            }
        }
        for (unsigned rem = __ballot_sync(FULL, is_long); rem; rem &= rem - 1) {
            const int src = __ffs(rem) - 1;
            const int32_t lvs = __shfl_sync(FULL, vs, src);
            const uint32_t ls2 = __shfl_sync(FULL, s2, src), le2 = __shfl_sync(FULL, e2, src);
            const int64_t lrow = __shfl_sync(FULL, row, src);
            int64_t ln = 0;
            for (uint32_t p = ls2; p < le2; p += 32) {
                const uint32_t k = p + lane;
                int rsv = -1;
                const int32_t s = k < le2 ? dependent_server(g, k, rsv) : -1;
                const int64_t c = s >= 0 ? server_rows(A, s) : 0;
                int64_t inc = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int64_t v = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += v; }
                if (FILL && s >= 0) copy_server_rows(A, lrow + ln + inc - c, s, lvs, rsv);
                ln += __shfl_sync(FULL, inc, 31);
            }
            if (lane == src) n = ln;
        }
        if (!FILL && u < g.n) A.x_toff[u] = n;
    }
}

// ---- per call: each finding's rows and links from the tables.  Ids that are out of range or not findings have none; thread
// n_findings writes the 0 that the exclusive scan turns into the total.
__global__ void finding_rows_kernel(const PathsArgs A) {
    const int64_t fi = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x, nf = A.io.n_findings;
    if (fi > nf) return;
    int64_t rows = 0;
    int2 fl = make_int2(0, 0);
    if (fi < nf) {
        const int32_t f = __ldg(A.io.findings + fi);
        if (f >= 0 && f < A.g.n) {
            const int64_t l0 = __ldg(A.x_loff + f);
            fl = make_int2(static_cast<int32_t>(l0), static_cast<int32_t>(__ldg(A.x_loff + f + 1) - l0));
            rows = __ldg(A.x_rows + f);
        }
        A.f_link[fi] = fl;
    }
    A.f_cnt[fi] = rows;
    if (A.f_lcnt) A.f_lcnt[fi] = fl.y;
}

// ---- host result (abb_paths_host / abb_exposure_host): the batch's links with their flat rows, and its vulnerable sources flagged
__global__ void batch_links_kernel(const PathsArgs A, const int64_t *link_off, int32_t *link_vs, int8_t *link_rel, int64_t *link_roff, uint8_t *need) {
    const int64_t fi = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x, nf = A.io.n_findings;
    if (fi == nf) link_roff[link_off[nf]] = A.io.f_off[nf];
    if (fi >= nf) return;
    const int2 fl = A.f_link[fi];
    const int64_t o0 = link_off[fi], r0 = A.io.f_off[fi];
    for (int k = 0; k < fl.y; k++) {
        const LinkRec l = __ldg(A.x_link + fl.x + k);
        link_vs[o0 + k] = l.x; link_rel[o0 + k] = static_cast<int8_t>(l.y); link_roff[o0 + k] = r0 + l.z;
        need[l.x] = 1;
    }
}

// template lengths of the batch's distinct vulnerable sources (ulist, node order)
__global__ void batch_template_counts_kernel(const PathsArgs A, const int32_t *ulist, const unsigned long long *n_unique, int64_t *t_cnt) {
    const int64_t ui = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (ui < static_cast<int64_t>(*n_unique)) t_cnt[ui] = template_rows(A, ulist[ui]);
}

// one warp per distinct vulnerable source: its template rows to the batch's offset t_off[ui]
__global__ void batch_templates_kernel(const PathsArgs A, const int32_t *ulist, const unsigned long long *n_unique, const int64_t *t_off,
                                       int64_t *t_off_node, int4 *t_row, int8_t *t_rel) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int64_t nu = static_cast<int64_t>(*n_unique);
    for (int64_t ui = warp; ui < nu; ui += nwarps) {
        const int32_t vs = ulist[ui];
        const int64_t s = A.x_toff[vs], e = A.x_toff[vs + 1], o = t_off[ui];
        for (int64_t k = lane; k < e - s; k += 32) {
            t_row[o + k] = A.t_row[s + k];
            reinterpret_cast<uint16_t *>(t_rel)[o + k] = reinterpret_cast<const uint16_t *>(A.t_rel)[s + k];
        }
        if (lane == 0) t_off_node[vs] = o;
    }
}

__global__ void batch_link_toff_kernel(int64_t n_links, const int32_t *link_vs, const int64_t *t_off_node, int64_t *link_toff) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n_links) link_toff[i] = t_off_node[link_vs[i]];
}

// ---- replicate: every finding copies its links' templates, substituting the finding.
// Row-parallel: the flat rows [0, R) are cut into tiles of ROW_TILE, and a block takes a contiguous run of tiles.  Warp w of the
// block takes ROW_ITEMS * 32 consecutive rows of a tile, 32 at a time, so each output stream is written in whole coalesced lines.
// The findings of a tile are found in the block's shared copy of the io.f_off window that starts at the tile's first finding
// (ROW_WIN findings, stored relative to the tile's first row).  A warp carries its current finding from step to step: a lane
// searches only when its row lies past that finding's end, which in long findings (most rows) is one shared-memory compare.  A
// tile that spans more findings than the window holds (a run of zero-row findings) searches the rest in global memory.  Each lane
// keeps its last row's finding, first link and template, so a row of the same finding with one link (most of them) loads nothing
// but its template row; a finding with several links searches their first rows.
// The tile size and 6 resident blocks per SM for replicate_kernel are what measured fastest at L on the H100: a block's two
// barriers and window load per tile are exposed latency, which larger tiles and more resident warps hide (unrolling steps to
// keep more loads in flight per warp cost registers, hence occupancy, and did not help).
constexpr int ROW_THREADS = 256, ROW_ITEMS = 32, ROW_TILE = ROW_THREADS * ROW_ITEMS, ROW_WIN = 1024;

// last l in [lo, hi) with roff[l] <= r, given roff[lo] <= r
template <class T, class I>
__device__ __forceinline__ I last_le(const T *roff, I lo, I hi, T r) {
    while (hi - lo > 1) { const I mid = (lo + hi) >> 1; if (roff[mid] <= r) lo = mid; else hi = mid; }
    return lo;
}

// the link holding row q of a finding whose links are x_link[fl.x .. fl.x + fl.y), fl.y >= 1
__device__ __forceinline__ LinkRec link_of_row(const PathsArgs &A, int2 fl, int32_t q) {
    int32_t lo = fl.x, hi = fl.x + fl.y;
    const int32_t *first_row = reinterpret_cast<const int32_t *>(A.x_link) + 2;   // .z of record k at 4 * k
    while (hi - lo > 1) { const int32_t mid = (lo + hi) >> 1; if (__ldg(first_row + 4 * static_cast<int64_t>(mid)) <= q) lo = mid; else hi = mid; }
    return __ldg(A.x_link + lo);
}

// what locates one flat row: its template row, vulnerable source, finding node, (vs, finding) relationship and finding index
struct RowRef {
    int64_t t;
    int32_t vs, f, rel;
    int64_t fi;
};

// Visits every flat row once as fn(row, RowRef).  Every thread of the block must call it (ROW_THREADS per block).
template <class Fn>
__device__ __forceinline__ void for_each_row(const PathsArgs &A, const Fn &fn) {
    __shared__ int32_t s_roff[ROW_WIN + 1];   // f_off[l0 + i] - r0, clamped to [-1, ROW_TILE + 1]: exact for every comparison with a row of the tile
    __shared__ int64_t s_l0;
    const int lane = threadIdx.x & 31, w0 = (threadIdx.x >> 5) * ROW_ITEMS * 32;
    const int64_t *foff = A.io.f_off;
    const int64_t NF = A.io.n_findings, R = foff[NF];
    const int64_t ntiles = (R + ROW_TILE - 1) / ROW_TILE, per = (ntiles + gridDim.x - 1) / gridDim.x;
    const int64_t tb = blockIdx.x * per, te = min(ntiles, tb + per);
    if (tb >= te) return;
    if (threadIdx.x == 0) s_l0 = last_le(foff, int64_t{0}, NF, tb * ROW_TILE);
    // this lane's last finding: index, node, whether it has several links, else its link's source, relationship and the template
    // row of flat row 0 (a row's template row is ct0 + row)
    int64_t ct0 = 0;
    int32_t cfi = -1, cf = 0, cvs = 0, crel = 0;
    bool cmulti = false;
    for (int64_t tile = tb; tile < te; tile++) {
        __syncthreads();
        const int64_t l0 = s_l0, r0 = tile * ROW_TILE;
        const int n = static_cast<int>(min(static_cast<int64_t>(ROW_TILE), R - r0));   // rows of this tile
        const int nw = static_cast<int>(min(static_cast<int64_t>(ROW_WIN), NF - l0));  // window: findings l0 .. l0+nw-1, bounds s_roff[0..nw]
        for (int i = threadIdx.x; i <= nw; i += ROW_THREADS) {
            const int64_t d = foff[l0 + i] - r0;
            s_roff[i] = d < 0 ? -1 : static_cast<int32_t>(min(d, static_cast<int64_t>(ROW_TILE + 1)));
        }
        __syncthreads();
        const int wend = s_roff[nw];   // tile rows below this lie in the window's findings
        int j = 0;                     // warp-uniform: window finding of the warp's last row so far
        for (int it = 0; it < ROW_ITEMS && w0 + it * 32 < n; it++) {
            const int k = w0 + it * 32 + lane;
            int jl = j;
            if (k < n) {
                int64_t l;
                if (k < wend) {
                    if (s_roff[jl + 1] <= k) jl = last_le(s_roff, jl + 1, nw, static_cast<int32_t>(k));
                    l = l0 + jl;
                } else {
                    l = last_le(foff, l0 + nw, NF, r0 + k);
                }
                if (static_cast<int32_t>(l) != cfi) {
                    cfi = static_cast<int32_t>(l); cf = __ldg(A.io.findings + l);
                    const int2 fl = __ldg(A.f_link + l);
                    cmulti = fl.y > 1;
                    if (!cmulti) { const LinkRec rec = __ldg(A.x_link + fl.x); cvs = rec.x; crel = rec.y; ct0 = rec.w - rec.z - __ldg(foff + l); }
                }
                if (!cmulti) {
                    fn(r0 + k, RowRef{ct0 + r0 + k, cvs, cf, crel, l});
                } else {
                    const int32_t q = static_cast<int32_t>(r0 + k - __ldg(foff + l));
                    const LinkRec rec = link_of_row(A, __ldg(A.f_link + l), q);
                    fn(r0 + k, RowRef{rec.w + static_cast<int64_t>(q - rec.z), rec.x, cf, rec.y, l});
                }
            }
            j = __shfl_sync(FULL, jl, 31);   // rows ascend with the lane; a partial step is the tile's last
        }
        if (threadIdx.x == 0 && r0 + ROW_TILE < R)
            s_l0 = ROW_TILE < wend ? l0 + last_le(s_roff, 0, nw, static_cast<int32_t>(ROW_TILE)) : last_le(foff, l0 + nw, NF, r0 + ROW_TILE);
    }
}

// what one flat row needs: its template row and relationships, and its link's vulnerable source, finding and (vs, finding) relationship
struct RowValue {
    int4 tr;
    uint32_t rp;   // (agent,server) and (server,vs) relationships
    int32_t vs, f, rel;
};

__device__ __forceinline__ RowValue row_value(const PathsArgs &A, const RowRef &x) {
    return RowValue{__ldg(A.t_row + x.t), __ldg(reinterpret_cast<const uint16_t *>(A.t_rel) + x.t), x.vs, x.f, x.rel};
}

__device__ __forceinline__ void emit_row(const PathsArgs &A, int64_t out, const RowValue &v) {
    const int32_t srv = v.tr.y;
    const uint32_t ras = v.rp & 0xFF, rsv = v.rp >> 8;
    reinterpret_cast<int4 *>(A.io.hops)[out] = make_int4(v.tr.x, srv, (v.vs != srv) ? v.vs : -1, v.f);
    // rels are stored 4 bytes per row (the 4th is padding) so a row's relationships are one aligned word
    const uint32_t packed = (v.vs != srv) ? (ras | (rsv << 8) | ((v.rel & 0xFF) << 16) | (0xFEu << 24))
                                          : (ras | ((v.rel & 0xFF) << 8) | (0xFEu << 16) | (0xFEu << 24));
    reinterpret_cast<uint32_t *>(A.io.rels)[out] = packed;
    A.io.ncred[out] = v.tr.z;
    A.io.ntool[out] = v.tr.w;
}

struct ReplicateRows {
    const PathsArgs &A;
    __device__ __forceinline__ void operator()(int64_t r, const RowRef &x) const { emit_row(A, r, row_value(A, x)); }
};

__global__ void __launch_bounds__(ROW_THREADS, 6) replicate_kernel(const PathsArgs A) { for_each_row(A, ReplicateRows{A}); }


// ---- ranking (reference api/routes/graph.py:762-786): sort key of every row, then the requested page is gathered.
// key (descending) = (risk rank, #hops, #distinct credential labels, #distinct tool labels); ties keep emission order
// (Python's stable sort with reverse=True) — the radix sort below is stable on the complemented key.
//
// Focus (the fix-first view's cve / package / agent filter, reference _path_matches_focus, api/routes/graph.py:448-476).  The
// host passes one byte per node; norm(s) = s.strip().lower(), computed on the host with Python string semantics, and nodes
// without a record (ghosts) get 0:
//
//   bit                  set on node u when                                                          checked at hop
//   ABB_FOCUS_CVE        norm(u.label) == cve_n, or u is VULNERABILITY / MISCONFIGURATION              any hop
//                        and norm(u.label or u.id) == cve_n
//   ABB_FOCUS_CVE_FINDING norm((u.label or u.id).strip()) == cve_n  (the path's vuln_ids entry)       the finding hop only
//   ABB_FOCUS_PACKAGE    u is PACKAGE and norm(u.label or u.id) == package_n                          any hop
//   ABB_FOCUS_AGENT      u is AGENT / USER / GROUP / SERVICE_ACCOUNT and norm(u.label or u.id) == agent_n  any hop
//
// The asymmetry is the reference's: the cve test looks at every hop's bare label, but at `label or id` only for finding-typed
// hops and the path's own vuln_ids.  A row (agent, server, vulnerable source, finding) matches when every category named in
// `need` (ABB_FOCUS_CVE / _PACKAGE / _AGENT; a CVE_FINDING bit on the finding counts as CVE) is set on at least one of its hops.
// A focused pass writes row = ~0u for rows that do not match; they are compacted away (order preserved) before the sort.
struct RankArgs {
    const int32_t *base_id;       // [n_findings] index of the finding's base risk value
    const uint32_t *risk_rank;    // [n_base * 5 * 15] dense rank of round(min(100, base + min(10, 3c) + min(10, .75t)), 2), c<=4, t<=14
    const int32_t *ncu;           // [n_nodes] distinct credential labels of a server
    const int32_t *ntu;           // [n_nodes] distinct tool labels of a server
    unsigned long long *keys;     // [n_rows] complemented sort key
    uint32_t *rows;               // [n_rows] row index, ~0u when the row misses the focus
    const uint8_t *focus;         // [n_nodes] focus bits of every node, or nullptr: every row matches
    uint32_t need;               // categories every matching row must satisfy
};

constexpr uint32_t ROW_UNMATCHED = 0xFFFFFFFFu;

__device__ __forceinline__ bool row_matches(const RankArgs &R, int32_t agent, int32_t server, int32_t vs, int32_t f) {
    const uint32_t on_hops = (__ldg(R.focus + agent) | __ldg(R.focus + server) | __ldg(R.focus + vs)) & ~ABB_FOCUS_CVE_FINDING;
    const uint32_t on_f = __ldg(R.focus + f);
    const uint32_t got = on_hops | on_f | ((on_f & ABB_FOCUS_CVE_FINDING) ? ABB_FOCUS_CVE : 0u);
    return (got & R.need) == R.need;
}

struct RankRows {
    const PathsArgs &A;
    const RankArgs &R;
    __device__ __forceinline__ void operator()(int64_t r, const RowRef &x) const {
        const int4 tr = __ldg(A.t_row + x.t);
        const int nc = tr.z < 4 ? tr.z : 4, nt = tr.w < 14 ? tr.w : 14;
        const unsigned long long rr = R.risk_rank[(static_cast<int64_t>(R.base_id[x.fi]) * 5 + nc) * 15 + nt];
        const unsigned long long nh = (x.vs != tr.y) ? 4ull : 3ull;
        const unsigned long long cu = static_cast<unsigned long long>(min(R.ncu[tr.y], 0x3FFFF)), tu = static_cast<unsigned long long>(min(R.ntu[tr.y], 0x3FFFF));
        R.keys[r] = ~((rr << 40) | (nh << 36) | (cu << 18) | tu);
        const bool hit = !R.focus || row_matches(R, tr.x, tr.y, x.vs, x.f);
        R.rows[r] = hit ? static_cast<uint32_t>(r) : ROW_UNMATCHED;
    }
};

__global__ void __launch_bounds__(ROW_THREADS) rank_keys_kernel(const PathsArgs A, const RankArgs R) { for_each_row(A, RankRows{A, R}); }

// cub::DeviceSelect predicate of the focused pass
struct RowMatched {
    __host__ __device__ __forceinline__ bool operator()(uint32_t row) const { return row != ROW_UNMATCHED; }
};

// keys of the compacted rows (their rows ascend, so the stable sort still breaks ties in emission order)
__global__ void gather_keys_kernel(const unsigned long long *keys, const uint32_t *rows, int64_t n, unsigned long long *out) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = keys[rows[i]];
}

// the page [first, first+count) of the sorted order -> flat rows (+ the risk rank so the host can print the float)
__global__ void rank_gather_kernel(const PathsArgs A, const RankArgs R, const uint32_t *sorted_rows, int64_t first, int64_t count, uint32_t *out_rank,
                                   int64_t *out_row) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int64_t row = sorted_rows[first + i];
    // finding = last f with f_off[f] <= row, then the finding's link that holds the row
    const int64_t fi = last_le(A.io.f_off, int64_t{0}, A.io.n_findings, row);
    const int32_t q = static_cast<int32_t>(row - A.io.f_off[fi]);
    const LinkRec l = link_of_row(A, A.f_link[fi], q);
    const RowValue v = row_value(A, RowRef{l.w + static_cast<int64_t>(q - l.z), l.x, A.io.findings[fi], l.y, fi});
    emit_row(A, i, v);
    const int4 tr = v.tr;
    const int nc = tr.z < 4 ? tr.z : 4, nt = tr.w < 14 ? tr.w : 14;
    out_rank[i] = R.risk_rank[(static_cast<int64_t>(R.base_id[fi]) * 5 + nc) * 15 + nt];
    out_row[i] = row;
}

}  // namespace abb
