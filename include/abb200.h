/*
 * abb200.h — C ABI of the H100 blast-radius engine (libabb200.so).
 *
 * This is the drop-in boundary for agent-bom's exposure-graph hot path: every
 * entry point below replaces one reference interface (file:line under
 * /root/reference/src/agent_bom/).  Plain pointers and sizes only — no torch,
 * no C++ types.  INTEGRATION.md shows the ctypes binding a reference
 * maintainer would add (the reference is pure Python, so the FFI is ctypes).
 *
 * Conventions
 *   - every function returns ABB_OK (0) or a negative abb_status; the message
 *     of the last failure on the calling thread is abb_last_error().
 *   - "device" pointers are CUDA global-memory addresses on the graph's
 *     device; "host" pointers are ordinary (ideally pinned) host memory.
 *   - node ids are dense int32 indices (host keeps the string table); an id
 *     that occurs only as an edge endpoint is a "ghost" (node_type 255).
 *   - there is no CPU fallback anywhere in this library: without a CUDA
 *     device every compute entry point fails with ABB_ERR_CUDA.
 */
#ifndef ABB200_H
#define ABB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ABB_VERSION 110

typedef enum abb_status {
    ABB_OK = 0,
    ABB_ERR_CUDA = -1,      /* CUDA runtime failure or no device */
    ABB_ERR_ARG = -2,       /* invalid argument */
    ABB_ERR_CAPACITY = -3,  /* caller-provided arena too small (needed sizes are reported) */
    ABB_ERR_NOMEM = -4
} abb_status;

/* adjacency-entry meta byte (device format, DESIGN.md §3) */
#define ABB_META_REL_MASK 0x1Fu
#define ABB_META_TRAVERSABLE 0x20u
#define ABB_META_FIRST_PAIR 0x40u   /* first entry of its row with this neighbour (set by the CSR build) */
#define ABB_META_REVERSED_COPY 0x80u
/* per-edge input flags of the edge stream */
#define ABB_EDGE_TRAVERSABLE 1u
#define ABB_EDGE_BIDIRECTIONAL 2u

#define ABB_NODE_GHOST 255u
#define ABB_N_ENTITY_TYPES 24
#define ABB_N_REL_TYPES 31

const char *abb_last_error(void);
int abb_version(void);
int abb_device_count(void);

/* ------------------------------------------------------------------------
 * (a1) adjacency model — replaces UnifiedGraph.add_edge's adjacency /
 * reverse_adjacency dict-of-lists (graph/container.py:97-101,146-198).
 *
 * Row u of the forward CSR is graph.adjacency[u] in list order, row u of the
 * reverse CSR is graph.reverse_adjacency[u] in list order: original edge i
 * (graph.edges order) contributes (row=src,nbr=dst,eid2=2i) forward and
 * (row=dst,nbr=src,eid2=2i) reverse; a bidirectional edge also contributes
 * its reversed copy (row=dst,nbr=src,eid2=2i+1) forward and
 * (row=src,nbr=dst,eid2=2i+1) reverse.  meta = rel(5 bits) | TRAVERSABLE |
 * FIRST_PAIR | REVERSED_COPY.  Entries of adjacency[a] with neighbour b and
 * entries of reverse_adjacency[b] with neighbour a correspond one-to-one in the
 * same order, so FIRST_PAIR on either side marks the edge whose relationship
 * the reference's by_pair.setdefault((a,b)) keeps (api/routes/graph.py:492-497).
 * ---------------------------------------------------------------------- */
typedef struct abb_csr {
    int32_t n_nodes;          /* real nodes + ghosts */
    int64_t n_entries;        /* entries per direction = n_edges + #bidirectional */
    const uint32_t *fwd_off;  /* [n_nodes+1] */
    const int32_t *fwd_nbr;   /* [n_entries] */
    const uint8_t *fwd_meta;  /* [n_entries] */
    const uint32_t *fwd_eid;  /* [n_entries] eid2 = 2*edge_index + reversed_copy */
    const uint32_t *rev_off;
    const int32_t *rev_nbr;
    const uint8_t *rev_meta;
    const uint32_t *rev_eid;
    const uint8_t *node_type; /* [n_nodes] entity code, 255 = ghost */
    const int32_t *node_rank; /* [n_nodes] rank of the id string among all ids (for sorted() outputs); may be NULL */
} abb_csr;

/* number of adjacency entries per direction for an edge stream */
int64_t abb_csr_entries(int64_t n_edges, const uint8_t *flags);

/* Host-side stable CSR build (counting sort, insertion order preserved).  All
 * output arrays are caller-allocated: *_off[n_nodes+1], others [abb_csr_entries]. */
int abb_csr_build_host(int32_t n_nodes, int64_t n_edges, const int32_t *src, const int32_t *dst, const uint8_t *rel,
                       const uint8_t *flags, uint32_t *fwd_off, int32_t *fwd_nbr, uint8_t *fwd_meta, uint32_t *fwd_eid,
                       uint32_t *rev_off, int32_t *rev_nbr, uint8_t *rev_meta, uint32_t *rev_eid);

typedef struct abb_graph abb_graph; /* device-resident CSR pair + node types */

/* copy a host CSR to `device` (library-owned device memory) */
int abb_graph_upload(int device, const abb_csr *host, abb_graph **out);
/* wrap device arrays owned by the caller (e.g. torch tensors filled by an NCCL broadcast) */
int abb_graph_adopt(int device, const abb_csr *dev, abb_graph **out);
/* device pointers of a graph (for broadcast / inspection) */
int abb_graph_view(const abb_graph *g, abb_csr *out);
int64_t abb_graph_bytes(const abb_graph *g);
/* Root-frontier de-duplication of single-source batches (on by default; env ABB_DEDUP=0 disables at creation).
 * Sources whose depth-1 frontier is identical share one traversal and one result slice; results are
 * bit-identical either way (q_start of different queries may then alias the same arena range). */
int abb_graph_set_dedup(abb_graph *g, int enabled);
int abb_graph_device(const abb_graph *g);
/* Tuning / test switches of a handle; results never depend on them.  Names: "dedup" (0/1), "block_tiers" (bit 0 = the
 * 8-warp mid tier, bit 1 = the 32-warp big tier of csrc/walkb.cuh; env ABB_BLOCK_TIERS at creation), "mid_qcap" /
 * "big_qcap" (queue entries a block tier accepts before it hands a query to the next tier — the GPU tests shrink them so
 * every hand-off is exercised on small graphs), "big_limit" (the big tier takes the forecast-heavy queries of a batch when there are
 * at most this many, otherwise they go first in line to the warp tier; default 24 per SM), "zero_copy" (0/1).  get returns -1 for an unknown name. */
int abb_graph_set_option(abb_graph *g, const char *name, int64_t value);
int64_t abb_graph_get_option(const abb_graph *g, const char *name);
void abb_graph_free(abb_graph *g);

/* ------------------------------------------------------------------------
 * Batched ordered frontier BFS ("walk").  One spec covers every traversal of
 * the reference engine; the abb_spec_* constructors below state the mapping.
 *
 * Semantics (identical to the reference's deque loops): FIFO queue seeded
 * with the query's roots in order; a node is expanded only while
 * depth < max_depth (max_depth < 0: unbounded); candidates of a node are its
 * forward row (direction & 1) then its reverse row (direction & 2) in list
 * order; a candidate passes iff its relationship bit is in rel_mask and
 * (not TRAVERSABLE_ONLY or the entry is traversable); every passing candidate
 * counts toward max_edges; an unvisited neighbour is appended (visited is
 * marked at enqueue) unless max_nodes visited nodes already exist.  Output
 * order == the reference's discovery order, parents == first-discoverer.
 * ---------------------------------------------------------------------- */
#define ABB_DIR_FORWARD 1
#define ABB_DIR_REVERSE 2
#define ABB_DIR_BOTH 3

#define ABB_WALK_TRAVERSABLE_ONLY 0x001u /* skip non-traversable entries */
#define ABB_WALK_MARK_ROOTS 0x002u       /* roots start visited (include_roots / single-source BFS) */
#define ABB_WALK_OMIT_ROOTS 0x004u       /* do not emit the seeded root entries */
#define ABB_WALK_PARENTS 0x008u          /* emit parent position (within the query's full queue, -1 for roots) */
#define ABB_WALK_DEPTHS 0x010u           /* emit depth per emitted node */
#define ABB_WALK_EDGES 0x020u            /* emit eid2 of every passing candidate in scan order */
#define ABB_WALK_HIST 0x040u             /* per-query histogram of entity types over emitted non-root nodes */
#define ABB_WALK_REAL_ROOTS 0x080u       /* roots that are ghosts / out of range are dropped (query flag bit1 if none left) */
#define ABB_WALK_TARGET 0x100u           /* stop at first discovery of targets[q] (shortest_path) */

#define ABB_QFLAG_TRUNCATED 1   /* a max_nodes / max_edges budget was hit */
#define ABB_QFLAG_NO_ROOT 2     /* no valid root (reference returns its empty result) */
#define ABB_QFLAG_TARGET_FOUND 4

typedef struct abb_walk_spec {
    int32_t direction;  /* ABB_DIR_* */
    int32_t max_depth;  /* < 0: unbounded */
    uint32_t rel_mask;  /* bit r set = relationship code r allowed (bit 31 = "other") */
    uint32_t flags;     /* ABB_WALK_* */
    int64_t max_nodes;  /* < 0: unbounded */
    int64_t max_edges;  /* < 0: unbounded */
    uint32_t emit_types;/* bit t set = emit nodes of entity code t; bit 31 = ghosts/other; 0xFFFFFFFF = all */
    uint32_t reserved;
} abb_walk_spec;

/* UnifiedGraph.impact_of(node, max_depth) — graph/container.py:230-279 */
abb_walk_spec abb_spec_impact_of(int32_t max_depth);
/* UnifiedGraph.bfs(source, max_depth, traversable_only) — graph/container.py:367-391 */
abb_walk_spec abb_spec_bfs(int32_t max_depth, int32_t traversable_only);
/* UnifiedGraph.reachable_from(source, max_depth, traversable_only) — graph/container.py:411-436 */
abb_walk_spec abb_spec_reachable_from(int32_t max_depth, int32_t traversable_only);
/* UnifiedGraph.shortest_path(source, target) — graph/container.py:393-409 */
abb_walk_spec abb_spec_shortest_path(void);
/* UnifiedGraph.traverse_subgraph(...) — graph/container.py:438-538; rel_mask = relationship_types (0 = all) */
abb_walk_spec abb_spec_traverse_subgraph(int32_t direction, int32_t max_depth, int64_t max_nodes, int64_t max_edges,
                                         int32_t traversable_only, uint32_t rel_mask, int32_t static_only,
                                         int32_t dynamic_only, int32_t include_roots);
/* _bfs_distances_along(graph, start, allowed) — graph/dependency_reach.py:169-198 */
abb_walk_spec abb_spec_distances_along(uint32_t rel_mask, uint32_t emit_types);

/* Device-buffer form.  All pointers are device memory on the graph's device
 * except where noted; optional outputs may be NULL when the matching flag is
 * clear.  Results of query q occupy nodes[q_start[q] .. q_start[q]+q_count[q])
 * (and edges[q_estart[q] .. +q_ecount[q])).  Slices are bump-allocated, so
 * their order in the arena is unspecified; their contents are deterministic. */
typedef struct abb_walk_io {
    int64_t n_queries;
    const int32_t *roots;     /* [root_off[n_queries]] or [n_queries] when root_off == NULL */
    const int64_t *root_off;  /* NULL: query q has the single root roots[q] */
    const int32_t *targets;   /* [n_queries], ABB_WALK_TARGET only */
    int64_t *q_start;         /* [n_queries] */
    int32_t *q_count;         /* [n_queries] */
    int32_t *q_maxd;          /* [n_queries] max depth reached */
    int32_t *q_flags;         /* [n_queries] ABB_QFLAG_* */
    int64_t *q_estart;        /* [n_queries] (EDGES) */
    int64_t *q_ecount;        /* [n_queries] (EDGES) recorded candidates */
    uint32_t *q_hist;         /* [n_queries*24] (HIST) */
    int32_t *nodes;           /* [node_cap] */
    int32_t *parent;          /* [node_cap] (PARENTS) */
    int32_t *depth;           /* [node_cap] (DEPTHS) */
    int64_t node_cap;
    uint32_t *edges;          /* [edge_cap] (EDGES) */
    int64_t edge_cap;
    unsigned long long *totals; /* device [2]: nodes / edges needed; zeroed by the launch */
} abb_walk_io;

/* Enqueue the walk on `stream` (a cudaStream_t, NULL = default stream).  Asynchronous.  One walk may be in flight per
 * graph handle (the tiers share the handle's scratch); serialise callers or use one handle per stream. */
int abb_walk_launch(abb_graph *g, const abb_walk_spec *spec, const abb_walk_io *io, void *stream);
/* 64-bit signature of each single-source query's depth-1 frontier (device arrays).  Sources with equal signatures
 * share one traversal when walked in the same batch, so multi-GPU runs shard the source list by signature
 * (sig mod world) instead of by position; bit 63 marks sources that are walked individually. */
int abb_walk_signatures(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, int64_t n, unsigned long long *sig, void *stream);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
int64_t abb_launch_count(void);
/* Timing hooks: elapsed milliseconds of the walk kernels of the most recent
 * abb_walk_launch / *_host call on this graph (CUDA events on the launch stream;
 * synchronises that stream). */
float abb_last_walk_ms(abb_graph *g);
/* {queries, frontier groups walked once, sources walked individually, sources eligible for sharing} of the most recent
 * walk on this graph (zeros after the first when the batch was not de-duplicated).  Synchronises the device. */
int abb_last_walk_stats(abb_graph *g, int64_t *out4);
/* Hand-offs between the storage tiers of the most recent walk: out8[0..3] = {queries S1 handed on, of which forecast-heavy
 * (taken by the big block tier, or first in line for G1), queries the mid block tier handed on, queries G1 handed to GX} for
 * the first pass (canonical walks when de-duplicated), out8[4..7] the same for the individual pass.
 * Diagnostics for bench.py / the tier tests.  Synchronises the device. */
int abb_last_walk_tier_counts(abb_graph *g, int64_t *out8);
float abb_last_paths_ms(abb_graph *g);

/* Host-buffer form (the call the Python store makes): H2D of the roots, the
 * walk, D2H of the results, arenas sized automatically.  The result owns
 * pinned host arrays; accessors return pointers valid until abb_walk_result_free. */
typedef struct abb_walk_result abb_walk_result;
int abb_walk_host(abb_graph *g, const abb_walk_spec *spec, const int32_t *roots, const int64_t *root_off,
                  const int32_t *targets, int64_t n_queries, abb_walk_result **out);
int64_t abb_walk_result_queries(const abb_walk_result *r);
int64_t abb_walk_result_total_nodes(const abb_walk_result *r);
int64_t abb_walk_result_total_edges(const abb_walk_result *r);
const int64_t *abb_walk_result_start(const abb_walk_result *r);
const int32_t *abb_walk_result_count(const abb_walk_result *r);
const int32_t *abb_walk_result_maxd(const abb_walk_result *r);
const int32_t *abb_walk_result_flags(const abb_walk_result *r);
const int64_t *abb_walk_result_estart(const abb_walk_result *r);
const int64_t *abb_walk_result_ecount(const abb_walk_result *r);
const uint32_t *abb_walk_result_hist(const abb_walk_result *r);
/* Histograms as they crossed PCIe (batches of >= 1024 queries, option "hist_pack", default on): only the entity-type columns
 * that are non-zero somewhere in the batch (bit t of *columns_mask = column t, ascending), row-major [n_queries x popcount(mask)],
 * counts of *bytes_per_count bytes (2 unless a count exceeds 65 535, else 4).  This is the reference's `affected_by_type`
 * (graph/container.py:268-276: a dict holding only the types present).  abb_walk_result_hist rebuilds the dense
 * [n_queries x ABB_N_ENTITY_TYPES] uint32 table from it on first call.  Returns NULL when the result holds the dense table. */
const void *abb_walk_result_hist_packed(const abb_walk_result *r, uint32_t *columns_mask, int32_t *bytes_per_count);
const int32_t *abb_walk_result_nodes(const abb_walk_result *r);
const int32_t *abb_walk_result_parent(const abb_walk_result *r);
const int32_t *abb_walk_result_depth(const abb_walk_result *r);
const uint32_t *abb_walk_result_edges(const abb_walk_result *r);
int64_t abb_walk_result_h2d_bytes(const abb_walk_result *r);
int64_t abb_walk_result_d2h_bytes(const abb_walk_result *r);
void abb_walk_result_free(abb_walk_result *r);

/* ------------------------------------------------------------------------
 * Derived exposure paths — replaces _derived_attack_paths' topology walk
 * (api/routes/graph.py:686-760) and _edge_relationships_for_hops (:488-503).
 * One row per (agent, server, vulnerable_source, finding), in the reference's
 * emission order (findings in the given order, in-edges in graph.edges order,
 * agents sorted by node_rank).  Risk scoring and the final stable sort
 * (:762-786) need Python floats and are done by the host layer.
 *   hops [n_paths*4] : agent, server, vulnerable_source (-1 when it is the server), finding
 *   rels [n_paths*4] : relationship code per consecutive hop pair (3 used, the 4th byte pads the row to one
 *                      aligned word); -1 = the pair has no edge (the reference skips it); -2 = not applicable
 *   ncred/ntool      : EXPOSES_CRED / PROVIDES_TOOL out-edges of the server (un-deduplicated)
 * ---------------------------------------------------------------------- */
typedef struct abb_paths_io {
    int64_t n_findings;
    const int32_t *findings;  /* device [n_findings] */
    int64_t *f_off;           /* device [n_findings+1] exclusive scan of per-finding path counts */
    int32_t *hops;            /* device [row_cap*4], 16-byte aligned */
    int8_t *rels;             /* device [row_cap*4], 4-byte aligned */
    int32_t *ncred;           /* device [row_cap] */
    int32_t *ntool;           /* device [row_cap] */
    int64_t row_cap;
} abb_paths_io;

/* pass 1: per-finding counts + exclusive scan into f_off (f_off[n_findings] = total rows) */
int abb_paths_count_launch(abb_graph *g, const abb_paths_io *io, void *stream);
/* pass 2: fill rows (requires row_cap >= total) */
int abb_paths_fill_launch(abb_graph *g, const abb_paths_io *io, void *stream);

/* Host-buffer form.  What crosses PCIe is the factorised result — per finding its links (vulnerable source +
 * relationship of the pair (source, finding)), per link the template slice of that source — which determines every
 * row; the flat hops/rels/ncred/ntool arrays are expanded from it on the host the first time they are asked for. */
typedef struct abb_paths_result abb_paths_result;
int abb_paths_host(abb_graph *g, const int32_t *findings, int64_t n_findings, abb_paths_result **out);
int64_t abb_paths_result_links(const abb_paths_result *r);
int64_t abb_paths_result_template_rows(const abb_paths_result *r);
const int64_t *abb_paths_result_link_off(const abb_paths_result *r);      /* [n_findings+1] links of finding i */
const int32_t *abb_paths_result_link_source(const abb_paths_result *r);   /* [n_links] vulnerable source */
const int8_t *abb_paths_result_link_rel(const abb_paths_result *r);       /* [n_links] relationship (source, finding) */
const int64_t *abb_paths_result_link_row_off(const abb_paths_result *r);  /* [n_links+1] first flat row of each link */
const int64_t *abb_paths_result_link_template(const abb_paths_result *r); /* [n_links] first template row of the link's source */
const int32_t *abb_paths_result_template(const abb_paths_result *r);      /* [n_template_rows*4] agent, server, ncred, ntool */
const int8_t *abb_paths_result_template_rel(const abb_paths_result *r);   /* [n_template_rows*2] (agent,server), (server,source) */
int64_t abb_paths_result_rows(const abb_paths_result *r);
const int64_t *abb_paths_result_off(const abb_paths_result *r); /* [n_findings+1] */
const int32_t *abb_paths_result_hops(const abb_paths_result *r);
const int8_t *abb_paths_result_rels(const abb_paths_result *r);
const int32_t *abb_paths_result_ncred(const abb_paths_result *r);
const int32_t *abb_paths_result_ntool(const abb_paths_result *r);
int64_t abb_paths_result_h2d_bytes(const abb_paths_result *r);
int64_t abb_paths_result_d2h_bytes(const abb_paths_result *r);
void abb_paths_result_free(abb_paths_result *r);

/* Ranked page of exposure-path rows — the ordering of _derived_attack_paths (api/routes/graph.py:782-786): descending by
 * (composite risk, #hops, #distinct credential labels, #distinct tool labels), ties in emission order.  The float
 * formula (:762-771, Python round) stays on the host: the caller passes, per finding, the index of its base risk
 * value, and a table risk_rank[n_base][5][15] with the dense rank of the rounded score for each (base, min(ncred,4),
 * min(ntool,14)); ncu / ntu are the per-server counts of distinct credential / tool labels.  Returns rows
 * [offset, offset+limit) of the sorted order plus the total row count. */
typedef struct abb_rank_result abb_rank_result;
int abb_paths_rank_host(abb_graph *g, const int32_t *findings, int64_t n_findings, const int32_t *base_id, const uint32_t *risk_rank,
                        int64_t n_base, const int32_t *ncu, const int32_t *ntu, int64_t offset, int64_t limit, abb_rank_result **out);

/* Focused ranking — the fix-first view's cve / package / agent filter (api/routes/graph.py:448-476).  node_focus[n_nodes]
 * holds ABB_FOCUS_* bits per node (see the table in csrc/paths.cuh); a row matches when every category in `need`
 * (ABB_FOCUS_CVE | ABB_FOCUS_PACKAGE | ABB_FOCUS_AGENT) is set on one of its hops, ABB_FOCUS_CVE_FINDING counting as CVE on the
 * finding hop only.  Only the matched rows are sorted (same order as above); the page is taken from them.  total stays the
 * count of all rows, matched counts the rows that pass.  node_focus == NULL: every row matches (abb_paths_rank_host). */
#define ABB_FOCUS_CVE 0x1u
#define ABB_FOCUS_CVE_FINDING 0x2u
#define ABB_FOCUS_PACKAGE 0x4u
#define ABB_FOCUS_AGENT 0x8u
int abb_paths_rank_focus_host(abb_graph *g, const int32_t *findings, int64_t n_findings, const int32_t *base_id, const uint32_t *risk_rank,
                              int64_t n_base, const int32_t *ncu, const int32_t *ntu, const uint8_t *node_focus, uint32_t need, int64_t offset,
                              int64_t limit, abb_rank_result **out);
int64_t abb_rank_result_matched(const abb_rank_result *r);
int64_t abb_rank_result_total(const abb_rank_result *r);
int64_t abb_rank_result_count(const abb_rank_result *r);
const int32_t *abb_rank_result_hops(const abb_rank_result *r);       /* [count*4] */
const int8_t *abb_rank_result_rels(const abb_rank_result *r);        /* [count*4] */
const int32_t *abb_rank_result_ncred(const abb_rank_result *r);
const int32_t *abb_rank_result_ntool(const abb_rank_result *r);
const uint32_t *abb_rank_result_risk_rank(const abb_rank_result *r); /* [count] index into the caller's sorted score list */
const int64_t *abb_rank_result_row(const abb_rank_result *r);        /* [count] emission-order row index */
void abb_rank_result_free(abb_rank_result *r);

/* ------------------------------------------------------------------------
 * One "exposure traversal" per finding = impact_of(f, max_depth) + f's derived
 * exposure paths (the unit of BASELINE.json's metric).  Host-buffer form used
 * by the store's batched API and by bench.py's e2e leg: both kernels are
 * enqueued back to back and the result copies overlap.
 * ---------------------------------------------------------------------- */
int abb_exposure_host(abb_graph *g, const int32_t *findings, int64_t n_findings, int32_t max_depth,
                      abb_walk_result **impact_out, abb_paths_result **paths_out);

/* ------------------------------------------------------------------------
 * Finding context — the graph_context block of UnifiedGraph.to_ocsf_events
 * (graph/container.py:628-654) for a batch of findings:
 *   - the finding's in-neighbours (sources_of: reverse_adjacency[f] in list
 *     order, reversed twins of bidirectional edges included, duplicates kept)
 *     whose entity type is agent / server / package / credential, one list per
 *     ABB_CTX_* bucket; ghosts and every other kind are not listed;
 *   - impact_of(f, max_depth)'s affected_count, max depth, flags and entity-type
 *     histogram (the impact walk, unchanged).
 * The walk's node slices stay in device memory: they never cross PCIe, whatever
 * the zero_copy / chunks options say.  What comes back, per finding q:
 * count / maxd / flags (int32), the histogram (packed as abb_walk_result_hist_packed
 * describes, or dense), start (int64) and bucket counts (int32 [n*ABB_CTX_BUCKETS]);
 * sources[start[q] ..] holds bucket 0's sources, then bucket 1's, ... in row order.
 * An invalid or ghost finding index has empty lists (and the walk's NO_ROOT flag).
 * ---------------------------------------------------------------------- */
#define ABB_CTX_AGENT 0
#define ABB_CTX_SERVER 1
#define ABB_CTX_PACKAGE 2
#define ABB_CTX_CREDENTIAL 3
#define ABB_CTX_BUCKETS 4
#define ABB_CTX_NONE 255
typedef struct abb_finding_context_result abb_finding_context_result;
int abb_finding_context_host(abb_graph *g, int32_t max_depth, const int32_t *findings, int64_t n_findings, abb_finding_context_result **out);
int64_t abb_finding_context_result_queries(const abb_finding_context_result *r);
const int32_t *abb_finding_context_result_count(const abb_finding_context_result *r);
const int32_t *abb_finding_context_result_maxd(const abb_finding_context_result *r);
const int32_t *abb_finding_context_result_flags(const abb_finding_context_result *r);
/* packed histogram (same contract as abb_walk_result_hist_packed); NULL when the dense table was shipped */
const void *abb_finding_context_result_hist_packed(const abb_finding_context_result *r, uint32_t *columns_mask, int32_t *bytes_per_count);
const uint32_t *abb_finding_context_result_hist(const abb_finding_context_result *r);     /* dense [n*ABB_N_ENTITY_TYPES] */
const int64_t *abb_finding_context_result_start(const abb_finding_context_result *r);     /* [n] */
const int32_t *abb_finding_context_result_bucket_counts(const abb_finding_context_result *r); /* [n*ABB_CTX_BUCKETS] */
int64_t abb_finding_context_result_total_sources(const abb_finding_context_result *r);
const int32_t *abb_finding_context_result_sources(const abb_finding_context_result *r);   /* [total_sources] */
int64_t abb_finding_context_result_h2d_bytes(const abb_finding_context_result *r);
int64_t abb_finding_context_result_d2h_bytes(const abb_finding_context_result *r);
/* device time of the impact walk and of the context kernels (CUDA events; the two run on different streams and overlap) */
float abb_finding_context_result_walk_ms(const abb_finding_context_result *r);
float abb_finding_context_result_context_ms(const abb_finding_context_result *r);
void abb_finding_context_result_free(abb_finding_context_result *r);

/* ------------------------------------------------------------------------
 * compute_dependency_reach — graph/dependency_reach.py:109-220.
 * Pass 1: walk from every agent along rel_mask (unbounded depth), keeping
 * package nodes and hop counts.  Pass 2 (device sort/segment): per package the
 * reaching agents sorted by node_rank + min hops; per vulnerability the
 * attached packages (affects / vulnerable_to in either list), the union of
 * their agents and the min of their mins.
 * All outputs are host arrays owned by the result.
 * ---------------------------------------------------------------------- */
typedef struct abb_reach_result abb_reach_result;
int abb_dependency_reach_host(abb_graph *g, const int32_t *agents, int64_t n_agents, uint32_t rel_mask,
                              uint32_t vuln_pkg_mask, abb_reach_result **out);
int64_t abb_reach_n_packages(const abb_reach_result *r);
const int32_t *abb_reach_pkg_ids(const abb_reach_result *r);     /* package nodes in node order */
const int64_t *abb_reach_pkg_off(const abb_reach_result *r);     /* [n_packages+1] */
const int32_t *abb_reach_pkg_agents(const abb_reach_result *r);  /* agents sorted by node_rank */
const int32_t *abb_reach_pkg_minhop(const abb_reach_result *r);  /* 0 when unreached */
int64_t abb_reach_n_vulns(const abb_reach_result *r);
const int32_t *abb_reach_vuln_ids(const abb_reach_result *r);
const int64_t *abb_reach_vuln_poff(const abb_reach_result *r);
const int32_t *abb_reach_vuln_pkgs(const abb_reach_result *r);   /* sorted by node_rank */
const int64_t *abb_reach_vuln_aoff(const abb_reach_result *r);
const int32_t *abb_reach_vuln_agents(const abb_reach_result *r); /* sorted by node_rank */
const int32_t *abb_reach_vuln_minhop(const abb_reach_result *r);
void abb_reach_result_free(abb_reach_result *r);

/* ---- sampled bottleneck score -----------------------------------------------------------------------------------
 * Replaces the BFS loop of UnifiedGraph.bottleneck_nodes (agent_bom/graph/container.py:548-567) and
 * InMemoryBackend.bottleneck_nodes (agent_bom/graph_backend.py:127-155): from each source an unbounded forward BFS
 * over every adjacency entry; each node strictly inside the first-discoverer path to a reached node gets +1.
 * scores_out: host [n_nodes] — the un-normalised integer scores summed over all sources (the caller divides by their
 * sum and sorts, as the reference does).  Sources must be nodes with a record (ghost / invalid sources add nothing). */
int abb_bottleneck_host(abb_graph *g, const int32_t *sources, int64_t n_sources, uint64_t *scores_out);

/* ---- NetworkX analysis backend ----------------------------------------------------------------------------------
 * The answers of the reference's NetworkXBackend (agent_bom/graph_backend.py:158-242), bit for bit with networkx 3.6.1.
 * The graph is an nx.DiGraph exported in node order: forward row u = G.succ[u] in dict order, reverse row u = G.pred[u]
 * in dict order, no row repeating a neighbour, every node real.  Option "nx_batch" caps the betweenness sources per batch and
 * the path-search slots (results never depend on it).
 *
 * PageRank — nx.pagerank(G) (_pagerank_scipy, alpha 0.85, max_iter 100, tol 1e-6, weight "weight"): weights[n_entries] is
 * the edge weight of each forward entry as f64.  scores_out: host [n_nodes]; *iterations_out: power iterations run.
 * ABB_ERR_ARG when the iteration does not converge (networkx raises PowerIterationFailedConvergence). */
int abb_pagerank_host(abb_graph *g, const double *weights, double *scores_out, int32_t *iterations_out);
/* Betweenness — nx.betweenness_centrality(G): exact Brandes from every source, normalised, endpoints excluded. */
int abb_betweenness_host(abb_graph *g, double *scores_out);
/* Shortest paths — nx.shortest_path(G, s, t) (_bidirectional_pred_succ) for a batch of pairs of valid node indices: the path
 * of pair q is nodes[start[q] .. start[q]+length[q]), source first; length 0 = no path; s == t gives [s]. */
typedef struct abb_bidir_result abb_bidir_result;
int abb_bidir_paths_host(abb_graph *g, const int32_t *sources, const int32_t *targets, int64_t n_pairs, abb_bidir_result **out);
const int64_t *abb_bidir_result_start(const abb_bidir_result *r);   /* [n_pairs] */
const int32_t *abb_bidir_result_length(const abb_bidir_result *r);  /* [n_pairs] */
int64_t abb_bidir_result_total(const abb_bidir_result *r);
const int32_t *abb_bidir_result_nodes(const abb_bidir_result *r);   /* [total] */
void abb_bidir_result_free(abb_bidir_result *r);

/* ---- lateral-movement path search -------------------------------------------------------------------------------
 * Replaces the queue loop of find_lateral_paths (agent_bom/context_graph.py:397-477) for a batch of sources: a FIFO of
 * simple paths over graph.adjacency, at most 100 recorded paths and 10 000 waiting paths per source, paths no longer
 * than max_depth+1 nodes, in the reference's discovery order (the caller scores and sorts them, :574-593).
 * adj_off[n_nodes+1] / adj_nbr / adj_kind: graph.adjacency rows in list order (edge kind 0..15);
 * node_kind: 0 agent, 1 server, 2 credential, 3 tool, 4 vulnerability, 5 iam_role, 255 = id without a node record;
 * node_key: agents: id of the label; credentials / tools: id of metadata["agent"], -1 when absent or empty; others ignored;
 * sources / source_key: start node (-1 = unknown id: no paths) and the id of the source's agent name.
 * max_depth 0..7.  max_pops: safety valve per source (<= 0: 50 M); a source that hits it has flag bit0 set and its result
 * must be discarded.  Records: W+2 int32 words — length, edge kinds (4 bits per hop, first hop lowest), W node ids. */
typedef struct abb_lateral_result abb_lateral_result;
int abb_lateral_paths_host(int device, int32_t n_nodes, const int64_t *adj_off, const int32_t *adj_nbr, const uint8_t *adj_kind,
                           const uint8_t *node_kind, const int32_t *node_key, int64_t n_sources, const int32_t *sources,
                           const int32_t *source_key, int32_t max_depth, int64_t max_pops, abb_lateral_result **out);
const int64_t *abb_lateral_result_off(const abb_lateral_result *r);      /* [n_sources+1] */
const int32_t *abb_lateral_result_records(const abb_lateral_result *r);  /* [off[n_sources]][W+2] */
const int32_t *abb_lateral_result_flags(const abb_lateral_result *r);    /* [n_sources] */
int32_t abb_lateral_result_width(const abb_lateral_result *r);           /* W = max_depth + 2 */
double abb_lateral_result_ms(const abb_lateral_result *r);
void abb_lateral_result_free(abb_lateral_result *r);

/* Enrichment of found lateral paths: what _build_lateral_path (agent_bom/context_graph.py:495-572) folds into each path,
 * computed for many paths at once.  Per path: the kept labels in first-add order, each category << 30 | label id (category 0
 * credential, 1 tool, 2 vulnerability; a credential name carried by a shares_credential link shares the credential ids), the
 * number of execute-capable tools and the highest severity score among first-added labels.
 * adj_* as for abb_lateral_paths_host; adj_name: per entry, for shares_server_kind entries the surface of the link's server
 * name, for shares_credential_kind entries the credential id of the link's credential name, -1 when the name is empty or absent.
 * node_label: label id of credential / tool / vulnerability nodes (< 2^30); node_value: tools 1 execute / 0 not, vulnerabilities
 * their severity score, -1 when the node's test raised; node_surface: a server node's surface, -1 when it has none.
 * surface_off[n_surfaces+1] / surface_node: per surface the credential / tool / vulnerability nodes that first add each label of
 * it, in order (each server's exposes / provides / vulnerable_to entries, and per shared server name those of every server with
 * that label in node order).  records: [n_paths][width+2] as abb_lateral_result_records gives them.
 * flags bit0: a first-added label's value is -1 (the caller re-derives that path to raise what the reference raises). */
typedef struct abb_lateral_enrich_result abb_lateral_enrich_result;
int abb_lateral_enrich_host(int device, int32_t n_nodes, const int64_t *adj_off, const int32_t *adj_nbr, const uint8_t *adj_kind,
                            const int32_t *adj_name, int32_t shares_server_kind, int32_t shares_credential_kind, const uint8_t *node_kind,
                            const int32_t *node_label, const float *node_value, const int32_t *node_surface, int32_t n_surfaces,
                            const int64_t *surface_off, const int32_t *surface_node, int64_t n_paths, int32_t width, const int32_t *records,
                            abb_lateral_enrich_result **out);
const int64_t *abb_lateral_enrich_result_off(const abb_lateral_enrich_result *r);     /* [n_paths+1] */
const int32_t *abb_lateral_enrich_result_items(const abb_lateral_enrich_result *r);   /* [off[n_paths]] */
const int32_t *abb_lateral_enrich_result_exec(const abb_lateral_enrich_result *r);    /* [n_paths] */
const float *abb_lateral_enrich_result_severity(const abb_lateral_enrich_result *r);  /* [n_paths] */
const int32_t *abb_lateral_enrich_result_flags(const abb_lateral_enrich_result *r);   /* [n_paths] */
double abb_lateral_enrich_result_ms(const abb_lateral_enrich_result *r);
void abb_lateral_enrich_result_free(abb_lateral_enrich_result *r);

/* ---- per-group union of member item lists (effective-reach scoring) ------------------------------------------
 * Replaces the per-vulnerability reduction of agent_bom/effective_reach.py:372-426 (`compute`): for every group
 * (a vulnerability) over its members (the servers VULNERABLE_TO it, effective_reach.py:265-279) return
 *   - the sorted, de-duplicated union of the members' item lists (label ranks of reachable tools / credentials /
 *     agents, :281-353 — the caller encodes the category in the top bits of the item so one call serves all three),
 *   - the maximum of two per-member byte weights (strongest tool capability / credential tier, :389-398).
 * member_off[n_groups+1] / members[]: CSR of member indices per group; item_off[n_members+1] / items[]: CSR of
 * non-negative int32 items per member; w0 / w1: [n_members] or NULL.  All pointers are host memory.
 * Result: off[n_groups+1], items[off[n_groups]] ascending within a group, w0[n_groups], w1[n_groups]. */
typedef struct abb_union_result abb_union_result;
int abb_group_union_host(int device, int64_t n_groups, const int64_t *member_off, const int32_t *members, int64_t n_members,
                         const int64_t *item_off, const int32_t *items, const uint8_t *w0, const uint8_t *w1,
                         abb_union_result **out);
const int64_t *abb_union_result_off(const abb_union_result *r);
const int32_t *abb_union_result_items(const abb_union_result *r);
const uint8_t *abb_union_result_w0(const abb_union_result *r);
const uint8_t *abb_union_result_w1(const abb_union_result *r);
double abb_union_result_ms(const abb_union_result *r);            /* device time of the kernels, CUDA events */
void abb_union_result_free(abb_union_result *r);

/* ---- semantic clusters ---------------------------------------------------------------------------------------
 * Replaces the roll-ups of build_semantic_clusters (agent_bom/graph/semantic_clusters.py:81-124).  The host interns each
 * node's cluster keys into codes [n_nodes][2] (int32 in [0, k), -1 = none; ghosts have none) and passes per node a severity
 * level (0 critical, 1 high, 2 medium, 3 low, 4 none), the rounded risk (f64, >= 0) and an entity-type index (< 64).
 * abb_clusters_build_host builds the graph-constant tables (replacing earlier ones) and writes per cluster: member count,
 * max risk, severity histogram [k][5], entity-type bit mask, and the number of distinct relationship codes its edges carry.
 * An original edge counts once for each distinct cluster among its endpoints; relationship code 31 (a string outside the
 * enum) is not counted here.  All pointers are host memory.
 * abb_clusters_fetch_host copies, for the selected clusters in selection order, the member node indices in id-string order
 * (count[c] each) and the (relationship code, edge count) pairs in code order (rel_nnz[c] each). */
int abb_clusters_build_host(abb_graph *g, int64_t k, const int32_t *codes, const uint8_t *level, const double *risk, const uint8_t *etype,
                            int64_t *count_out, double *max_risk_out, int64_t *hist_out, uint64_t *type_mask_out, int64_t *rel_nnz_out);
int abb_clusters_fetch_host(abb_graph *g, int64_t n_sel, const int32_t *sel, int32_t *members_out, uint8_t *rel_out, int64_t *rel_count_out);

/* ---- snapshot diff -------------------------------------------------------------------------------------------
 * Replaces the set arithmetic of diff_snapshots (agent_bom/db/graph_store.py:671-738) and the direction / traversable / weight
 * part of _edge_change_fingerprint (:764-773).  abb_delta_table_host stores a graph's diff tables (replacing earlier ones):
 * the UTF-8 bytes of every node id (ghosts included) with offsets id_off[n_nodes + 1], perm[n_nodes] (sorted position -> node,
 * the inverse of node_rank), per real node the label bytes with offsets label_off[n_real + 1], a status and a severity code
 * (255: a string the host compares itself) and the risk (f64, compared with ==), and per original edge (graph.edges order) a
 * relationship slot (< 64), flags (1 traversable, 2 bidirectional) and optionally the weight (NULL: not compared).
 * abb_delta_build_host diffs two graphs with tables on one device.  relmap_* [64] map each graph's relationship slots to the
 * rank of the relationship string among both graphs' strings.  It fails when the union of both id sets exceeds 2^27 ids (or
 * the graphs' "delta_union_limit" option).  sizes_out[6] = {nodes added, nodes removed, node pairs changed, edges added, edges
 * removed, edge pairs changed}; only real nodes count.  The answer stays on the device in *out, owned by the caller, so diffs
 * may run concurrently on shared graphs.  abb_delta_fetch_host copies it: added nodes (new
 * indices) and removed nodes (old indices) in id order; changed node pairs (new index, old index, flag: 1 changed, 2 equal
 * unless a code-255 string or the OTHER entity type differs) in id order; added / removed edges (edge indices) and changed edge
 * pairs (new edge, old edge) in (source, target, relationship) order.  All pointers are host memory. */
int abb_delta_table_host(abb_graph *g, int32_t n_real, const uint8_t *ids, const int64_t *id_off, const int32_t *perm, const uint8_t *labels,
                         const int64_t *label_off, const uint8_t *status, const uint8_t *severity, const double *risk, int64_t n_edges,
                         const uint8_t *erel, const uint8_t *eflag, const double *weight);
int64_t abb_delta_table_bytes(const abb_graph *g);               /* device bytes of the diff tables, 0 when none */
typedef struct abb_delta_result abb_delta_result;
int abb_delta_build_host(abb_graph *old_g, abb_graph *new_g, const uint8_t *relmap_old, const uint8_t *relmap_new, abb_delta_result **out,
                         int64_t *sizes_out);
void abb_delta_result_free(abb_delta_result *r);
int abb_delta_fetch_host(const abb_delta_result *r, int32_t *nodes_added, int32_t *nodes_removed, int32_t *changed_new, int32_t *changed_old,
                         uint8_t *changed_flag, int32_t *edges_added, int32_t *edges_removed, int32_t *echanged_new, int32_t *echanged_old);
/* Shared edges of a diff (changed_edges_between_scans, :799-841, needs the unchanged ones too): abb_delta_shared_host finds, once per
 * result, the new graph's edges whose (source, target, relationship) key the old graph also has and writes their number to
 * *count_out; abb_delta_shared_fetch_host copies them as (new edge, old edge) index pairs in key order.  Neither changes what
 * abb_delta_fetch_host returns. */
int abb_delta_shared_host(abb_delta_result *r, int64_t *count_out);
int abb_delta_shared_fetch_host(const abb_delta_result *r, int32_t *shared_new, int32_t *shared_old);

/* ---- snapshot lookups -----------------------------------------------------------------------------------------
 * Replace the per-request edge-row scans of edges_for_node_ids, node_context and the unfiltered snapshot_stats
 * (agent_bom/api/graph_store.py:889-948, 1139-1240, 1315-1344).  abb_lookup_table_host stores the graph's lookup table
 * (replacing an earlier one; freed with the graph): erel[n_edges] is, per original edge in graph.edges order (every edge of
 * the graph), the rank (< 64) of its relationship string among the graph's relationship strings.  It also writes the snapshot
 * statistics: type_counts_out[256] counts the real nodes (index < n_real) by entity-type code, sev_counts_out[256] by the
 * caller's severity[n_real] code, and rel_counts_out[64] the original edges whose endpoints are both real nodes by erel.
 * abb_lookup_edges_host finds the original edges with at least one endpoint among nodes[k] (duplicates allowed) and
 * abb_lookup_context_host those of one node, sorted by (rank(source), rank(target), erel); the context needs the lookup table
 * and fails when the graph has more than 2^27 nodes.  Both answers stay on the device in *out, owned by the caller, so lookups
 * may run concurrently on one graph; *count_out is the number of edges.  abb_lookup_fetch_host copies the edge indices (the
 * edge set ascending, the context in its order).  All pointers are host memory. */
int abb_lookup_table_host(abb_graph *g, int32_t n_real, const uint8_t *severity, int64_t n_edges, const uint8_t *erel, int64_t *type_counts_out,
                          int64_t *sev_counts_out, int64_t *rel_counts_out);
int64_t abb_lookup_table_bytes(const abb_graph *g);              /* device bytes of the lookup table, 0 when none */
typedef struct abb_lookup_result abb_lookup_result;
int abb_lookup_edges_host(abb_graph *g, int64_t k, const int32_t *nodes, abb_lookup_result **out, int64_t *count_out);
int abb_lookup_context_host(abb_graph *g, int32_t node, abb_lookup_result **out, int64_t *count_out);
int abb_lookup_fetch_host(const abb_lookup_result *r, int32_t *edges_out);
void abb_lookup_result_free(abb_lookup_result *r);

/* ---- node search ----------------------------------------------------------------------------------------------
 * Replace the per-request FTS5 MATCH / LIKE scan, COUNT(*) and sort of search_nodes and page_nodes
 * (agent_bom/api/graph_store.py:1242-1313, 1346-1468).  The graph's search table (freed with the graph) is built in two calls:
 * abb_search_text_host stores the stored search_text bytes of n nodes (text_off[n+1], int64; an empty row for a node without an
 * index row) and sets, in cp_bits_out[0x110000 / 32], the bit of every code point >= 0x80 the text holds;
 * abb_search_table_host folds the text into token text with fold[0x110000] (per code point: -1 separator, 0 folds away, else the
 * code point it folds to; it must cover ASCII and every code point marked) and stores per node severity_id (INT32_MIN for NULL),
 * risk (NaN for NULL), label rank, entity-type code (< n_types), compliance and data-source codes (< n_cmp / n_src, both -1 for a
 * node without an index row).  Nodes are in id order: a node's index is its id rank.
 * abb_search_host runs one call: mode 0 matches every node (page_nodes), mode 1 the nodes whose token text holds every pattern
 * at a token start (FTS phrases: folded tokens joined by one space, none empty), mode 2 those whose raw text holds the one
 * pattern (LIKE).  type_ok / cmp_ok / src_ok (NULL: off) are byte tables indexed by code; use_min_rank keeps severity_id >=
 * min_rank.  *total_out counts the matches, *selected_out those that also pass the cursor (severity_id < cur_sev OR (= AND risk <
 * cur_risk) OR (= AND = AND label rank >= cur_label_gt) OR (= AND = AND label rank == cur_label_eq AND node >= cur_id_gt), a
 * NULL severity never passing and a NULL risk, or cur_risk_null, passing only through the first clause).  The page, positions
 * [offset, offset + take) of the selection in (severity desc, risk desc, label, id) order with NULLs last, stays on the device
 * in *out, owned by the caller; *count_out is its length and abb_search_fetch_host copies it.  All pointers are host memory. */
typedef struct abb_search_spec {
    int32_t mode, n_patterns;
    const uint8_t *patterns;           /* pattern bytes */
    const int64_t *pattern_off;        /* [n_patterns + 1] */
    const uint8_t *type_ok, *cmp_ok, *src_ok;
    int32_t n_types, n_cmp, n_src;     /* lengths of the tables given; must equal the search table's */
    int32_t use_min_rank;
    int64_t min_rank;
    int32_t has_cursor, cur_risk_null;
    int64_t cur_sev;
    double cur_risk;
    int64_t cur_label_gt, cur_label_eq, cur_id_gt;
    int64_t offset, take;
} abb_search_spec;
int abb_search_text_host(abb_graph *g, int32_t n, const int64_t *text_off, const uint8_t *text, uint32_t *cp_bits_out);
int abb_search_table_host(abb_graph *g, const int32_t *fold, const int32_t *severity, const double *risk, const uint32_t *label_rank,
                          const int32_t *type_code, const int32_t *cmp_code, const int32_t *src_code, int32_t n_types, int32_t n_cmp, int32_t n_src);
int64_t abb_search_table_bytes(const abb_graph *g);              /* device bytes of the search table, 0 when none */
typedef struct abb_search_result abb_search_result;
int abb_search_host(abb_graph *g, const abb_search_spec *spec, abb_search_result **out, int64_t *total_out, int64_t *selected_out, int64_t *count_out);
int abb_search_fetch_host(const abb_search_result *r, int32_t *nodes_out);
void abb_search_result_free(abb_search_result *r);

/* ---- compliance posture ---------------------------------------------------------------------------------------
 * Replace the per-request decode and Python loop over every (node, tag) pair of compliance_summary
 * (agent_bom/api/graph_store.py:950-1031).  abb_compliance_table_host builds the graph's compliance table (freed with the graph,
 * replacing an earlier one) from n tagged rows in id order: per row a text code (< n_texts), severity code (< n_sev) and
 * entity-type code (< n_types); per text its tag codes text_tags[text_off[t] .. text_off[t+1]) (int64 offsets, repeats kept);
 * per tag its framework code tag_fw[tag] (< n_fw).  Tags and frameworks are coded in the order their names sort.  It rolls up
 * every (row, tag) pair and sets sizes_out[4]: the number of (framework, severity) runs, (framework, type) runs, distinct
 * (framework, tag) pairs and node ids.  abb_compliance_fetch_host copies the table: each run array is [4][runs] int64 (framework,
 * code, pairs, first row) in (framework, code) order; node_count[n_fw] the distinct rows per framework; node_rows the first 100
 * of them per framework in row order, frameworks in order.  All pointers are host memory. */
int abb_compliance_table_host(abb_graph *g, int32_t n, const int32_t *row_text, const int32_t *row_sev, const int32_t *row_type, int32_t n_texts,
                              const int64_t *text_off, const int32_t *text_tags, int32_t n_tags, const int32_t *tag_fw, int32_t n_fw, int32_t n_sev,
                              int32_t n_types, int64_t *sizes_out);
int64_t abb_compliance_table_bytes(const abb_graph *g);          /* device bytes of the compliance table, 0 when none */
int abb_compliance_fetch_host(abb_graph *g, int64_t *sev_runs, int64_t *type_runs, int64_t *tag_runs, int64_t *node_count, int32_t *node_rows);

/* ---- edge lifecycle: versions active at a timestamp -------------------------------------------------------------
 * Replaces the row-dict build and keyed selection of active_edges_at (agent_bom/db/graph_store.py:775-796).
 * abb_lifecycle_build_host builds one tenant's edge history on `device`: per stored edge row, in (created_at, scan_id) order,
 * the ranks of its source and target id (< n_ids) and relationship (< n_rels) in sorted dictionaries, and the ranks of its
 * snapshot's created_at, its effective valid_from and its valid_to in one sorted dictionary of timestamp strings (0x7FFFFFFF:
 * absent; an absent valid_from is never <= at, an absent valid_to is open).  It fails when n_ids exceeds id_limit (at most
 * 2^27) or n_rels exceeds 2^10.  The history is owned by the caller (abb_lifecycle_free) and *n_seg_out receives its number of
 * distinct keys.  abb_lifecycle_active_host takes r, the number of dictionary strings <= at, and writes to rows_out (room for
 * n_seg entries) the row index of the last version of each key whose created_at and valid_from are <= at and whose valid_to is
 * > at, in (source, target, relationship) order; *count_out receives their number and ms_out (optional) the device time.
 * Calls on one history are serialised.  All pointers are host memory. */
typedef struct abb_lifecycle_history abb_lifecycle_history;
int abb_lifecycle_build_host(int device, int64_t n_rows, const int32_t *src, const int32_t *tgt, const int32_t *rel, const int32_t *created,
                             const int32_t *valid_from, const int32_t *valid_to, int64_t n_ids, int64_t n_rels, int64_t id_limit,
                             abb_lifecycle_history **out, int64_t *n_seg_out);
int abb_lifecycle_active_host(abb_lifecycle_history *h, int32_t r, int32_t *rows_out, int64_t *count_out, float *ms_out);
int64_t abb_lifecycle_bytes(const abb_lifecycle_history *h);      /* device bytes of the history and its workspace */
void abb_lifecycle_free(abb_lifecycle_history *h);

/* ---- multi-hop blast-radius expansion --------------------------------------------------------------------------
 * Replaces the per-blast-radius BFS of expand_blast_radius_hops (agent_bom/scanners/blast_radius.py:16-97).  Inputs, all host
 * memory with int64 offsets: name -> servers (name_srv_off[n_names + 1], name_srv; the last agent object of a name), server ->
 * agent occurrences (srv_occ_off[n_servers + 1]; per occurrence its name and credential set), credential sets (cset_off,
 * cset_cred), and per signature the agent names and servers to mark visited and the first-level queue's servers (first_off,
 * first_srv; global entry id = list position).  max_depth is the clamped depth, 2..5.  `batch` > 0 caps how many signatures
 * are searched at once (0: as many as a quarter of free device memory allows).  The result (abb_hops_result_free) holds:
 *   counts: {discoveries, entries of levels >= 2, credential keys, batches, batch size}; times: {upload, search, readback} ms;
 *   per discovery, in (batch, level, signature, queue) order: signature, occurrence, hop and parent entry id;
 *   per later entry, in the same order (global ids n_first, n_first + 1, ...): server and parent discovery id;
 *   the sorted unique (signature << 32 | credential id) keys. */
typedef struct abb_hops_result abb_hops_result;
int abb_hops_host(int device, int32_t max_depth, int32_t n_names, const int64_t *name_srv_off, const int32_t *name_srv, int32_t n_servers,
                  const int64_t *srv_occ_off, const int32_t *occ_name, const int32_t *occ_cset, int32_t n_csets, const int64_t *cset_off,
                  const int32_t *cset_cred, int64_t n_sigs, const int64_t *mark_agent_off, const int32_t *mark_agent, const int64_t *mark_srv_off,
                  const int32_t *mark_srv, const int64_t *first_off, const int32_t *first_srv, int64_t batch, abb_hops_result **out);
void abb_hops_result_counts(const abb_hops_result *r, int64_t *out);
void abb_hops_result_times(const abb_hops_result *r, double *out);
const int32_t *abb_hops_result_disc_sig(const abb_hops_result *r);
const int32_t *abb_hops_result_disc_occ(const abb_hops_result *r);
const int32_t *abb_hops_result_disc_hop(const abb_hops_result *r);
const int64_t *abb_hops_result_disc_parent(const abb_hops_result *r);
const int32_t *abb_hops_result_entry_server(const abb_hops_result *r);
const int64_t *abb_hops_result_entry_parent(const abb_hops_result *r);
const unsigned long long *abb_hops_result_cred(const abb_hops_result *r);
void abb_hops_result_free(abb_hops_result *r);

#ifdef __cplusplus
}
#endif
#endif /* ABB200_H */
