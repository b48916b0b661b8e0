// lateral.cuh — capped simple-path search behind find_lateral_paths (sm_90a).
//
// Reference: agent_bom/context_graph.py:397-477.  From a source node a FIFO of *paths* is expanded over the mirrored
// adjacency; a path whose end is a "lateral target" (an agent other than the source's, or a credential / tool owned by
// another agent) is recorded and not extended — unless the same node sequence was recorded already (it can arrive
// twice through parallel edges of different kinds), in which case it IS extended.  The search stops at 100 recorded
// paths or an empty queue; a popped path is not extended while 10 000 or more paths wait in the queue, and paths longer
// than max_depth+1 nodes are dropped.  All of that is order-sensitive, so one warp replays the reference's queue
// exactly for one source: the pop is serial, the expansion of the popped node's adjacency row is lane-parallel with a
// ballot / prefix append that keeps adjacency order.  Sources (the CLI and the REST route call this for every agent)
// are the data-parallel axis: one warp each, a private ring of path records in global memory.
//
// Record layout (int32 words): [0] length, [1] edge kinds (4 bits per hop), [2 .. 2+W) node ids; W = max_depth + 2.
#pragma once
#include <cstdint>

namespace abb {

constexpr int LAT_MAX_PATHS = 100;      // _MAX_PATHS
constexpr int LAT_MAX_QUEUE = 10000;    // _MAX_QUEUE_SIZE
constexpr int LAT_MAX_W = 9;            // max_depth <= 7: 8 hops x 4 bits of edge kind fit one word
constexpr uint8_t LAT_KIND_AGENT = 0, LAT_KIND_CRED = 2, LAT_KIND_TOOL = 3, LAT_KIND_GHOST = 255;

struct LateralArgs {
    int32_t n;                   // nodes
    const int64_t *off;          // [n+1] adjacency rows (graph.adjacency[id], list order)
    const int32_t *nbr;          // entry target
    const uint8_t *ekind;        // entry edge kind (0..15)
    const uint8_t *nkind;        // node kind; 255 = id without a node record
    const int32_t *nkey;         // agents: id of the label; credentials / tools: id of metadata["agent"]; -1 = absent or empty
    int64_t n_sources;
    const int32_t *src;          // source node per search (-1: not in graph.nodes -> no paths)
    const int32_t *src_key;      // id of the source's agent name ("" has an id of its own)
    int32_t max_depth;
    int32_t W;                   // node slots per record
    int32_t ring_cap;            // records per ring (> LAT_MAX_QUEUE + longest row)
    int32_t *ring;               // [n_warps][ring_cap][W+2]
    long long max_pops;          // safety valve per source; exceeding it sets the overflow flag instead of running on
    int32_t *out_count;          // [n_sources]
    int32_t *out_paths;          // [n_sources][LAT_MAX_PATHS][W+2]
    int32_t *out_flags;          // [n_sources] bit0 = safety valve hit
};

__global__ void __launch_bounds__(128) lateral_search_kernel(LateralArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int R = A.W + 2;
    int32_t *ring = A.ring + warp * static_cast<int64_t>(A.ring_cap) * R;
    for (int64_t q = warp; q < A.n_sources; q += nwarps) {
        int32_t *found = A.out_paths + q * static_cast<int64_t>(LAT_MAX_PATHS) * R;
        const int32_t s = A.src[q];
        int npaths = 0, flags = 0;
        if (s >= 0 && s < A.n && A.nkind[s] != LAT_KIND_GHOST) {
            const int32_t skey = A.src_key[q];
            int head = 0, count = 1;
            if (lane == 0) { ring[0] = 1; ring[1] = 0; ring[2] = s; }
            __syncwarp();
            long long pops = 0;
            // every quantity that steers control flow below is read from the same record by all lanes: the warp never diverges
            while (count > 0 && npaths < LAT_MAX_PATHS) {
                if (++pops > A.max_pops) { flags |= 1; break; }
                const int32_t *e = ring + static_cast<int64_t>(head) * R;
                const int len = e[0];
                const uint32_t kinds = static_cast<uint32_t>(e[1]);
                int32_t pn[LAT_MAX_W];                               // the popped path, whole, in every lane (broadcast loads)
#pragma unroll
                for (int k = 0; k < LAT_MAX_W; k++) pn[k] = k < len ? e[2 + k] : -1;
                head = head + 1 == A.ring_cap ? 0 : head + 1;
                count--;
                if (len > A.max_depth + 1) continue;
                const int32_t cur = e[2 + len - 1];
                if (len > 1) {
                    const uint8_t ck = A.nkind[cur];
                    const int32_t key = A.nkey[cur];
                    bool lateral = false;
                    if (ck == LAT_KIND_AGENT) lateral = key != skey;
                    else if (ck == LAT_KIND_CRED || ck == LAT_KIND_TOOL) lateral = key >= 0 && key != skey;
                    if (lateral) {
                        bool dup = false;                               // same node sequence recorded before?
                        for (int base = 0; base < npaths; base += 32) {
                            const int i = base + lane;
                            bool same = false;
                            if (i < npaths) {
                                const int32_t *f = found + static_cast<int64_t>(i) * R;
                                same = f[0] == len;
#pragma unroll
                                for (int k = 0; k < LAT_MAX_W; k++) if (k < len) same = same && f[2 + k] == pn[k];
                            }
                            dup = dup || __any_sync(0xFFFFFFFFu, same);
                        }
                        if (!dup) {
                            int32_t *f = found + static_cast<int64_t>(npaths) * R;
                            if (lane == 0) {
                                f[0] = len; f[1] = static_cast<int32_t>(kinds);
#pragma unroll
                                for (int k = 0; k < LAT_MAX_W; k++) if (k < A.W) f[2 + k] = pn[k];
                            }
                            npaths++;
                            __syncwarp();
                            continue;                                   // a recorded target is not extended
                        }
                    }
                }
                if (count >= LAT_MAX_QUEUE) continue;                   // len(queue) after the pop
                const int64_t a = A.off[cur], b = A.off[cur + 1];
                for (int64_t p0 = a; p0 < b; p0 += 32) {
                    const int64_t p = p0 + lane;
                    int32_t nb = -1; uint32_t ek = 0;
                    bool ok = p < b;
                    if (ok) { nb = A.nbr[p]; ek = A.ekind[p]; }
#pragma unroll
                    for (int k = 0; k < LAT_MAX_W; k++) if (k < len) ok = ok && nb != pn[k];
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                    if (ok) {
                        int slot = head + count + __popc(m & ((1u << lane) - 1u));
                        if (slot >= A.ring_cap) slot -= A.ring_cap;
                        int32_t *w = ring + static_cast<int64_t>(slot) * R;
                        w[0] = len + 1;
                        w[1] = static_cast<int32_t>(kinds | (ek << (4 * (len - 1))));
#pragma unroll
                        for (int k = 0; k < LAT_MAX_W; k++) if (k < len) w[2 + k] = pn[k];
                        w[2 + len] = nb;
                    }
                    count += __popc(m);
                }
                __syncwarp();
            }
        }
        if (lane == 0) { A.out_count[q] = npaths; A.out_flags[q] = flags; }
        __syncwarp();
    }
}

// ---- enrichment of found paths (reference: context_graph.py:495-572) -------------------------------------------------------
// Per path the reference builds three first-seen-ordered label lists (credentials, tools, vulnerabilities), counts the
// execute-capable tools and keeps the highest severity score, both judged on the node that first adds a label.  Its item
// stream is: each hop in order (credential / tool / vulnerability nodes add themselves, a server adds its surface), then each
// sharing hop in edge order (shares_server adds the surface of every server carrying the link's server name, shares_credential
// adds the link's credential name).  Surfaces are precomputed and de-duplicated once per server and once per shared name.
//   plan:   one warp per path resolves its pieces (a node, a surface, a credential name) and counts its items;
//   emit:   items as keys path << 32 | category << 30 | label, with their stream position as the sort value;
//   a stable radix sort by key puts each (path, category, label) run in stream order: the run head is the first add;
//   reduce: per path, over its kept items in stream order: credentials, execute tools, highest severity, error flag.
// No array is sized paths x labels: everything is sized by the number of items the paths' streams hold.
constexpr int LAT_PIECES = 2 * LAT_MAX_W;                              // one per hop and one per sharing hop
constexpr uint32_t LAT_PIECE_SURF = 1u, LAT_PIECE_NODE = 2u, LAT_PIECE_CRED = 3u;   // piece word: type << 30 | payload
constexpr uint8_t LAT_KIND_SERVER = 1, LAT_KIND_VULN = 4;
constexpr int LAT_CAT_CRED = 0, LAT_CAT_TOOL = 1, LAT_CAT_VULN = 2;   // category << 30 | label

struct EnrichArgs {
    int32_t n;                   // nodes
    const int64_t *off;          // adjacency rows, as for the search
    const int32_t *nbr;
    const uint8_t *ekind;
    const int32_t *ename;        // per entry: shares_server -> surface of its server name, shares_credential -> credential label; -1 none
    int32_t code_ss, code_sc;    // edge-kind codes of shares_server / shares_credential (-1: absent)
    const uint8_t *nkind;        // node kind, as for the search
    const int32_t *nlabel;       // credential / tool / vulnerability nodes: label id in its category
    const float *nval;           // tools: 1 execute, 0 not, -1 the test raised; vulnerabilities: severity score, -1 the lookup raised
    const int32_t *nsurf;        // server nodes: their surface, -1 when empty
    const int64_t *surf_off;     // [n_surfaces+1]
    const int32_t *surf_node;    // surface items: the node that first adds each label of the surface, in surface order
    int64_t n_paths;
    int32_t R;                   // words per record (W + 2)
    const int32_t *rec;          // [n_paths][R] search records
    uint32_t *pieces;            // [n_paths][LAT_PIECES]
    int64_t *count;              // [n_paths+1] items per path, scanned into item_off
    const int64_t *item_off;     // [n_paths+1]
    unsigned long long *keys;    // [items]
    int32_t *pos;                // [items] stream position (sort value)
    int32_t *item;               // [items] category << 30 | label
    int32_t *inode;              // [items] node that adds it, -1 for a credential name
};

__device__ __forceinline__ int lat_category(uint8_t kind) { return kind == LAT_KIND_CRED ? LAT_CAT_CRED : kind == LAT_KIND_TOOL ? LAT_CAT_TOOL : LAT_CAT_VULN; }

__global__ void __launch_bounds__(128) lateral_enrich_plan_kernel(EnrichArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t path = warp; path < A.n_paths; path += nwarps) {
        const int32_t *r = A.rec + path * A.R;
        const int len = r[0];
        const uint32_t kinds = static_cast<uint32_t>(r[1]);
        uint32_t *pc = A.pieces + path * LAT_PIECES;
        int np = 0;
        int64_t cnt = 0;
        for (int h = 0; h < len; h++) {                                // every lane walks the same hops: no divergence
            const int32_t v = r[2 + h];
            const uint8_t k = A.nkind[v];
            if (k == LAT_KIND_SERVER) {
                const int32_t s = A.nsurf[v];
                if (s >= 0) {
                    if (lane == 0) pc[np] = LAT_PIECE_SURF << 30 | static_cast<uint32_t>(s);
                    np++;
                    cnt += A.surf_off[s + 1] - A.surf_off[s];
                }
            } else if (k == LAT_KIND_CRED || k == LAT_KIND_TOOL || k == LAT_KIND_VULN) {
                if (lane == 0) pc[np] = LAT_PIECE_NODE << 30 | static_cast<uint32_t>(v);
                np++;
                cnt++;
            }
        }
        for (int i = 0; i + 1 < len; i++) {
            const int32_t ek = static_cast<int32_t>((kinds >> (4 * i)) & 15u);
            if (ek != A.code_ss && ek != A.code_sc) continue;
            const int32_t u = r[2 + i], w = r[3 + i];
            const int64_t a = A.off[u], b = A.off[u + 1];
            int64_t first = -1;
            for (int64_t p0 = a; p0 < b; p0 += 32) {                     // the first entry u -> w of that kind
                const int64_t p = p0 + lane;
                const unsigned m = __ballot_sync(0xFFFFFFFFu, p < b && A.nbr[p] == w && A.ekind[p] == ek);
                if (m) { first = p0 + __ffs(m) - 1; break; }
            }
            const int32_t name = first >= 0 ? A.ename[first] : -1;
            if (name < 0) continue;
            if (ek == A.code_ss) {
                if (lane == 0) pc[np] = LAT_PIECE_SURF << 30 | static_cast<uint32_t>(name);
                cnt += A.surf_off[name + 1] - A.surf_off[name];
            } else {
                if (lane == 0) pc[np] = LAT_PIECE_CRED << 30 | static_cast<uint32_t>(name);
                cnt++;
            }
            np++;
        }
        if (lane == 0) {
            for (int k = np; k < LAT_PIECES; k++) pc[k] = 0;
            A.count[path] = cnt;
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(128) lateral_enrich_emit_kernel(EnrichArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t path = warp; path < A.n_paths; path += nwarps) {
        const uint32_t *pc = A.pieces + path * LAT_PIECES;
        const unsigned long long hi = static_cast<unsigned long long>(path) << 32;
        int64_t at = A.item_off[path];
        for (int k = 0; k < LAT_PIECES; k++) {
            const uint32_t piece = pc[k];
            const uint32_t type = piece >> 30, payload = piece & 0x3FFFFFFFu;
            if (type == 0) break;
            if (type == LAT_PIECE_SURF) {
                const int64_t a = A.surf_off[payload], b = A.surf_off[payload + 1];
                for (int64_t j = a + lane; j < b; j += 32) {
                    const int32_t v = A.surf_node[j];
                    const uint32_t it = static_cast<uint32_t>(lat_category(A.nkind[v])) << 30 | static_cast<uint32_t>(A.nlabel[v]);
                    const int64_t o = at + (j - a);
                    A.keys[o] = hi | it; A.pos[o] = static_cast<int32_t>(o); A.item[o] = static_cast<int32_t>(it); A.inode[o] = v;
                }
                at += b - a;
            } else {
                if (lane == 0) {
                    const int32_t v = type == LAT_PIECE_NODE ? static_cast<int32_t>(payload) : -1;
                    const uint32_t it = type == LAT_PIECE_NODE ? static_cast<uint32_t>(lat_category(A.nkind[v])) << 30 | static_cast<uint32_t>(A.nlabel[v])
                                                               : static_cast<uint32_t>(LAT_CAT_CRED) << 30 | payload;
                    A.keys[at] = hi | it; A.pos[at] = static_cast<int32_t>(at); A.item[at] = static_cast<int32_t>(it); A.inode[at] = v;
                }
                at++;
            }
        }
    }
}

// keep[stream position] = 1 for the first item of each (path, category, label) run of the stably sorted keys
__global__ void lateral_enrich_heads_kernel(int64_t m, const unsigned long long *sorted, const int32_t *pos, uint8_t *keep) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < m; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        keep[pos[i]] = i == 0 || sorted[i] != sorted[i - 1];
}

// per path over its kept items: how many, execute-capable tools, highest severity, bit0 = a first add whose value raised
__global__ void __launch_bounds__(128) lateral_enrich_reduce_kernel(int64_t n_paths, const int64_t *item_off, const uint8_t *keep, const int32_t *item,
                                                                    const int32_t *inode, const float *nval, int32_t *n_kept, int32_t *n_exec, float *sev,
                                                                    int32_t *flags) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t path = warp; path < n_paths; path += nwarps) {
        int kept = 0, ex = 0, err = 0;
        float s = 0.f;
        for (int64_t i = item_off[path] + lane; i < item_off[path + 1]; i += 32) {
            if (!keep[i]) continue;
            kept++;
            const int cat = static_cast<int>(static_cast<uint32_t>(item[i]) >> 30);
            if (cat == LAT_CAT_CRED) continue;
            const float v = nval[inode[i]];
            if (v < 0.f) err = 1;
            else if (cat == LAT_CAT_TOOL) ex += v > 0.f;
            else s = fmaxf(s, v);
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) {
            kept += __shfl_xor_sync(0xFFFFFFFFu, kept, d);
            ex += __shfl_xor_sync(0xFFFFFFFFu, ex, d);
            err |= __shfl_xor_sync(0xFFFFFFFFu, err, d);
            s = fmaxf(s, __shfl_xor_sync(0xFFFFFFFFu, s, d));
        }
        if (lane == 0) { n_kept[path] = kept; n_exec[path] = ex; sev[path] = s; flags[path] = err; }
    }
}

}  // namespace abb
