// lookup.cuh — per-request lookups over a cached snapshot (sm_90a).
//
// Reference: the SQLite store's edges_for_node_ids, node_context and snapshot_stats (api/graph_store.py:889-948, 1139-1240,
// 1315-1344), which each read every edge row of the scan.  Here:
//   - incident edges of a node set: one thread per incident row entry.  An exclusive scan over the members' forward + reverse
//     row lengths gives each entry a global position; a thread binary-searches that position back to its member.  An entry
//     whose reversed bit is clear names an original edge (forward entry at its source, reverse entry at its target); its bit
//     is set in an edge bitmap, so self loops and edges with both endpoints in the set count once.  The bitmap is compacted
//     in edge-id order (= load order = rowid order) with a popcount scan;
//   - one node's context order: the same entries of one node, each original edge emitted once (a self loop is taken from the
//     forward row only) as the key rank(src) << 33 | rank(tgt) << 6 | relrank and radix-sorted.  relrank is the rank of the
//     edge's relationship string among the graph's strings; UTF-8 byte order is SQLite's BINARY collation, so ascending keys
//     are ORDER BY source_id, target_id, relationship;
//   - snapshot statistics: a warp-aggregated histogram of the real nodes' entity-type and severity codes and of the
//     relationship slots of original edges whose endpoints are both real nodes.
#pragma once
#include <cstdint>

namespace abb {

constexpr int LK_REL_SLOTS = 64;                // relationship strings per graph (relrank has 6 bits)
constexpr int64_t LK_RANK_LIMIT = 1ll << 27;    // node ranks in the context key (27 bits each)

// original edges: forward entries whose reversed bit is clear (one per edge)
__global__ void lookup_count_edges_kernel(int64_t m, const uint8_t *__restrict__ fmeta, unsigned long long *__restrict__ count) {
    unsigned long long mine = 0;
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; p < m; p += static_cast<int64_t>(gridDim.x) * blockDim.x)
        mine += !(fmeta[p] & 0x80u);
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(count, mine);
}

// entries of member i: forward row, then reverse row
__global__ void lookup_len_kernel(int64_t k, const int32_t *__restrict__ nodes, const uint32_t *__restrict__ foff, const uint32_t *__restrict__ roff,
                                  int64_t *__restrict__ len) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < k; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t u = nodes[i];
        len[i] = static_cast<int64_t>(foff[u + 1] - foff[u]) + static_cast<int64_t>(roff[u + 1] - roff[u]);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) len[k] = 0;
}

// member of global entry position t: last i with start[i] <= t
__device__ __forceinline__ int64_t lookup_member(const int64_t *__restrict__ start, int64_t k, int64_t t) {
    int64_t lo = 0, hi = k - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (start[mid] <= t) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void lookup_mark_kernel(int64_t total, int64_t k, const int32_t *__restrict__ nodes, const int64_t *__restrict__ start, GraphView g,
                                   uint32_t *__restrict__ ebits) {
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t i = lookup_member(start, k, t);
        const int32_t u = nodes[i];
        const int64_t local = t - start[i];
        const int64_t flen = g.foff[u + 1] - g.foff[u];
        uint8_t meta; uint32_t eid2;
        if (local < flen) {
            const uint32_t p = g.foff[u] + static_cast<uint32_t>(local);
            meta = g.fmeta[p]; eid2 = g.feid[p];
        } else {
            const uint32_t p = g.roff[u] + static_cast<uint32_t>(local - flen);
            meta = g.rmeta[p]; eid2 = g.reid[p];
        }
        if (meta & 0x80u) continue;           // reversed copy of a bidirectional edge: its original entry is also incident
        const uint32_t e = eid2 >> 1;
        atomicOr(ebits + (e >> 5), 1u << (e & 31));
    }
}

__global__ void lookup_popc_kernel(int64_t words, const uint32_t *__restrict__ ebits, int64_t *__restrict__ cnt) {
    for (int64_t w = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; w <= words; w += static_cast<int64_t>(gridDim.x) * blockDim.x)
        cnt[w] = w < words ? __popc(ebits[w]) : 0;
}

__global__ void lookup_compact_kernel(int64_t words, const uint32_t *__restrict__ ebits, const int64_t *__restrict__ off, int32_t *__restrict__ out) {
    for (int64_t w = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; w < words; w += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        uint32_t b = ebits[w];
        int64_t o = off[w];
        while (b) {
            const int bit = __ffs(b) - 1;
            out[o++] = static_cast<int32_t>((w << 5) + bit);
            b &= b - 1;
        }
    }
}

// node u's original incident edges as (key, edge) pairs at slots taken from *count
__global__ void lookup_context_keys_kernel(int32_t u, GraphView g, const uint8_t *__restrict__ erel, unsigned long long *__restrict__ keys,
                                           int32_t *__restrict__ vals, unsigned int *__restrict__ count) {
    const int64_t flen = g.foff[u + 1] - g.foff[u];
    const int64_t total = flen + (g.roff[u + 1] - g.roff[u]);
    for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        uint8_t meta; uint32_t eid2; int32_t s, d;
        if (t < flen) {
            const uint32_t p = g.foff[u] + static_cast<uint32_t>(t);
            meta = g.fmeta[p]; eid2 = g.feid[p]; s = u; d = g.fnbr[p];
        } else {
            const uint32_t p = g.roff[u] + static_cast<uint32_t>(t - flen);
            meta = g.rmeta[p]; eid2 = g.reid[p]; s = g.rnbr[p]; d = u;
            if (s == u) continue;             // a self loop: already emitted from the forward row
        }
        if (meta & 0x80u) continue;
        const uint32_t e = eid2 >> 1;
        const unsigned int slot = atomicAdd(count, 1u);
        keys[slot] = (static_cast<unsigned long long>(g.rank[s]) << 33) | (static_cast<unsigned long long>(g.rank[d]) << 6) | erel[e];
        vals[slot] = static_cast<int32_t>(e);
    }
}

// add one to hist[code], one atomic per distinct code in the warp
__device__ __forceinline__ void lookup_warp_count(unsigned int *hist, unsigned active, int code) {
    const unsigned peers = __match_any_sync(active, code);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(hist + code, static_cast<unsigned int>(__popc(peers)));
}

// type [256] and severity [256] codes of the real nodes, relationship slots [64] of original edges between real nodes
__global__ void lookup_stats_kernel(int32_t n_real, const uint8_t *__restrict__ sev, GraphView g, const uint8_t *__restrict__ erel,
                                    unsigned long long *__restrict__ type_out, unsigned long long *__restrict__ sev_out,
                                    unsigned long long *__restrict__ rel_out) {
    __shared__ unsigned int h_type[256], h_sev[256], h_rel[LK_REL_SLOTS];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) { h_type[i] = 0; h_sev[i] = 0; if (i < LK_REL_SLOTS) h_rel[i] = 0; }
    __syncthreads();
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    // whole warps step together so every lane of an active warp reaches __match_any_sync
    for (int64_t i0 = base - (threadIdx.x & 31); i0 < n_real; i0 += stride) {
        const int64_t i = i0 + (threadIdx.x & 31);
        const unsigned active = __ballot_sync(0xFFFFFFFFu, i < n_real);
        if (i < n_real) {
            lookup_warp_count(h_type, active, g.ntype[i]);
            lookup_warp_count(h_sev, active, sev[i]);
        }
    }
    for (int64_t p0 = base - (threadIdx.x & 31); p0 < g.m; p0 += stride) {
        const int64_t p = p0 + (threadIdx.x & 31);
        bool take = false;
        int code = 0;
        if (p < g.m && !(g.fmeta[p] & 0x80u)) {
            const int32_t u = row_of_entry(g.foff, g.n, static_cast<uint32_t>(p));
            take = u < n_real && g.fnbr[p] < n_real;
            code = erel[g.feid[p] >> 1];
        }
        const unsigned active = __ballot_sync(0xFFFFFFFFu, take);
        if (take) lookup_warp_count(h_rel, active, code);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        if (h_type[i]) atomicAdd(type_out + i, static_cast<unsigned long long>(h_type[i]));
        if (h_sev[i]) atomicAdd(sev_out + i, static_cast<unsigned long long>(h_sev[i]));
        if (i < LK_REL_SLOTS && h_rel[i]) atomicAdd(rel_out + i, static_cast<unsigned long long>(h_rel[i]));
    }
}

}  // namespace abb
