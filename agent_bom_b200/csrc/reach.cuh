// reach.cuh — pass 2 of compute_dependency_reach (graph/dependency_reach.py:132-164) on the device.
//
// Pass 1 is a walk from every agent (abb_spec_distances_along) that keeps only
// package nodes and their hop counts.  The kernels here invert that
// (agent -> packages) relation into (package -> sorted agents, min hops) and
// roll it up per vulnerability, using 64-bit (group << 32 | rank) keys so one
// stable radix sort yields the reference's `tuple(sorted(...))` orders.
#pragma once
#include "walk.cuh"

namespace abb {

constexpr int ET_PACKAGE = 2;

// q_count widened to int64 plus one trailing zero: the input of the exclusive scan that gives every query its output range
__global__ void reach_qcount_kernel(int64_t nq, const int32_t *q_count, int64_t *out) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i <= nq) out[i] = i < nq ? q_count[i] : 0;
}

// one thread per emitted (agent q, package) pair of pass 1.
// A de-duplicated walk points every member of a frontier group at the group's one slice, so the slice at q_start[q] may be
// shared by several queries: outputs are indexed by qoff (exclusive scan of q_count), not q_start.
__global__ void reach_invert_kernel(int64_t nq, const int32_t *agents, const int64_t *q_start, const int32_t *q_count, const int64_t *qoff,
                                    const int32_t *nodes, const int32_t *depth, const int32_t *rank, unsigned long long *keys, int32_t *vals,
                                    unsigned long long *cnt, int32_t *minhop) {
    // a warp per query keeps the slice reads coalesced
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t q = warp; q < nq; q += nwarps) {
        const int64_t s = q_start[q], w = qoff[q];
        const int c = q_count[q];
        const int32_t a = agents[q];
        const unsigned long long ar = static_cast<uint32_t>(rank[a]);
        for (int i = lane; i < c; i += 32) {
            int32_t pkg = nodes[s + i];
            keys[w + i] = (static_cast<unsigned long long>(static_cast<uint32_t>(pkg)) << 32) | ar;
            vals[w + i] = a;
            atomicAdd(cnt + pkg, 1ull);
            atomicMin(minhop + pkg, depth[s + i]);
        }
    }
}

// packages attached to a vulnerability: affects / vulnerable_to in adjacency OR reverse_adjacency,
// other endpoint must be a PACKAGE (dependency_reach.py:201-220).  COUNT pass then FILL pass.
template <bool FILL>
__global__ void reach_vuln_pkgs_kernel(GraphView g, int64_t nv, const int32_t *vulns, uint32_t mask, const int64_t *off, int64_t *counts,
                                       unsigned long long *keys, int32_t *vals) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    const int32_t v = vulns[i];
    int64_t n = 0, w = FILL ? off[i] : 0;
    for (int pass = 0; pass < 2; pass++) {
        const uint32_t *o = pass ? g.roff : g.foff; const int32_t *nb = pass ? g.rnbr : g.fnbr; const uint8_t *me = pass ? g.rmeta : g.fmeta;
        for (uint32_t p = o[v]; p < o[v + 1]; p++) {
            if (!((mask >> (me[p] & ABB_META_REL_MASK)) & 1u)) continue;
            int32_t u = nb[p];
            if (g.ntype[u] != ET_PACKAGE) continue;
            if (FILL) {
                keys[w + n] = (static_cast<unsigned long long>(static_cast<uint32_t>(i)) << 32) | static_cast<uint32_t>(g.rank[u]);
                vals[w + n] = u;
            }
            n++;
        }
    }
    if (!FILL) counts[i] = n;
}

// per unique (vuln slot, package) pair: number of agents reaching the package (+ min-hop roll-up)
__global__ void reach_pair_counts_kernel(int64_t np, const unsigned long long *pair_keys, const int32_t *pair_pkg, const unsigned long long *pkg_cnt,
                                         const int32_t *pkg_minhop, int64_t *counts, int32_t *vmin) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= np) return;
    const int32_t pkg = pair_pkg[i];
    const unsigned long long c = pkg_cnt[pkg];
    counts[i] = static_cast<int64_t>(c);
    if (c) atomicMin(vmin + static_cast<uint32_t>(pair_keys[i] >> 32), pkg_minhop[pkg]);
}

__global__ void reach_pair_fill_kernel(int64_t np, const unsigned long long *pair_keys, const int32_t *pair_pkg, const int64_t *pair_off,
                                       const int64_t *pkg_off, const int32_t *pkg_agents, const int32_t *rank, unsigned long long *keys, int32_t *vals) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t i = warp; i < np; i += nwarps) {
        const int32_t pkg = pair_pkg[i];
        const int64_t a0 = pkg_off[pkg], a1 = pkg_off[pkg + 1], w = pair_off[i];
        const unsigned long long hi = pair_keys[i] & 0xFFFFFFFF00000000ull;
        for (int64_t k = lane; k < a1 - a0; k += 32) {
            int32_t a = pkg_agents[a0 + k];
            keys[w + k] = hi | static_cast<uint32_t>(rank[a]);
            vals[w + k] = a;
        }
    }
}

// histogram of the high 32 bits of sorted unique keys -> per-group counts
__global__ void reach_group_counts_kernel(int64_t n, const unsigned long long *keys, unsigned long long *cnt) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(cnt + static_cast<uint32_t>(keys[i] >> 32), 1ull);
}

__global__ void fill_i32_kernel(int32_t *p, int64_t n, int32_t v) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void minhop_finalize_kernel(int32_t *p, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n && p[i] == 0x7FFFFFFF) p[i] = 0;   // "0 when no agent reaches it" (dependency_reach.py:137-139,163)
}

}  // namespace abb
