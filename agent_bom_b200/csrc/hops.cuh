// hops.cuh — multi-hop blast-radius expansion: ordered, depth-bounded BFS over agents and MCP server names (sm_90a).
//
// Reference: expand_blast_radius_hops (scanners/blast_radius.py:16-97).  The host interns agent names, server names and credential
// names and hands over two CSRs: name -> servers (the last agent object of a name wins) and server -> agent occurrences (one per
// (agent object, server) pair, in agents order then mcp_servers order), each occurrence carrying its object's credential set.
// Blast radii that share a signature (affected agent names, direct servers) are searched once.  Per signature the host marks
// the visited agents (the affected names) and servers (the direct ones and the first-level queue), and lists the first-level
// queue entries (server, root).
//
// The reference pops a FIFO queue.  All entries of hop h are enqueued before any of hop h + 1 is popped, so the queue is a
// sequence of levels, and within a level the order is the order of enqueueing.  One level on the device:
//   - agents: every entry (rank i, in queue order) claims each unvisited occurrence name at position p of its server's list with
//     atomicMin on (i << 32 | p).  The winners are exactly the reference's discoveries, and (i, p) order is its discovery order.
//     A count, an exclusive scan and an ordered write append them; each winner marks its name visited and resets the claim.
//   - servers (while hop + 1 < max_depth): every discovery (rank j) claims each unvisited server at position q of its name's
//     list with (j << 32 | q), and the same count, scan and write append the next level's entries in queue order.
// Several signatures run at once, each with its own visited and claim rows in the batch's scratch (slot = signature - first
// signature of the batch).  Entries and discoveries of one level are ordered by signature first, so global ranks keep every
// signature's order.
#pragma once
#include <cstdint>

namespace abb {

constexpr unsigned long long HOP_UNCLAIMED = ~0ull;

// One warp per signature of the batch: marks its visited agents and servers.
__global__ void hops_mark_kernel(int64_t s0, int64_t n_batch, const int64_t *__restrict__ ag_off, const int32_t *__restrict__ ag,
                                 const int64_t *__restrict__ sv_off, const int32_t *__restrict__ sv, int64_t n_names, int64_t n_servers,
                                 uint8_t *__restrict__ avis, uint8_t *__restrict__ svis) {
    const int lane = threadIdx.x & 31;
    for (int64_t b = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; b < n_batch; b += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
        const int64_t s = s0 + b;
        for (int64_t k = ag_off[s] + lane; k < ag_off[s + 1]; k += 32) avis[b * n_names + ag[k]] = 1;
        for (int64_t k = sv_off[s] + lane; k < sv_off[s + 1]; k += 32) svis[b * n_servers + sv[k]] = 1;
    }
}

// Claim pass.  Item i (an entry or a discovery) of signature sig[i] walks the list lst[off[key[i]] ..] and claims every item
// not yet visited in its signature's row.
__global__ void hops_claim_kernel(int64_t n, int64_t s0, const int32_t *__restrict__ sig, const int32_t *__restrict__ key,
                                  const int32_t *__restrict__ key_map, const int64_t *__restrict__ off, const int32_t *__restrict__ lst,
                                  int64_t width, const uint8_t *__restrict__ vis, unsigned long long *__restrict__ claim) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t k = key_map ? key_map[key[i]] : key[i];
        const int64_t row = (sig[i] - s0) * width, lo = off[k], hi = off[k + 1];
        for (int64_t p = lo; p < hi; p++) {
            const int64_t c = row + lst[p];
            if (!vis[c]) atomicMin(&claim[c], (static_cast<unsigned long long>(i) << 32) | static_cast<unsigned long long>(p - lo));
        }
    }
}

// Count pass: how many claims item i won (cnt[i]); cnt[n] = 0 so the exclusive scan's last element is the total.
__global__ void hops_count_kernel(int64_t n, int64_t s0, const int32_t *__restrict__ sig, const int32_t *__restrict__ key,
                                  const int32_t *__restrict__ key_map, const int64_t *__restrict__ off, const int32_t *__restrict__ lst,
                                  int64_t width, const unsigned long long *__restrict__ claim, int64_t *__restrict__ cnt) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i <= n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (i == n) { cnt[n] = 0; continue; }
        const int32_t k = key_map ? key_map[key[i]] : key[i];
        const int64_t row = (sig[i] - s0) * width, lo = off[k], hi = off[k + 1];
        int64_t c = 0;
        for (int64_t p = lo; p < hi; p++)
            c += claim[row + lst[p]] == ((static_cast<unsigned long long>(i) << 32) | static_cast<unsigned long long>(p - lo));
        cnt[i] = c;
    }
}

// Write pass: item i appends its won claims at pos[i] onward in list order: the signature, the list position (an occurrence
// index for agents, a server id for servers) and the parent (parent_base + i).  Each winner marks its item visited and resets
// the claim; only the winner's key equals the claim, so the reset cannot change another item's outcome.
__global__ void hops_write_kernel(int64_t n, int64_t s0, const int32_t *__restrict__ sig, const int32_t *__restrict__ key,
                                  const int32_t *__restrict__ key_map, const int64_t *__restrict__ off, const int32_t *__restrict__ lst,
                                  int64_t width, uint8_t *__restrict__ vis, unsigned long long *__restrict__ claim, const int64_t *__restrict__ pos,
                                  bool emit_list_value, int64_t parent_base, int32_t *__restrict__ out_sig, int32_t *__restrict__ out_item,
                                  int64_t *__restrict__ out_parent) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t k = key_map ? key_map[key[i]] : key[i];
        const int64_t row = (sig[i] - s0) * width, lo = off[k], hi = off[k + 1];
        int64_t w = pos[i];
        for (int64_t p = lo; p < hi; p++) {
            const int64_t c = row + lst[p];
            if (claim[c] != ((static_cast<unsigned long long>(i) << 32) | static_cast<unsigned long long>(p - lo))) continue;
            claim[c] = HOP_UNCLAIMED;
            vis[c] = 1;
            out_sig[w] = sig[i];
            out_item[w] = emit_list_value ? lst[p] : static_cast<int32_t>(p);
            out_parent[w] = parent_base + i;
            w++;
        }
    }
}

// Credential keys: discovery i contributes (signature << 32 | credential) for every credential of its occurrence's set.
__global__ void hops_cred_count_kernel(int64_t n, const int32_t *__restrict__ occ, const int32_t *__restrict__ occ_cset,
                                       const int64_t *__restrict__ cs_off, int64_t *__restrict__ cnt) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i <= n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (i == n) { cnt[n] = 0; continue; }
        const int32_t c = occ_cset[occ[i]];
        cnt[i] = cs_off[c + 1] - cs_off[c];
    }
}

__global__ void hops_cred_fill_kernel(int64_t n, const int32_t *__restrict__ sig, const int32_t *__restrict__ occ, const int32_t *__restrict__ occ_cset,
                                      const int64_t *__restrict__ cs_off, const int32_t *__restrict__ cs_cred, const int64_t *__restrict__ pos,
                                      unsigned long long *__restrict__ keys) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t c = occ_cset[occ[i]];
        const unsigned long long hi = static_cast<unsigned long long>(sig[i]) << 32;
        int64_t w = pos[i];
        for (int64_t p = cs_off[c]; p < cs_off[c + 1]; p++) keys[w++] = hi | static_cast<unsigned long long>(static_cast<uint32_t>(cs_cred[p]));
    }
}

}  // namespace abb
