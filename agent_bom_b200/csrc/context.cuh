// context.cuh — typed in-neighbour lists of findings for the OCSF export's graph_context (sm_90a).
//
// Device restatement of the neighbour half of UnifiedGraph.to_ocsf_events (graph/container.py:628-654):
//
//   sources = [e.source for e in reverse_adjacency[f]]          (list order, reversed twins included, duplicates kept)
//   affected_agents / servers / packages / exposed_credentials = the sources with a node record of that entity type
//
// Row u of the reverse CSR is reverse_adjacency[u] in list order, so the lists are the entries of f's reverse row filtered by
// the neighbour's entity code.  The filter is a 256-entry table (entity code -> bucket) built in shared memory by every block;
// ghosts (code 255) and every other kind fall into CTX_NONE.  Two passes with one thread per finding, as links_kernel in
// paths.cuh: COUNT writes the four bucket counts and the per-finding total, which are scanned into start offsets; FILL writes
// each bucket's sources at start[q] + (counts of the buckets before it) in row order.  Reverse rows longer than LONG_ROW are
// handed to the whole warp, which ranks its entries with ballot / popc so the order is kept.  The blast-radius half
// (impact_of's count and type histogram) is the unchanged impact walk, run next to these kernels.
#pragma once
#include "walk.cuh"

namespace abb {

constexpr int CTX_BUCKETS = ABB_CTX_BUCKETS;
constexpr uint32_t CTX_LONG_ROW = 64;   // reverse rows longer than this are handled by the whole warp

struct CtxArgs {
    GraphView g;
    const int32_t *findings;    // [n] node index per finding; invalid / ghost = empty lists
    int64_t n;
    int32_t *bcnt;              // [n * CTX_BUCKETS] sources per bucket (COUNT writes, FILL reads)
    int64_t *cnt;               // [n + 1] sources per finding (COUNT), scanned into start
    const int64_t *start;       // [n + 1] first source of each finding (FILL)
    int32_t *src;               // [start[n]] source node indices, bucket-major within a finding, row order within a bucket
};

__device__ __forceinline__ uint8_t ctx_bucket_of(unsigned code) {
    switch (code) {
        case 0: return ABB_CTX_AGENT;         // agent
        case 1: return ABB_CTX_SERVER;        // server
        case 2: return ABB_CTX_PACKAGE;       // package
        case 10: return ABB_CTX_CREDENTIAL;   // credential
        default: return ABB_CTX_NONE;
    }
}

template <bool FILL>
__global__ void __launch_bounds__(256) context_kernel(const CtxArgs A) {
    __shared__ uint8_t bucket[256];
    bucket[threadIdx.x] = ctx_bucket_of(threadIdx.x);   // blockDim.x == 256
    __syncthreads();
    const GraphView &g = A.g;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < A.n; base += nwarps * 32) {
        const int64_t q = base + lane;
        uint32_t s0 = 0, e0 = 0;
        if (q < A.n) {
            const int32_t u = __ldg(A.findings + q);
            if (u >= 0 && u < g.n && __ldg(g.ntype + u) != ABB_NODE_GHOST) { s0 = __ldg(g.roff + u); e0 = __ldg(g.roff + u + 1); }
        }
        const bool is_long = e0 - s0 > CTX_LONG_ROW;
        int32_t c[CTX_BUCKETS] = {0, 0, 0, 0};
        int64_t o[CTX_BUCKETS] = {0, 0, 0, 0};     // FILL: first output slot of each bucket
        if (FILL && q < A.n) {
            o[0] = A.start[q];
            for (int b = 1; b < CTX_BUCKETS; b++) o[b] = o[b - 1] + A.bcnt[q * CTX_BUCKETS + b - 1];
        }
        if (!is_long) {
            for (uint32_t p = s0; p < e0; p++) {
                const int32_t v = __ldg(g.rnbr + p);
                const uint8_t b = bucket[__ldg(g.ntype + v)];
                if (b >= CTX_BUCKETS) continue;
                if (FILL) A.src[o[b] + c[b]] = v;
                c[b]++;
            }
        }
        for (unsigned rem = __ballot_sync(FULL, is_long); rem; rem &= rem - 1) {
            const int leader = __ffs(rem) - 1;
            const uint32_t ls0 = __shfl_sync(FULL, s0, leader), le0 = __shfl_sync(FULL, e0, leader);
            int64_t lo[CTX_BUCKETS];
#pragma unroll
            for (int b = 0; b < CTX_BUCKETS; b++) lo[b] = __shfl_sync(FULL, o[b], leader);
            int32_t lc[CTX_BUCKETS] = {0, 0, 0, 0};
            for (uint32_t p = ls0; p < le0; p += 32) {
                const uint32_t k = p + lane;
                const int32_t v = k < le0 ? __ldg(g.rnbr + k) : -1;
                const uint8_t mine = v >= 0 ? bucket[__ldg(g.ntype + v)] : static_cast<uint8_t>(ABB_CTX_NONE);
#pragma unroll
                for (int b = 0; b < CTX_BUCKETS; b++) {
                    const unsigned m = __ballot_sync(FULL, mine == b);
                    if (FILL && mine == b) A.src[lo[b] + lc[b] + __popc(m & lanemask_lt(lane))] = v;
                    lc[b] += __popc(m);
                }
            }
            if (lane == leader)
#pragma unroll
                for (int b = 0; b < CTX_BUCKETS; b++) c[b] = lc[b];
        }
        if (!FILL && q < A.n) {
            int64_t total = 0;
#pragma unroll
            for (int b = 0; b < CTX_BUCKETS; b++) { A.bcnt[q * CTX_BUCKETS + b] = c[b]; total += c[b]; }
            A.cnt[q] = total;
        }
    }
}

}  // namespace abb
