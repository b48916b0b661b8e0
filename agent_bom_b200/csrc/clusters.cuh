// clusters.cuh — semantic-cluster roll-ups (sm_90a).
//
// Reference: build_semantic_clusters (graph/semantic_clusters.py:81-124).  The host interns every node's cluster keys
// (at most two per node: source_environment and one kind-specific key) into int32 codes, codes[2u], codes[2u+1], -1 = none.
// Everything below is graph-constant and runs once per graph:
//   - node pass: per cluster member count, max risk, 5-bin severity histogram, entity-type mask and incident entries;
//   - member order: (cluster << 32 | node_rank) keys, radix-sorted, so each cluster is a segment of members in id order;
//   - relationship counts: every original edge (forward entry, reversed bit clear) counts once for each DISTINCT cluster
//     among its up to four endpoint codes (the reference's `source in S or target in S`).  The few heavy clusters (most
//     incident entries, e.g. a source_environment holding every node) count in per-block shared-memory counters; every
//     other (cluster, relationship) occurrence is emitted as a (cluster << 5 | rel) key, radix-sorted and run-length encoded.
// Relationship code 31 (a string outside the enum) is skipped here and counted by the host from the edge records.
#pragma once
#include <cstdint>

namespace abb {

constexpr int CL_HEAVY = 64;          // shared-memory relationship counters: CL_HEAVY clusters x 32 relationships
constexpr uint8_t CL_REL_OTHER = 31;

// Warp-aggregated roll-up: lanes holding the same cluster code combine with __reduce_*_sync over their match mask, and
// one leader per distinct code does the global atomics (the all-node cluster sees one atomic per warp, not per node).
__global__ void cluster_node_kernel(int64_t n, const int32_t *__restrict__ codes, const uint8_t *__restrict__ level,
                                    const double *__restrict__ risk, const uint8_t *__restrict__ etype, const uint32_t *__restrict__ foff,
                                    const uint32_t *__restrict__ roff, unsigned long long *cnt, unsigned long long *risk_bits,
                                    unsigned long long *hist, unsigned long long *tmask, unsigned long long *inc) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t base = warp0 * 32; base < n; base += nwarps * 32) {
        const int64_t u = base + lane;
        const bool valid = u < n;
        unsigned long long bits = 0;
        unsigned lv = 0, deg = 0;
        unsigned long long tbit = 0;
        if (valid) {
            bits = static_cast<unsigned long long>(__double_as_longlong(risk[u]));
            lv = level[u];
            tbit = 1ull << (etype[u] & 63);
            deg = min(foff[u + 1] - foff[u] + roff[u + 1] - roff[u], 1u << 26);
        }
        for (int j = 0; j < 2; j++) {
            const int32_t c = valid ? codes[2 * u + j] : -1;
            const unsigned grp = __match_any_sync(0xFFFFFFFFu, c);
            if (c < 0) continue;
            const bool leader = lane == __ffs(grp) - 1;
            const unsigned hi = __reduce_max_sync(grp, static_cast<unsigned>(bits >> 32));
            const unsigned lo = __reduce_max_sync(grp, static_cast<unsigned>(bits >> 32) == hi ? static_cast<unsigned>(bits) : 0u);
            const unsigned t_lo = __reduce_or_sync(grp, static_cast<unsigned>(tbit));
            const unsigned t_hi = __reduce_or_sync(grp, static_cast<unsigned>(tbit >> 32));
            const unsigned d = __reduce_add_sync(grp, deg);
            unsigned h[5];
#pragma unroll
            for (int k = 0; k < 5; k++) h[k] = __reduce_add_sync(grp, lv == static_cast<unsigned>(k) ? 1u : 0u);
            if (leader) {
                atomicAdd(&cnt[c], static_cast<unsigned long long>(__popc(grp)));
                atomicMax(&risk_bits[c], (static_cast<unsigned long long>(hi) << 32) | lo);   // non-negative doubles order as their bits
                atomicOr(&tmask[c], (static_cast<unsigned long long>(t_hi) << 32) | t_lo);
                atomicAdd(&inc[c], static_cast<unsigned long long>(d));
#pragma unroll
                for (int k = 0; k < 5; k++)
                    if (h[k]) atomicAdd(&hist[static_cast<int64_t>(c) * 5 + k], static_cast<unsigned long long>(h[k]));
            }
        }
    }
}

// One key per (node, cluster) membership: cluster in the high word, the node's id-string rank in the low word; absent
// memberships get ~0 and sort to the end.
__global__ void cluster_member_keys_kernel(int64_t n, const int32_t *__restrict__ codes, const int32_t *__restrict__ rank,
                                           unsigned long long *keys, int32_t *vals) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < 2 * n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t c = codes[i];
        const int64_t u = i >> 1;
        keys[i] = c < 0 ? ~0ull : (static_cast<unsigned long long>(c) << 32) | static_cast<uint32_t>(rank[u]);
        vals[i] = static_cast<int32_t>(u);
    }
}

__device__ __forceinline__ int32_t row_of_entry(const uint32_t *__restrict__ foff, int32_t n, uint32_t p) {
    int32_t lo = 0, hi = n;                 // last row whose offset is <= p
    while (hi - lo > 1) {
        const int32_t mid = (lo + hi) >> 1;
        if (__ldg(&foff[mid]) <= p) lo = mid; else hi = mid;
    }
    return lo;
}

// Relationship occurrences.  FILL = false: count the light (cluster, relationship) keys into *total.  FILL = true: write them
// at positions reserved from *total, used as a cursor (order is irrelevant, a sort follows), and count heavy clusters in
// shared memory.
template <bool FILL>
__global__ void cluster_rel_kernel(int64_t m, int32_t n, const uint32_t *__restrict__ foff, const int32_t *__restrict__ fnbr,
                                   const uint8_t *__restrict__ fmeta, const int32_t *__restrict__ codes, const int32_t *__restrict__ heavy_slot,
                                   unsigned long long *total, unsigned long long *keys, unsigned long long *heavy_cnt) {
    __shared__ unsigned s_heavy[FILL ? CL_HEAVY * 32 : 1];
    __shared__ unsigned long long s_total;
    if (FILL) for (int i = threadIdx.x; i < CL_HEAVY * 32; i += blockDim.x) s_heavy[i] = 0;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    unsigned long long mine = 0;
    for (int64_t base = warp0 * 32; base < m; base += nwarps * 32) {
        const int64_t p = base + lane;
        int32_t c[4] = {-1, -1, -1, -1};
        uint32_t rel = 0;
        if (p < m) {
            const uint8_t meta = fmeta[p];
            rel = meta & 0x1Fu;
            if (!(meta & 0x80u) && rel != CL_REL_OTHER) {
                const int32_t u = row_of_entry(foff, n, static_cast<uint32_t>(p));
                const int32_t v = fnbr[p];
                c[0] = codes[2 * static_cast<int64_t>(u)]; c[1] = codes[2 * static_cast<int64_t>(u) + 1];
                c[2] = codes[2 * static_cast<int64_t>(v)]; c[3] = codes[2 * static_cast<int64_t>(v) + 1];
                if (c[1] == c[0]) c[1] = -1;
                if (c[2] == c[0] || c[2] == c[1]) c[2] = -1;
                if (c[3] == c[0] || c[3] == c[1] || c[3] == c[2]) c[3] = -1;
            }
        }
        unsigned light = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (c[k] < 0) continue;
            const int32_t s = heavy_slot[c[k]];
            if (s >= 0) {
                if (FILL) atomicAdd(&s_heavy[s * 32 + rel], 1u);
                c[k] = -1;
            } else {
                light++;
            }
        }
        if (!FILL) { mine += light; continue; }
        // warp-aggregated reservation of this warp's light keys
        unsigned incl = light;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
        const unsigned wsum = __shfl_sync(0xFFFFFFFFu, incl, 31);
        unsigned long long at = 0;
        if (lane == 31 && wsum) at = atomicAdd(total, static_cast<unsigned long long>(wsum));
        at = __shfl_sync(0xFFFFFFFFu, at, 31) + (incl - light);
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (c[k] >= 0) keys[at++] = (static_cast<unsigned long long>(c[k]) << 5) | rel;
    }
    if (!FILL) {
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
        if (lane == 0 && mine) atomicAdd(&s_total, mine);
        __syncthreads();
        if (threadIdx.x == 0 && s_total) atomicAdd(total, s_total);
        return;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < CL_HEAVY * 32; i += blockDim.x)
        if (s_heavy[i]) atomicAdd(&heavy_cnt[i], static_cast<unsigned long long>(s_heavy[i]));
}

// Non-zero (cluster, relationship) pairs per cluster.
__global__ void cluster_pair_count_kernel(int64_t npairs, const unsigned long long *__restrict__ keys, unsigned long long *nnz) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < npairs; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        atomicAdd(&nnz[keys[i] >> 5], 1ull);
}

__device__ __forceinline__ int64_t segment_of(const int64_t *__restrict__ out_off, int64_t nsel, int64_t i) {
    int64_t lo = 0, hi = nsel;              // last segment whose output offset is <= i
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (out_off[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// Gather of the requested clusters' segments into one contiguous output (selection order): members, or relationship pairs.
__global__ void cluster_gather_members_kernel(int64_t total, int64_t nsel, const int64_t *__restrict__ out_off, const int64_t *__restrict__ src_start,
                                              const int32_t *__restrict__ members, int32_t *out) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t s = segment_of(out_off, nsel, i);
        out[i] = members[src_start[s] + (i - out_off[s])];
    }
}

__global__ void cluster_gather_rels_kernel(int64_t total, int64_t nsel, const int64_t *__restrict__ out_off, const int64_t *__restrict__ src_start,
                                           const unsigned long long *__restrict__ keys, const int64_t *__restrict__ counts, uint8_t *rel_out,
                                           int64_t *count_out) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t s = segment_of(out_off, nsel, i);
        const int64_t j = src_start[s] + (i - out_off[s]);
        rel_out[i] = static_cast<uint8_t>(keys[j] & 31u);
        count_out[i] = counts[j];
    }
}

}  // namespace abb
