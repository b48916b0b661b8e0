// delta.cuh — scan-to-scan snapshot diff (sm_90a).
//
// Reference: diff_snapshots / changed_edges_between_scans (db/graph_store.py:671-842).  Two device graphs are compared:
//   - node matching: every node (ghost endpoints included) binary-searches its id bytes in the other graph's id list, walked
//     in sorted order through the other graph's permutation.  UTF-8 byte order is code-point order, which is the order of
//     Python's str comparison, so the result agrees with node_rank.  The search gives the node's partner (or -1) and the
//     number of the other graph's ids below it; rank + that count is the node's position in the sorted union of both id sets;
//   - node changes: a matched pair of real nodes differs when its entity type, status or severity code, label bytes or
//     risk (f64 ==) differ; codes the host could not map (a string outside the enum) are left to the host (flag 2);
//   - edge keys: one 64-bit key per original edge (forward entry, reversed bit clear), urank(src) << 33 | urank(tgt) << 6 |
//     relrank, radix-sorted per graph.  Ascending keys are sorted() over (source, target, relationship) string tuples;
//   - edge set difference: every sorted key binary-searches the other graph's sorted keys.  A shared key compares the
//     bidirectional and traversable flags and, when both graphs carry a weight column, the weight (f64 ==);
//   - shared edges (on request): the sorted keys of the new graph that have a partner, as (new edge, old edge) pairs in key order.
#pragma once
#include <cstdint>

namespace abb {

constexpr int DL_REL_SLOTS = 64;                    // relationship strings per graph (relrank has 6 bits)
constexpr int64_t DL_UNION_LIMIT = 1ll << 27;       // node ids in the union of both graphs (urank has 27 bits)
constexpr uint8_t DL_CODE_OTHER = 255;              // status / severity string outside the host's table

// -1 / 0 / 1 as bytes a compare to bytes b (shorter prefix first), like memcmp followed by a length compare.
__device__ __forceinline__ int dl_cmp(const uint8_t *__restrict__ a, int64_t la, const uint8_t *__restrict__ b, int64_t lb) {
    const int64_t l = la < lb ? la : lb;
    for (int64_t i = 0; i < l; i++) {
        const uint8_t x = a[i], y = b[i];
        if (x != y) return x < y ? -1 : 1;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

// For node i of graph A: lower bound of its id among B's ids in sorted order; partner = B's node at that position when equal.
// urank[i] = rank_A[i] + lower bound.
__global__ void delta_match_kernel(int64_t na, const uint8_t *__restrict__ a_ids, const int64_t *__restrict__ a_off, const int32_t *__restrict__ a_rank,
                                   int64_t nb, const uint8_t *__restrict__ b_ids, const int64_t *__restrict__ b_off, const int32_t *__restrict__ b_perm,
                                   int32_t *__restrict__ partner, int32_t *__restrict__ urank, unsigned long long *matched) {
    unsigned long long mine = 0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < na; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const uint8_t *s = a_ids + a_off[i];
        const int64_t ls = a_off[i + 1] - a_off[i];
        int64_t lo = 0, hi = nb;             // first sorted position whose id is >= s
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            const int32_t v = b_perm[mid];
            if (dl_cmp(b_ids + b_off[v], b_off[v + 1] - b_off[v], s, ls) < 0) lo = mid + 1; else hi = mid;
        }
        int32_t p = -1;
        if (lo < nb) {
            const int32_t v = b_perm[lo];
            if (dl_cmp(b_ids + b_off[v], b_off[v + 1] - b_off[v], s, ls) == 0) p = v;
        }
        partner[i] = p;
        urank[i] = a_rank[i] + static_cast<int32_t>(lo);
        mine += p >= 0;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(matched, mine);
}

// Per sorted position k of graph A (node i = perm[k]), a real node that has no real partner in B is flagged in `only`.
// When B is the old graph and A the new one (cmp = true), a real pair is also compared: changed = 1 when a column differs,
// 2 when only a code the host must compare as strings (type / status / severity outside the tables) is left.
template <bool CMP>
__global__ void delta_node_kernel(int64_t na, int32_t a_real, int32_t b_real, const int32_t *__restrict__ perm, const int32_t *__restrict__ partner,
                                  uint8_t *__restrict__ only, uint8_t *__restrict__ changed, const uint8_t *__restrict__ a_type,
                                  const uint8_t *__restrict__ b_type, const uint8_t *__restrict__ a_stat, const uint8_t *__restrict__ b_stat,
                                  const uint8_t *__restrict__ a_sev, const uint8_t *__restrict__ b_sev, const double *__restrict__ a_risk,
                                  const double *__restrict__ b_risk, const uint8_t *__restrict__ a_lbl, const int64_t *__restrict__ a_loff,
                                  const uint8_t *__restrict__ b_lbl, const int64_t *__restrict__ b_loff, uint8_t type_other) {
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < na; k += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t i = perm[k];
        uint8_t o = 0, c = 0;
        if (i < a_real) {
            const int32_t p = partner[i];
            if (p < 0 || p >= b_real) {
                o = 1;
            } else if (CMP) {
                const uint8_t ta = a_type[i], tb = b_type[p], sa = a_stat[i], sb = b_stat[p], va = a_sev[i], vb = b_sev[p];
                const bool differ = ta != tb || sa != sb || va != vb || !(a_risk[i] == b_risk[p]) ||
                                    dl_cmp(a_lbl + a_loff[i], a_loff[i + 1] - a_loff[i], b_lbl + b_loff[p], b_loff[p + 1] - b_loff[p]) != 0;
                c = differ ? 1 : ((ta == type_other || sa == DL_CODE_OTHER || va == DL_CODE_OTHER) ? 2 : 0);
            }
        }
        only[k] = o;
        if (CMP) changed[k] = c;
    }
}

// One key per original edge e = feid >> 1, written at position e with e as the value (row_of_entry: clusters.cuh).
__global__ void delta_edge_keys_kernel(int64_t m, int32_t n, const uint32_t *__restrict__ foff, const int32_t *__restrict__ fnbr,
                                       const uint8_t *__restrict__ fmeta, const uint32_t *__restrict__ feid, const int32_t *__restrict__ urank,
                                       const uint8_t *__restrict__ erel, const uint8_t *__restrict__ relmap, unsigned long long *__restrict__ keys,
                                       int32_t *__restrict__ vals) {
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; p < m; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (fmeta[p] & 0x80u) continue;
        const int32_t u = row_of_entry(foff, n, static_cast<uint32_t>(p));
        const int32_t v = fnbr[p];
        const uint32_t e = feid[p] >> 1;
        keys[e] = (static_cast<unsigned long long>(urank[u]) << 33) | (static_cast<unsigned long long>(urank[v]) << 6) | relmap[erel[e]];
        vals[e] = static_cast<int32_t>(e);
    }
}

// Per sorted key of graph A: `only` when B has no such key.  CMP (A new, B old): a shared key records B's edge in
// `partner` and is `changed` when direction, traversable or (both weights present) the weight differ.
template <bool CMP>
__global__ void delta_edge_diff_kernel(int64_t na, const unsigned long long *__restrict__ a_keys, const int32_t *__restrict__ a_vals, int64_t nb,
                                       const unsigned long long *__restrict__ b_keys, const int32_t *__restrict__ b_vals, uint8_t *__restrict__ only,
                                       uint8_t *__restrict__ changed, int32_t *__restrict__ partner, const uint8_t *__restrict__ a_flag,
                                       const uint8_t *__restrict__ b_flag, const double *__restrict__ a_w, const double *__restrict__ b_w) {
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < na; k += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const unsigned long long key = a_keys[k];
        int64_t lo = 0, hi = nb;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (b_keys[mid] < key) lo = mid + 1; else hi = mid;
        }
        const bool found = lo < nb && b_keys[lo] == key;
        only[k] = !found;
        if (CMP) {
            uint8_t c = 0;
            int32_t pe = -1;
            if (found) {
                const int32_t ea = a_vals[k];
                pe = b_vals[lo];
                c = a_flag[ea] != b_flag[pe];
                if (a_w && b_w && !(a_w[ea] == b_w[pe])) c = 1;
            }
            changed[k] = c;
            partner[k] = pe;
        }
    }
}

// flag[k] = 1 when sorted key k of the new graph has a partner in the old graph (a shared key).
__global__ void delta_shared_flag_kernel(int64_t n, const int32_t *__restrict__ partner, uint8_t *__restrict__ flag) {
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < n; k += static_cast<int64_t>(gridDim.x) * blockDim.x)
        flag[k] = partner[k] >= 0;
}

// out[j] = a[pos[j]], or b[a[pos[j]]] when b is given; flag_out[j] = flag[pos[j]] when both are given.
__global__ void delta_gather_kernel(int64_t n, const int32_t *__restrict__ pos, const int32_t *__restrict__ a, const int32_t *__restrict__ b,
                                    int32_t *__restrict__ out, const uint8_t *__restrict__ flag, uint8_t *__restrict__ flag_out) {
    for (int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t v = a[pos[j]];
        out[j] = b ? b[v] : v;
        if (flag && flag_out) flag_out[j] = flag[pos[j]];
    }
}

}  // namespace abb
