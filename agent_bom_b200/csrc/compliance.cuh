// compliance.cuh — per-framework compliance-tag roll-up of a cached snapshot (sm_90a).
//
// Reference: the SQLite store's compliance_summary (api/graph_store.py:950-1031), which decodes every tagged node's
// compliance_tags per request and loops over every (node, tag) pair in Python, de-duplicating member nodes with a list scan.
// Here the host reads the tagged rows once per graph and interns them (compliance_host.inl): per row a text code (its raw
// compliance_tags string), a severity code and an entity-type code; per distinct text its tag codes (tags are coded in sorted
// order); per tag its framework code (frameworks are coded in sorted order).  The framework rule itself stays on the host.
// The device then:
//   - expands the (row, tag position) pairs: an exclusive scan over each row's tag count places them, one thread per pair finds
//     its row by binary search over the offsets, so a row with many tags is spread over many threads;
//   - per roll-up, forms a 64-bit key framework << lb | x (x: the row's severity code, type code, the tag code or the row itself;
//     lb the bits x needs) and radix-sorts it, stable, carrying the row: within a run of equal keys the first value is its first
//     row in id order;
//   - reduces each sorted array at its run heads: (framework, severity) and (framework, type) runs with their count and first row;
//     distinct (framework, tag) pairs; distinct (framework, row) pairs, whose per-framework segments give node_count and the
//     first CM_NODE_IDS rows.
// No structure is sized frameworks x rows: every array is sized by pairs, runs or frameworks.
#pragma once
#include <cstdint>

namespace abb {

constexpr int32_t CM_NODE_IDS = 100;       // node_ids per framework (the reference's [:100])

// tag count of each row; cnt[n] = 0 so an exclusive scan over n + 1 values ends with the pair count
__global__ void compliance_count_kernel(int32_t n, const int32_t *__restrict__ row_text, const int64_t *__restrict__ text_off,
                                        int64_t *__restrict__ cnt) {
    for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r <= n; r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (r == n) { cnt[r] = 0; continue; }
        const int32_t t = row_text[r];
        cnt[r] = text_off[t + 1] - text_off[t];
    }
}

// pair p -> its row and tag code; poff[n + 1] is the exclusive scan of the tag counts
__global__ void compliance_expand_kernel(int64_t m, int32_t n, const int64_t *__restrict__ poff, const int32_t *__restrict__ row_text,
                                         const int64_t *__restrict__ text_off, const int32_t *__restrict__ text_tags, int32_t *__restrict__ p_row,
                                         int32_t *__restrict__ p_tag) {
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < m; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        int32_t lo = 0, hi = n - 1;                // last row r with poff[r] <= p (rows without tags have poff[r] == poff[r + 1])
        while (lo < hi) {
            const int32_t mid = lo + (hi - lo + 1) / 2;
            if (poff[mid] <= p) lo = mid; else hi = mid - 1;
        }
        p_row[p] = lo;
        p_tag[p] = text_tags[text_off[row_text[lo]] + (p - poff[lo])];
    }
}

// key of pair p for one roll-up: framework << lb | x, x = code[row] (severity, type), the tag, or the row (code == nullptr, use_tag)
__global__ void compliance_keys_kernel(int64_t m, int lb, const int32_t *__restrict__ p_row, const int32_t *__restrict__ p_tag,
                                       const int32_t *__restrict__ tag_fw, const int32_t *__restrict__ code, bool use_tag,
                                       unsigned long long *__restrict__ keys) {
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < m; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t row = p_row[p], tag = p_tag[p];
        const int32_t x = code ? code[row] : use_tag ? tag : row;
        keys[p] = (static_cast<unsigned long long>(tag_fw[tag]) << lb) | static_cast<unsigned long long>(x);
    }
}

__global__ void compliance_heads_kernel(int64_t m, const unsigned long long *__restrict__ keys, uint8_t *__restrict__ head) {
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < m; p += static_cast<int64_t>(gridDim.x) * blockDim.x)
        head[p] = p == 0 || keys[p] != keys[p - 1];
}

// runs[4][u_n] (int64, columns framework, x, count, first row) of the u_n runs starting at heads[]; rows == nullptr: no first row
__global__ void compliance_runs_kernel(int64_t u_n, int64_t m, int lb, const int64_t *__restrict__ heads, const unsigned long long *__restrict__ keys,
                                       const int32_t *__restrict__ rows, int64_t *__restrict__ runs) {
    const unsigned long long mask = (1ull << lb) - 1;
    for (int64_t u = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; u < u_n; u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t h = heads[u];
        const unsigned long long k = keys[h];
        runs[u] = static_cast<int64_t>(k >> lb);
        runs[u_n + u] = static_cast<int64_t>(k & mask);
        runs[2 * u_n + u] = (u + 1 < u_n ? heads[u + 1] : m) - h;
        runs[3 * u_n + u] = rows ? rows[h] : -1;
    }
}

// per framework, the [start, end) of its segment in the distinct (framework, row) list fw[u_n] (ascending); frameworks without
// a segment keep start = end = 0 (memset)
__global__ void compliance_segments_kernel(int64_t u_n, const int64_t *__restrict__ fw, int64_t *__restrict__ seg_start,
                                           int64_t *__restrict__ seg_end) {
    for (int64_t u = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; u < u_n; u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t f = fw[u];
        if (u == 0 || fw[u - 1] != f) seg_start[f] = u;
        if (u + 1 == u_n || fw[u + 1] != f) seg_end[f] = u + 1;
    }
}

// node_count[f] = segment length; take[f] = min(node_count, CM_NODE_IDS); take[n_fw] = 0 (exclusive scan -> output offsets)
__global__ void compliance_node_count_kernel(int32_t n_fw, const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end,
                                             int64_t *__restrict__ node_count, int64_t *__restrict__ take) {
    for (int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; f <= n_fw; f += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (f == n_fw) { take[f] = 0; continue; }
        const int64_t c = seg_end[f] - seg_start[f];
        node_count[f] = c;
        take[f] = c < CM_NODE_IDS ? c : CM_NODE_IDS;
    }
}

// the first CM_NODE_IDS rows of each framework's segment, frameworks in order, into out at take_off[f]
__global__ void compliance_first_rows_kernel(int64_t u_n, const int64_t *__restrict__ fw, const int64_t *__restrict__ row,
                                             const int64_t *__restrict__ seg_start, const int64_t *__restrict__ take_off, int32_t *__restrict__ out) {
    for (int64_t u = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; u < u_n; u += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t f = fw[u], k = u - seg_start[f];
        if (k < CM_NODE_IDS) out[take_off[f] + k] = static_cast<int32_t>(row[u]);
    }
}

}  // namespace abb
