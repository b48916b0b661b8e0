// lifecycle.cuh — a tenant's edge history and the versions active at a timestamp (sm_90a).
//
// Reference: active_edges_at (db/graph_store.py:775-796).  The host reads every edge row of every snapshot of a tenant in
// (created_at, scan_id) order and codes each row: source, target and relationship as ranks in tenant-wide sorted dictionaries,
// and created_at, the effective valid_from and valid_to as ranks in one sorted dictionary of every timestamp string (LC_NONE for
// an absent one).  On the device:
//   - table build: one 64-bit key per row, src << 37 | tgt << 10 | rel, stably radix-sorted with the row index as value, so the
//     rows of a key keep their (created_at, scan_id) order.  Ascending keys are sorted() over (source, target, relationship)
//     string tuples.  Each sorted row stores (created, valid_from, valid_to, row) as one int4, and the run heads give the
//     segment starts;
//   - per call: with r = the number of dictionary strings <= at, a string s satisfies s <= at exactly when rank(s) < r, and
//     valid_to > at when rank(valid_to) >= r.  One thread per key walks its segment back from the last row and takes the first
//     row with created < r, valid_from < r and valid_to >= r (the reference keeps the last qualifying version of each key).
//     The winners are compacted in key order by a flagged select.
#pragma once
#include <cstdint>

namespace abb {

constexpr int64_t LC_ID_LIMIT = 1ll << 27;       // distinct source / target ids of one history (27 bits each in the key)
constexpr int64_t LC_REL_LIMIT = 1ll << 10;      // distinct relationship strings of one history (10 bits)
constexpr int32_t LC_NONE = 0x7FFFFFFF;          // rank of an absent timestamp: never < r, always >= r

__global__ void lc_keys_kernel(int64_t n, const int32_t *__restrict__ src, const int32_t *__restrict__ tgt, const int32_t *__restrict__ rel,
                               unsigned long long *__restrict__ keys, int32_t *__restrict__ vals) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        keys[i] = (static_cast<unsigned long long>(src[i]) << 37) | (static_cast<unsigned long long>(tgt[i]) << 10) | static_cast<unsigned long long>(rel[i]);
        vals[i] = static_cast<int32_t>(i);
    }
}

// Per sorted position k: the row's three ranks and its index, and whether k starts a key's segment.
__global__ void lc_rows_kernel(int64_t n, const unsigned long long *__restrict__ keys, const int32_t *__restrict__ vals,
                               const int32_t *__restrict__ created, const int32_t *__restrict__ vfrom, const int32_t *__restrict__ vto,
                               int4 *__restrict__ rows, uint8_t *__restrict__ head) {
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < n; k += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t i = vals[k];
        rows[k] = make_int4(created[i], vfrom[i], vto[i], i);
        head[k] = k == 0 || keys[k] != keys[k - 1];
    }
}

// Per key segment s (rows seg[s] .. seg[s + 1] - 1): the row index of its last version active at rank r, or -1.
__global__ void lc_active_kernel(int64_t n_seg, const int32_t *__restrict__ seg, const int4 *__restrict__ rows, int32_t r,
                                 int32_t *__restrict__ win, uint8_t *__restrict__ flag) {
    for (int64_t s = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < n_seg; s += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t lo = seg[s];
        int32_t w = -1;
        for (int32_t k = seg[s + 1] - 1; k >= lo; k--) {
            const int4 v = rows[k];
            if (v.x < r && v.y < r && v.z >= r) { w = v.w; break; }
        }
        win[s] = w;
        flag[s] = w >= 0;
    }
}

}  // namespace abb
