// search.cuh — node search and keyset pages over a cached snapshot (sm_90a).
//
// Reference: the SQLite store's search_nodes and page_nodes (api/graph_store.py:1242-1313, 1346-1468): an FTS5 MATCH (or a LIKE
// scan) over graph_node_search joined to graph_nodes, a COUNT(*) of every hit and a sort of every hit before the page.  Here the
// graph's search table (search_host.inl) holds, per node, the stored search_text bytes (raw text), the same text folded as FTS5's
// unicode61 tokenizer folds it with its tokens joined by one space (token text), the sort and filter keys, and the nodes in page
// order (order[]) with the inverse (pos[]).  A call:
//   - match: an FTS phrase is its folded tokens joined by one space, the last one a prefix, so it matches a row exactly when its
//     bytes occur in the token text at a token start; a LIKE pattern is an unanchored substring of the raw text.  A warp scans a
//     row (its lanes try 32 consecutive start positions at once); a row of SR_LONG bytes or more goes to a block;
//   - filter: entity-type, compliance and data-source byte tables indexed by interned string code, severity_id >= min_rank;
//   - cursor: the keyset predicate of the reference with SQL's NULL rules (a NULL severity never passes, a NULL risk passes only
//     through severity_id < ?); labels and ids compare as ranks, the cursor's label / id as insertion positions among them;
//   - output: two flags at pos[node], "matches" (counted for total) and "matches and passes the cursor"; the page is a flagged
//     select over order[].
// Table build: the code points >= 0x80 the raw text holds are marked in a 0x110000-bit bitmap; the host asks the SQLite library
// how unicode61 folds each of them (and ASCII) and uploads a dense fold table (-1 separator, 0 folds away, else the code point);
// one thread per row counts, then writes, the token text (count -> scan -> fill).  The page order is one radix sort of
// (severity desc, NULL last; risk desc, NULL last; label rank) over the nodes in id order, so equal keys stay in id order.
#pragma once
#include <cstdint>
#include <cuda/std/tuple>

namespace abb {

constexpr int64_t SR_LONG = 16384;             // rows at least this long are scanned by a block, shorter ones by a warp
constexpr int32_t SR_SEV_NULL = INT32_MIN;     // severity_id NULL (real values are above it)
constexpr int32_t SR_CODEPOINTS = 0x110000;

struct SrKey {
    uint32_t sev;                  // descending severity, NULL last
    uint32_t label;                // label rank
    unsigned long long risk;       // descending risk, NULL last
};

struct SrDecomposer {
    __host__ __device__ cuda::std::tuple<uint32_t &, unsigned long long &, uint32_t &> operator()(SrKey &k) const { return {k.sev, k.risk, k.label}; }
};

// per-call arguments on the device
struct SrCall {
    int32_t mode;                  // 0: no text predicate, 1: FTS phrases, 2: LIKE substring
    int32_t n_patterns;
    const uint8_t *pat; const int64_t *poff;
    const uint8_t *type_ok, *cmp_ok, *src_ok;    // nullptr: filter off
    int32_t use_min_rank; int64_t min_rank;
    int32_t has_cursor; int32_t cur_risk_null;
    int64_t cur_sev; double cur_risk;
    int64_t cur_label_gt;          // labels of rank >= this compare greater than the cursor's label
    int64_t cur_label_eq;          // rank equal to the cursor's label, -1 when no label equals it
    int64_t cur_id_gt;             // nodes (id order) from this index on have an id greater than the cursor's
};

// per-graph table on the device
struct SrTable {
    int32_t n;
    const uint8_t *raw; const int64_t *roff;
    const uint8_t *tok; const int64_t *toff;
    const int32_t *sev; const double *risk; const uint32_t *label;
    const int32_t *type, *cmp, *src;  // cmp / src are -1 for a node without an index row
    const int32_t *pos;
};

__device__ __forceinline__ int sr_utf8(const uint8_t *t, int64_t i, int64_t end, uint32_t *cp) {
    const uint32_t b = t[i];
    int k = b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4;
    if (i + k > end) k = 1;
    uint32_t c = k == 1 ? b : k == 2 ? (b & 0x1F) : k == 3 ? (b & 0x0F) : (b & 0x07);
    for (int j = 1; j < k; j++) c = (c << 6) | (t[i + j] & 0x3F);
    *cp = c < static_cast<uint32_t>(SR_CODEPOINTS) ? c : 0xFFFD;
    return k;
}

__device__ __forceinline__ int sr_put_utf8(uint8_t *o, uint32_t c) {
    if (c < 0x80) { o[0] = static_cast<uint8_t>(c); return 1; }
    if (c < 0x800) { o[0] = static_cast<uint8_t>(0xC0 | (c >> 6)); o[1] = static_cast<uint8_t>(0x80 | (c & 0x3F)); return 2; }
    if (c < 0x10000) {
        o[0] = static_cast<uint8_t>(0xE0 | (c >> 12)); o[1] = static_cast<uint8_t>(0x80 | ((c >> 6) & 0x3F)); o[2] = static_cast<uint8_t>(0x80 | (c & 0x3F));
        return 3;
    }
    o[0] = static_cast<uint8_t>(0xF0 | (c >> 18)); o[1] = static_cast<uint8_t>(0x80 | ((c >> 12) & 0x3F));
    o[2] = static_cast<uint8_t>(0x80 | ((c >> 6) & 0x3F)); o[3] = static_cast<uint8_t>(0x80 | (c & 0x3F));
    return 4;
}

__device__ __forceinline__ int sr_utf8_len(uint32_t c) { return c < 0x80 ? 1 : c < 0x800 ? 2 : c < 0x10000 ? 3 : 4; }

// code points >= 0x80 present in the text: one bit each
__global__ void search_codepoints_kernel(int64_t bytes, const uint8_t *__restrict__ text, uint32_t *__restrict__ bits) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < bytes; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (text[i] < 0xC0) continue;         // ASCII or a continuation byte
        uint32_t c;
        sr_utf8(text, i, bytes, &c);
        atomicOr(bits + (c >> 5), 1u << (c & 31));
    }
}

// token text of row r: unicode61 tokens (maximal runs of non-separators), each code point folded, tokens that fold to nothing
// dropped, joined by one space.  FILL = false writes the length into len[r], FILL = true the bytes at off[r].
template <bool FILL>
__global__ void search_normalize_kernel(int32_t n, const uint8_t *__restrict__ raw, const int64_t *__restrict__ roff, const int32_t *__restrict__ fold,
                                        int64_t *__restrict__ len_or_off, uint8_t *__restrict__ tok) {
    for (int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < n; r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t end = roff[r + 1];
        int64_t o = FILL ? len_or_off[r] : 0;
        bool any = false, in_tok = false, tok_out = false;
        for (int64_t i = roff[r]; i < end;) {
            uint32_t c;
            i += sr_utf8(raw, i, end, &c);
            const int32_t f = fold[c];
            if (f < 0) { in_tok = false; continue; }
            if (!in_tok) { in_tok = true; tok_out = false; }
            if (f == 0) continue;
            if (!tok_out) {
                if (any) { if (FILL) tok[o] = ' '; o++; }
                tok_out = any = true;
            }
            if (FILL) o += sr_put_utf8(tok + o, static_cast<uint32_t>(f));
            else o += sr_utf8_len(static_cast<uint32_t>(f));
        }
        if (!FILL) len_or_off[r] = o;
    }
    if (!FILL && blockIdx.x == 0 && threadIdx.x == 0) len_or_off[n] = 0;
}

// page-order keys of every node (values: the node, i.e. its id rank)
__global__ void search_keys_kernel(int32_t n, const int32_t *__restrict__ sev, const double *__restrict__ risk, const uint32_t *__restrict__ label,
                                   SrKey *__restrict__ keys, int32_t *__restrict__ vals) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        SrKey k;
        k.sev = ~(static_cast<uint32_t>(sev[i]) ^ 0x80000000u);       // SR_SEV_NULL maps to the largest key: last
        double x = risk[i];
        if (x != x) {
            k.risk = ~0ull;                                             // NULL (NaN) last
        } else {
            if (x == 0.0) x = 0.0;                                      // -0.0 = 0.0 in SQLite's comparison
            unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(x));
            b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);           // ascending order-preserving transform
            k.risk = ~b;                                                // descending
        }
        k.label = label[i];
        keys[i] = k;
        vals[i] = static_cast<int32_t>(i);
    }
}

__global__ void search_pos_kernel(int32_t n, const int32_t *__restrict__ order, int32_t *__restrict__ pos) {
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < n; k += static_cast<int64_t>(gridDim.x) * blockDim.x)
        pos[order[k]] = static_cast<int32_t>(k);
}

// filters of the call (everything but the text and the cursor)
__device__ __forceinline__ bool sr_filters(const SrTable &t, const SrCall &q, int64_t i) {
    if (q.mode && t.cmp[i] < 0) return false;                          // no index row: never found by a search
    if (q.type_ok && !q.type_ok[t.type[i]]) return false;
    if (q.use_min_rank && (t.sev[i] == SR_SEV_NULL || t.sev[i] < q.min_rank)) return false;
    if (q.cmp_ok && !q.cmp_ok[t.cmp[i]]) return false;
    if (q.src_ok && !q.src_ok[t.src[i]]) return false;
    return true;
}

// severity_id < ? OR (= AND risk_score < ?) OR (= AND = AND label > ?) OR (= AND = AND = AND id > ?), NULL never true
__device__ __forceinline__ bool sr_cursor(const SrTable &t, const SrCall &q, int64_t i) {
    if (!q.has_cursor) return true;
    const int32_t s = t.sev[i];
    if (s == SR_SEV_NULL) return false;
    if (s < q.cur_sev) return true;
    if (s != q.cur_sev) return false;
    const double r = t.risk[i];
    if (r != r || q.cur_risk_null) return false;
    if (r < q.cur_risk) return true;
    if (r != q.cur_risk) return false;
    const int64_t l = t.label[i];
    if (l >= q.cur_label_gt) return true;
    if (l != q.cur_label_eq) return false;
    return i >= q.cur_id_gt;
}

__device__ __forceinline__ bool sr_at(const uint8_t *s, int64_t j, const uint8_t *p, int64_t L) {
    for (int64_t k = 0; k < L; k++)
        if (s[j + k] != p[k]) return false;
    return true;
}

__device__ __forceinline__ void sr_row_text(const SrTable &t, const SrCall &q, int64_t i, const uint8_t **s, int64_t *len) {
    const uint8_t *base = q.mode == 1 ? t.tok : t.raw;
    const int64_t *off = q.mode == 1 ? t.toff : t.roff;
    *s = base + off[i];
    *len = off[i + 1] - off[i];
}

__device__ __forceinline__ void sr_flag(const SrTable &t, const SrCall &q, int64_t i, bool m, uint8_t *match, uint8_t *pass) {
    const int32_t p = t.pos[i];
    match[p] = m;
    pass[p] = m && sr_cursor(t, q, i);
}

// one warp per row shorter than SR_LONG (every row in mode 0); `total` counts the matching rows
__global__ void search_match_warp_kernel(SrTable t, SrCall q, uint8_t *__restrict__ match, uint8_t *__restrict__ pass,
                                         unsigned long long *__restrict__ total) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    unsigned long long mine = 0;
    for (int64_t i = warp; i < t.n; i += warps) {
        const uint8_t *s = nullptr;
        int64_t len = 0;
        if (q.mode) {
            sr_row_text(t, q, i, &s, &len);
            if (len >= SR_LONG) continue;                               // search_match_block_kernel's row
        }
        bool m = sr_filters(t, q, i);
        for (int p = 0; m && p < q.n_patterns; p++) {
            const uint8_t *pat = q.pat + q.poff[p];
            const int64_t L = q.poff[p + 1] - q.poff[p];
            bool found = false;
            for (int64_t j0 = 0; j0 + L <= len && !found; j0 += 32) {
                const int64_t j = j0 + lane;
                const bool hit = j + L <= len && (q.mode == 2 || j == 0 || s[j - 1] == ' ') && sr_at(s, j, pat, L);
                found = __any_sync(0xFFFFFFFFu, hit);
            }
            m = found;
        }
        if (lane == 0) {
            sr_flag(t, q, i, m, match, pass);
            mine += m;
        }
    }
    if (lane == 0 && mine) atomicAdd(total, mine);
}

// one block per listed row of SR_LONG bytes or more
__global__ void search_match_block_kernel(SrTable t, SrCall q, int64_t n_long, const int32_t *__restrict__ rows, uint8_t *__restrict__ match,
                                          uint8_t *__restrict__ pass, unsigned long long *__restrict__ total) {
    for (int64_t b = blockIdx.x; b < n_long; b += gridDim.x) {
        const int64_t i = rows[b];
        const uint8_t *s;
        int64_t len;
        sr_row_text(t, q, i, &s, &len);
        if (len < SR_LONG) continue;                                     // the warp kernel's row (mode 1 and 2 lengths differ)
        bool m = sr_filters(t, q, i);
        for (int p = 0; m && p < q.n_patterns; p++) {
            const uint8_t *pat = q.pat + q.poff[p];
            const int64_t L = q.poff[p + 1] - q.poff[p];
            int found = 0;
            for (int64_t j0 = 0; j0 + L <= len && !found; j0 += blockDim.x) {
                const int64_t j = j0 + threadIdx.x;
                const bool hit = j + L <= len && (q.mode == 2 || j == 0 || s[j - 1] == ' ') && sr_at(s, j, pat, L);
                found = __syncthreads_or(hit);
            }
            m = found;
        }
        if (threadIdx.x == 0) {
            sr_flag(t, q, i, m, match, pass);
            if (m) atomicAdd(total, 1ull);
        }
        __syncthreads();
    }
}

}  // namespace abb
