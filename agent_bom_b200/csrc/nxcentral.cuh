// nxcentral.cuh — the NetworkX analysis backend's device work (sm_90a): exact Brandes betweenness, scipy-order PageRank and
// the batched bidirectional shortest-path search.
//
// References (networkx 3.6.1): betweenness_centrality = _single_source_shortest_path_basic + _accumulate_basic + _rescale;
// pagerank = _pagerank_scipy; shortest_path(G, s, t) = bidirectional_shortest_path -> _bidirectional_pred_succ.  Every result
// must equal NetworkX's bit for bit, so every floating-point operation here is an explicit round-to-nearest intrinsic (no FMA
// contraction) applied in the order NetworkX / numpy / scipy apply it; the comments say which order that is.
#pragma once
#include <cstdint>

namespace abb {
namespace nx {

// ---------------------------------------------------------------- numpy's pairwise summation
// DOUBLE_pairwise_sum: fewer than 8 items are summed from -0.0; up to 128 with 8 strided accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added in order; longer runs split at n/2 rounded down to a multiple of 8.
__device__ __forceinline__ double pairwise_leaf(const double *a, int64_t n) {
    if (n < 8) {
        double r = -0.0;
        for (int64_t i = 0; i < n; i++) r = __dadd_rn(r, a[i]);
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] = __dadd_rn(r[j], a[i + j]);
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; i++) res = __dadd_rn(res, a[i]);
    return res;
}

// numpy's recursion pw(a, n) = pw(a, h) + pw(a + h, n - h) walked with an explicit stack (left half first, as C evaluates it)
constexpr int PW_DEPTH = 40;   // halving from 2^40 items down to 128 takes fewer levels
__device__ double pairwise_sum(const double *a, int64_t n) {
    if (n <= 128) return pairwise_leaf(a, n);
    int64_t r_off[PW_DEPTH], r_len[PW_DEPTH];
    double left[PW_DEPTH];
    bool have_left[PW_DEPTH];
    int sp = 0;
    int64_t o = 0, m = n;
    for (;;) {
        while (m > 128) {
            int64_t h = m / 2;
            h -= h % 8;
            r_off[sp] = o + h; r_len[sp] = m - h; have_left[sp] = false; sp++;
            m = h;
        }
        double acc = pairwise_leaf(a + o, m);
        while (sp > 0 && have_left[sp - 1]) { acc = __dadd_rn(left[sp - 1], acc); sp--; }
        if (sp == 0) return acc;
        left[sp - 1] = acc; have_left[sp - 1] = true;
        o = r_off[sp - 1]; m = r_len[sp - 1];
    }
}

// ---------------------------------------------------------------- PageRank (_pagerank_scipy)
// scipy's row sums S = A.sum(axis=1) are np.add.reduceat over each row's weights in ascending column order: w0 + pw(w1..).
// inv = 1/S where S != 0, else 0; a row is dangling when inv == 0 (is_dangling = S == 0 after S[S != 0] = 1/S), so a sum that
// overflowed to +-inf is dangling too.
__global__ void pr_rowsum_kernel(int32_t n, const uint32_t *off, const double *w_sorted, double *inv, uint8_t *dangling) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t a = off[i], k = static_cast<int64_t>(off[i + 1]) - a;
        double s = 0.0;
        if (k == 1) s = w_sorted[a];
        else if (k > 1) s = __dadd_rn(w_sorted[a], pairwise_sum(w_sorted + a + 1, k - 1));
        const double r = s != 0.0 ? __ddiv_rn(1.0, s) : 0.0;
        inv[i] = r;
        dangling[i] = r == 0.0;
    }
}

// edge weight by edge index (forward entry e carries edge feid[e] >> 1)
__global__ void pr_edge_weight_kernel(int64_t m, const uint32_t *feid, const double *w, double *w_edge) {
    for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < m; e += static_cast<int64_t>(gridDim.x) * blockDim.x)
        w_edge[feid[e] >> 1] = w[e];
}

// reverse entry r of row k = in-edge (j -> k): key j, value A[j,k] = inv[j] * w (scipy's Q @ A).  Q = dia_array((1/S, 0)) drops
// a zero diagonal entry, so a row with inv 0 has no entries in Q @ A; its value is 0.0, which leaves a finite sum as it was
// (never 0 * inf = NaN).
__global__ void pr_rev_values_kernel(int64_t m, const int32_t *rnbr, const uint32_t *reid, const double *inv, const double *w_edge, int32_t *key,
                                     double *val) {
    for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r < m; r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t j = rnbr[r];
        const double ij = inv[j];
        key[r] = j;
        val[r] = ij == 0.0 ? 0.0 : __dmul_rn(ij, w_edge[reid[r] >> 1]);
    }
}

// dsum = sum(x[is_dangling]): Python's builtin sum over numpy scalars — sequential in index order.  Inherently serial: one thread.
__global__ void pr_dangling_sum_kernel(const int *done, int64_t nd, const int32_t *dangling_idx, const double *x, double *dsum) {
    if (*done) return;
    double s = 0.0;
    for (int64_t i = 0; i < nd; i++) s = __dadd_rn(s, x[dangling_idx[i]]);
    *dsum = s;
}

// x' = alpha*(x @ A + dsum*p) + (1-alpha)*p with (x @ A)[k] = sum over j ascending of A[j,k]*x[j], summed from 0.0
// (scipy's transposed matvec); diff = |x' - x| for the convergence test.
__global__ void pr_step_kernel(const int *done, int32_t n, const uint32_t *roff, const int32_t *key, const double *val, const double *x, const double *dsum,
                               double alpha, double one_minus_alpha, double p, double *x_next, double *diff) {
    if (*done) return;
    const double dp = __dmul_rn(*dsum, p), tp = __dmul_rn(one_minus_alpha, p);
    for (int64_t k = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; k < n; k += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        double y = 0.0;
        for (int64_t r = roff[k]; r < roff[k + 1]; r++) y = __dadd_rn(y, __dmul_rn(val[r], x[key[r]]));
        const double xn = __dadd_rn(__dmul_rn(alpha, __dadd_rn(y, dp)), tp);
        x_next[k] = xn;
        diff[k] = fabs(__dsub_rn(xn, x[k]));
    }
}

// err = np.absolute(x' - x).sum() (pairwise over all N); stop when err < N*tol.  One thread: the sum's order is numpy's.
__global__ void pr_converge_kernel(int *done, int32_t n, const double *diff, double limit, int iteration, int *iterations) {
    if (*done) return;
    if (pairwise_sum(diff, n) < limit) { *done = 1; *iterations = iteration + 1; }
}

// ---------------------------------------------------------------- Brandes betweenness
// One warp per source of the batch.  The ordered walk supplied the queue (source, then its slice) with depths.  Pass 1:
// sigma[w] += sigma[v] for every v in queue order and every successor w one level deeper — a DiGraph row holds each neighbour
// once, so the lanes of one row never collide and each sigma[w] receives its terms in queue order of v (NetworkX builds P[w]
// in that order).  Pass 2: w in reverse queue order, coeff = (1 + delta[w]) / sigma[w], delta[v] += sigma[v] * coeff over the
// predecessors v one level up; each delta[v] receives its terms in decreasing queue position of w, as _accumulate_basic adds them.
// Per-source dense state [batch][n]: dist (-1 = unreached), sigma, delta; zeroed by the caller.
__global__ void brandes_kernel(int64_t nb, int32_t first_source, int32_t n, const uint32_t *foff, const int32_t *fnbr, const uint32_t *roff,
                               const int32_t *rnbr, const int64_t *q_start, const int32_t *q_count, const int32_t *nodes, const int32_t *depth,
                               int32_t *dist_all, double *sigma_all, double *delta_all) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
    for (int64_t b = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; b < nb; b += warps) {
        const int32_t s = first_source + static_cast<int32_t>(b);
        int32_t *dist = dist_all + b * static_cast<int64_t>(n);
        double *sigma = sigma_all + b * static_cast<int64_t>(n);
        double *delta = delta_all + b * static_cast<int64_t>(n);
        const int32_t *q = nodes + q_start[b];
        const int32_t *qd = depth + q_start[b];
        const int32_t cnt = q_count[b];
        for (int32_t i = lane; i < cnt; i += 32) dist[q[i]] = qd[i];
        if (lane == 0) { dist[s] = 0; sigma[s] = 1.0; }
        __syncwarp();
        for (int32_t i = -1; i < cnt; i++) {                 // queue position i + 1: -1 is the source
            const int32_t v = i < 0 ? s : q[i];
            const int32_t dn = (i < 0 ? 0 : qd[i]) + 1;
            const double sv = sigma[v];
            for (uint32_t e = foff[v] + lane; e < foff[v + 1]; e += 32) {
                const int32_t w = fnbr[e];
                if (dist[w] == dn) sigma[w] = __dadd_rn(sigma[w], sv);
            }
            __syncwarp();
        }
        for (int32_t i = cnt - 1; i >= 0; i--) {
            const int32_t w = q[i];
            const int32_t du = qd[i] - 1;
            const double coeff = __ddiv_rn(__dadd_rn(1.0, delta[w]), sigma[w]);
            for (uint32_t e = roff[w] + lane; e < roff[w + 1]; e += 32) {
                const int32_t v = rnbr[e];
                if (dist[v] == du) delta[v] = __dadd_rn(delta[v], __dmul_rn(sigma[v], coeff));
            }
            __syncwarp();
        }
    }
}

// b[v] += delta_s[v] for the batch's sources in source order; the source's own delta is not added.  Unreached nodes add 0.0.
__global__ void brandes_accumulate_kernel(int64_t nb, int32_t first_source, int32_t n, const double *delta_all, double *bc) {
    for (int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; v < n; v += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        double acc = bc[v];
        for (int64_t b = 0; b < nb; b++)
            if (first_source + b != v) acc = __dadd_rn(acc, delta_all[b * static_cast<int64_t>(n) + v]);
        bc[v] = acc;
    }
}

__global__ void scale_kernel(int32_t n, double scale, double *x) {
    for (int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; v < n; v += static_cast<int64_t>(gridDim.x) * blockDim.x)
        x[v] = __dmul_rn(x[v], scale);
}

// ---------------------------------------------------------------- bidirectional shortest paths (_bidirectional_pred_succ)
// One warp per (source, target) pair, pairs taken grid-stride; each warp owns one scratch slot: dense pred / succ maps
// (-1 absent, -2 None) and the forward / reverse lists, every discovered node appended once, each fringe a contiguous range.
// The forward fringe is expanded when it is no longer than the reverse one; fringe nodes are scanned in order, each row in
// dict order (32 entries per step, appended in lane order), and the search stops at the first w of the scan that the other
// side already holds — lanes after it in that step take no effect.  The path (pred chain reversed, then the succ chain) is
// bump-allocated in `out`; when it does not fit, only the total is counted and the caller re-runs with a larger arena.
constexpr int32_t SP_ABSENT = -1, SP_NONE = -2;

__device__ __forceinline__ bool sp_expand(int32_t lo, int32_t hi, const int32_t *list_in, const uint32_t *off, const int32_t *nbr, int32_t *mine,
                                          const int32_t *other, int32_t *list_out, int32_t &len, int32_t &meet) {
    const int lane = threadIdx.x & 31;
    for (int32_t i = lo; i < hi; i++) {
        const int32_t v = list_in[i];
        for (uint32_t base = off[v]; base < off[v + 1]; base += 32) {
            const uint32_t e = base + lane;
            const bool valid = e < off[v + 1];
            const int32_t w = valid ? nbr[e] : 0;
            const unsigned hit = __ballot_sync(0xFFFFFFFFu, valid && other[w] != SP_ABSENT);
            const int first = hit ? __ffs(hit) - 1 : 32;
            const bool fresh = valid && lane <= first && mine[w] == SP_ABSENT;
            const unsigned fm = __ballot_sync(0xFFFFFFFFu, fresh);
            if (fresh) {
                list_out[len + __popc(fm & ((1u << lane) - 1u))] = w;
                mine[w] = v;
            }
            len += __popc(fm);
            __syncwarp();
            if (hit) { meet = __shfl_sync(0xFFFFFFFFu, w, first); return true; }
        }
    }
    return false;
}

__global__ void bidir_paths_kernel(int64_t np, const int32_t *src, const int32_t *dst, int32_t n, const uint32_t *foff, const int32_t *fnbr,
                                   const uint32_t *roff, const int32_t *rnbr, int32_t *scratch, int64_t slots, int32_t *out, int64_t cap,
                                   unsigned long long *used, int64_t *p_start, int32_t *p_len) {
    const int lane = threadIdx.x & 31;
    const int64_t slot = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
    if (slot >= slots) return;
    int32_t *pm = scratch + slot * 4 * static_cast<int64_t>(n);
    int32_t *sm = pm + n, *F = sm + n, *R = F + n;
    for (int64_t q = slot; q < np; q += slots) {
        const int32_t s = src[q], t = dst[q];
        int32_t fn = 1, rn = 1, meet = -1;
        if (lane == 0) { F[0] = s; pm[s] = SP_NONE; R[0] = t; sm[t] = SP_NONE; }
        __syncwarp();
        if (s == t) meet = s;
        int32_t fl = 0, fh = 1, rl = 0, rh = 1;
        while (meet < 0 && fh > fl && rh > rl) {
            if (fh - fl <= rh - rl) {
                sp_expand(fl, fh, F, foff, fnbr, pm, sm, F, fn, meet);
                fl = fh; fh = fn;
            } else {
                sp_expand(rl, rh, R, roff, rnbr, sm, pm, R, rn, meet);
                rl = rh; rh = rn;
            }
        }
        int32_t len = 0;
        if (meet >= 0) {
            int32_t a = 0, b = 0;
            for (int32_t u = meet; u != SP_NONE; u = pm[u]) a++;
            for (int32_t u = sm[meet]; u != SP_NONE; u = sm[u]) b++;
            len = a + b;
            unsigned long long at = 0;
            if (lane == 0) at = atomicAdd(used, static_cast<unsigned long long>(len));
            at = __shfl_sync(0xFFFFFFFFu, at, 0);
            if (lane == 0) {
                p_start[q] = static_cast<int64_t>(at);
                if (static_cast<int64_t>(at) + len <= cap) {
                    int32_t k = a - 1;
                    for (int32_t u = meet; u != SP_NONE; u = pm[u]) out[at + k--] = u;
                    k = a;
                    for (int32_t u = sm[meet]; u != SP_NONE; u = sm[u]) out[at + k++] = u;
                }
            }
        } else if (lane == 0) {
            p_start[q] = 0;
        }
        if (lane == 0) p_len[q] = len;
        __syncwarp();
        for (int32_t i = lane; i < fn; i += 32) pm[F[i]] = SP_ABSENT;
        for (int32_t i = lane; i < rn; i += 32) sm[R[i]] = SP_ABSENT;
        __syncwarp();
    }
}

}  // namespace nx
}  // namespace abb
