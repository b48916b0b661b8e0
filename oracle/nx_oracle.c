/*
 * nx_oracle.c — CPU restatement of the two centralities of the reference's NetworkXBackend (agent_bom/graph_backend.py:
 * 230-242) as networkx 3.6.1 computes them:
 *
 *   nxo_pagerank     nx.pagerank (_pagerank_scipy: alpha 0.85, max_iter 100, tol 1e-6, weight "weight")
 *   nxo_betweenness  nx.betweenness_centrality (_single_source_shortest_path_basic + _accumulate_basic + _rescale)
 *
 * TEST INFRASTRUCTURE ONLY, like oracle.c: tests/test_networkx_backend.py pins it on the NetworkX goldens
 * (tests/golden/context/networkx_backend.json.gz), and the GPU tests compare the device with it at sizes NetworkX cannot reach.
 * Built on its own (oracle/nx_oracle.py) with -ffp-contract=off: every a*b+c below must round twice, as numpy and Python do.
 *
 * Graph: n nodes in node order; forward row u = G.succ[u] in dict order (foff/fnbr), reverse row u = G.pred[u] (roff/rnbr);
 * w[e] = weight of forward entry e.  No row repeats a neighbour.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* numpy's DOUBLE_pairwise_sum */
static double pairwise(const double *a, int64_t n) {
    if (n < 8) {
        double r = -0.0;
        for (int64_t i = 0; i < n; i++) r += a[i];
        return r;
    }
    if (n <= 128) {
        double r[8];
        for (int j = 0; j < 8; j++) r[j] = a[j];
        int64_t i = 8;
        for (; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; j++) r[j] += a[i + j];
        double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; i++) res += a[i];
        return res;
    }
    int64_t h = n / 2;
    h -= h % 8;
    return pairwise(a, h) + pairwise(a + h, n - h);
}

typedef struct { int32_t col; double w; } entry;
static int cmp_entry(const void *x, const void *y) {
    const entry *a = x, *b = y;
    return (a->col > b->col) - (a->col < b->col);
}

/* returns the iterations run, 0 when the power iteration did not converge */
int nxo_pagerank(int32_t n, const int64_t *foff, const int32_t *fnbr, const double *w, double *out) {
    if (n == 0) return 0;
    const double alpha = 0.85, tol = 1e-6;
    const int64_t m = foff[n];
    entry *row = malloc(sizeof(entry) * (size_t)(m ? m : 1));
    double *ws = malloc(sizeof(double) * (size_t)(m ? m : 1));
    double *inv = malloc(sizeof(double) * (size_t)n);
    /* scipy's CSR holds each row in ascending column order; A.sum(axis=1) is np.add.reduceat: w0 + pairwise(w1..) */
    for (int32_t i = 0; i < n; i++) {
        const int64_t a = foff[i], k = foff[i + 1] - a;
        for (int64_t e = 0; e < k; e++) { row[a + e].col = fnbr[a + e]; row[a + e].w = w[a + e]; }
        qsort(row + a, (size_t)k, sizeof(entry), cmp_entry);
        for (int64_t e = 0; e < k; e++) ws[a + e] = row[a + e].w;
        double s = 0.0;
        if (k == 1) s = ws[a];
        else if (k > 1) s = ws[a] + pairwise(ws + a + 1, k - 1);
        inv[i] = s != 0.0 ? 1.0 / s : 0.0;
    }
    /* x @ A: y[k] = sum over j ascending of (inv[j] * w[j,k]) * x[j], from 0.0 — built as column lists in ascending j.  scipy's
     * Q = dia_array((1/S, 0)) drops a zero diagonal entry, so a row with inv 0 (dangling, or a sum that overflowed to inf) has
     * no entries in Q @ A: it contributes 0.0 (adding +-0 leaves a finite y as it was), never inv * w = 0 * inf = NaN. */
    int64_t *coff = calloc((size_t)n + 1, sizeof(int64_t));
    for (int64_t e = 0; e < m; e++) coff[row[e].col + 1]++;
    for (int32_t k = 0; k < n; k++) coff[k + 1] += coff[k];
    int64_t *fill = malloc(sizeof(int64_t) * (size_t)n);
    memcpy(fill, coff, sizeof(int64_t) * (size_t)n);
    int32_t *csrc = malloc(sizeof(int32_t) * (size_t)(m ? m : 1));
    double *cval = malloc(sizeof(double) * (size_t)(m ? m : 1));
    for (int32_t j = 0; j < n; j++)
        for (int64_t e = foff[j]; e < foff[j + 1]; e++) {
            const int64_t at = fill[row[e].col]++;
            csrc[at] = j;
            cval[at] = inv[j] == 0.0 ? 0.0 : inv[j] * row[e].w;
        }
    double *x = malloc(sizeof(double) * (size_t)n), *xn = malloc(sizeof(double) * (size_t)n), *diff = malloc(sizeof(double) * (size_t)n);
    const double p = 1.0 / n;
    for (int32_t i = 0; i < n; i++) x[i] = p;
    int iterations = 0;
    for (int it = 0; it < 100 && !iterations; it++) {
        double dsum = 0.0;                       /* Python's sum(x[is_dangling]): sequential in index order */
        for (int32_t i = 0; i < n; i++)
            if (inv[i] == 0.0) dsum += x[i];
        for (int32_t k = 0; k < n; k++) {
            double y = 0.0;
            for (int64_t e = coff[k]; e < coff[k + 1]; e++) y += cval[e] * x[csrc[e]];
            xn[k] = alpha * (y + dsum * p) + (1.0 - alpha) * p;
            diff[k] = fabs(xn[k] - x[k]);
        }
        double *t = x; x = xn; xn = t;
        if (pairwise(diff, n) < (double)n * tol) iterations = it + 1;
    }
    if (iterations) memcpy(out, x, sizeof(double) * (size_t)n);
    free(row); free(ws); free(inv); free(coff); free(fill); free(csrc); free(cval); free(x); free(xn); free(diff);
    return iterations;
}

/* Brandes from one source s into delta[n] (zeroed on entry); returns the forward entries scanned */
static int64_t brandes_one(int32_t n, const int64_t *foff, const int32_t *fnbr, const int64_t *roff, const int32_t *rnbr, int32_t s,
                           int32_t *queue, int32_t *dist, double *sigma, double *delta) {
    int64_t scanned = 0, head = 0, tail = 0;
    queue[tail++] = s; dist[s] = 0; sigma[s] = 1.0;
    while (head < tail) {
        const int32_t v = queue[head++];
        for (int64_t e = foff[v]; e < foff[v + 1]; e++) {
            const int32_t w = fnbr[e];
            if (dist[w] < 0) { queue[tail++] = w; dist[w] = dist[v] + 1; }
            if (dist[w] == dist[v] + 1) sigma[w] += sigma[v];
        }
        scanned += foff[v + 1] - foff[v];
    }
    /* down to queue position 1: the source (position 0) has no predecessor one level up, and at dist[s] - 1 == -1 its scan would
     * match every unreached in-neighbour, adding sigma 0 * coeff — NaN once path counts overflow to inf */
    for (int64_t i = tail - 1; i >= 1; i--) {
        const int32_t w = queue[i];
        const double coeff = (1.0 + delta[w]) / sigma[w];
        for (int64_t e = roff[w]; e < roff[w + 1]; e++) {
            const int32_t v = rnbr[e];
            if (dist[v] == dist[w] - 1) delta[v] += sigma[v] * coeff;
        }
    }
    for (int64_t i = 0; i < tail; i++) { dist[queue[i]] = -1; sigma[queue[i]] = 0.0; }
    delta[s] = 0.0;                              /* the source's own delta is not added */
    return scanned;
}

/* sources run in parallel in batches; each batch's deltas are added into out in source order */
int64_t nxo_betweenness(int32_t n, const int64_t *foff, const int32_t *fnbr, const int64_t *roff, const int32_t *rnbr, double *out, int threads) {
    int nt = threads > 0 ? threads : 1;
#ifdef _OPENMP
    if (threads <= 0) nt = omp_get_max_threads();
#endif
    for (int32_t v = 0; v < n; v++) out[v] = 0.0;
    if (n == 0) return 0;
    const int64_t B = (int64_t)nt * 8;
    double *delta = malloc(sizeof(double) * (size_t)B * (size_t)n);
    int64_t scanned = 0;
    for (int64_t s0 = 0; s0 < n; s0 += B) {
        const int64_t nb = (n - s0) < B ? (n - s0) : B;
        memset(delta, 0, sizeof(double) * (size_t)nb * (size_t)n);
#pragma omp parallel num_threads(nt) reduction(+ : scanned)
        {
            int32_t *queue = malloc(sizeof(int32_t) * (size_t)n), *dist = malloc(sizeof(int32_t) * (size_t)n);
            double *sigma = calloc((size_t)n, sizeof(double));
            for (int32_t v = 0; v < n; v++) dist[v] = -1;
#pragma omp for schedule(dynamic, 1)
            for (int64_t b = 0; b < nb; b++)
                scanned += brandes_one(n, foff, fnbr, roff, rnbr, (int32_t)(s0 + b), queue, dist, sigma, delta + b * (int64_t)n);
            free(queue); free(dist); free(sigma);
        }
        for (int64_t b = 0; b < nb; b++)
            for (int32_t v = 0; v < n; v++) out[v] += delta[b * (int64_t)n + v];
    }
    free(delta);
    if (n > 2) {
        const double scale = 1.0 / (double)(((int64_t)n - 1) * ((int64_t)n - 2));
        for (int32_t v = 0; v < n; v++) out[v] *= scale;
    }
    return scanned;
}
