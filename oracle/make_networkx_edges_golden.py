#!/usr/bin/env python3
"""Generate tests/golden/context/networkx_edges.json.gz: the NetworkX backend's answers at the edges the estate golden does not
reach, computed by networkx itself (``nx.pagerank``, ``nx.betweenness_centrality``, ``nx.shortest_path`` and the reference
backend's ``bfs`` = ``bfs_tree`` + one ``shortest_path`` per tree node).

Every graph is rebuilt from its generator parameters by ``case_ops`` (importable without networkx: the tests replay the same op
sequences into the backend and the oracle), so the fixture stores parameters and answers only:

- ``weights:*`` — a seeded 200-node DiGraph whose node ``x`` has one row of edge weights at the edge of IEEE arithmetic: zero,
  all-zero, zero-sum, negative and ``-0.0`` weights, a row sum that overflows to +-inf, ``inf`` / ``-inf`` / ``NaN`` weights,
  subnormal weights and a row sum whose inverse overflows.  PageRank and its iteration count, or ``iterations == 0`` where
  networkx raises ``PowerIterationFailedConvergence``.
- ``rows`` — one node per out-degree in {1..16, 127..130, 255..257, 1023..1025, 8191..8193, 65537} (every length around
  numpy's pairwise-sum block boundaries) with log-uniform weights from about 1e-8 to 1e8, and a sink with 20 000 in-edges from
  rows of mixed degree.  PageRank as a SHA-256 of the f64 scores in node order, plus the scores of the nodes of interest.
- ``chain`` — a width-2, 1 100-layer complete-bipartite chain: path counts overflow to inf, so betweenness is NaN on most nodes.
- ``long-path`` — a 4 000-node path with a diamond at every third node (the forward and the reverse search prefer different
  sides of it) and a few back edges, and far-apart pairs whose answers total well over 65 536 nodes and 8 per pair.

    python oracle/make_networkx_edges_golden.py
"""

from __future__ import annotations

import gzip
import hashlib
import json
import math
import platform
import random
from pathlib import Path

OUT = Path(__file__).resolve().parents[1] / "tests" / "golden" / "context" / "networkx_edges.json.gz"

INF, NAN = float("inf"), float("nan")
# label -> weights of node x's row, to targets t0, t1, ... in that order
WEIGHT_ROWS = {
    "zero-weights": [0.0, 1.0, 0.0, 2.5],
    "all-zero-row": [0.0, 0.0, 0.0],
    "zero-sum-row": [1.0, -1.0],
    "negative-weights": [-0.5, 2.0, 1.0, -0.25],
    "negative-zero": [-0.0, 1.5],
    "negative-zero-row": [-0.0, -0.0],
    "overflow-row-sum": [1e308, 1e308],
    "negative-overflow-row-sum": [-1e308, -1e308],
    "inf-weight": [INF, 1.0],
    "negative-inf-weight": [1.0, -INF],
    "inf-minus-inf": [INF, -INF],
    "subnormal-weights": [5e-324, 1e-310],
    "tiny-row-sum": [1e-309, 1e-310],
    "nan-weight": [NAN, 1.0],
}
ROW_DEGREES = [*range(1, 17), *range(127, 131), *range(255, 258), *range(1023, 1026), *range(8191, 8194), 65537]


def _weight(rng: random.Random) -> float:
    """Log-uniform in [2^-27, 2^27) (about 1e-8 to 1e8), exactly representable: built with ldexp, no libm rounding."""
    return math.ldexp(1.0 + rng.getrandbits(30) / (1 << 30), rng.randint(-27, 26))


def weights_ops(row: list[float], seed: int = 7) -> list:
    rng = random.Random(seed)
    names = [f"n{i:03d}" for i in range(199)]
    ops = [["n", v, "node", v, {}] for v in names]
    for _ in range(600):
        s, t = rng.sample(names, 2)
        ops.append(["e", s, t, "rel", rng.choice([1.0, 0.5, 2.0, 0.25, 3.0]), True, {}])
    for s in rng.sample(names, 12):
        ops.append(["e", s, "x", "rel", rng.choice([1.0, 0.5, 2.0]), True, {}])
    for t, w in zip(rng.sample(names, len(row)), row):
        ops.append(["e", "x", t, "rel", w, True, {}])
    return ops


def rows_ops(seed: int = 11, pool: int = 70_000, sink_in: int = 20_000) -> list:
    rng = random.Random(seed)
    ops = [["n", f"p{i:05d}", "node", "", {}] for i in range(pool)]
    for k in ROW_DEGREES:
        for t in rng.sample(range(pool), k):
            ops.append(["e", f"d{k}", f"p{t:05d}", "rel", _weight(rng), True, {}])
    for s in rng.sample(range(pool), sink_in):
        ops.append(["e", f"p{s:05d}", "sink", "rel", _weight(rng), True, {}])
        for t in rng.sample(range(pool), rng.choice([0, 0, 0, 1, 2, 3, 7, 8, 15])):
            if t != s:
                ops.append(["e", f"p{s:05d}", f"p{t:05d}", "rel", _weight(rng), True, {}])
    return ops


def chain_ops(width: int = 2, layers: int = 1100) -> list:
    return [["e", f"L{i:04d}_{a}", f"L{i + 1:04d}_{b}", "next", 1.0, True, {}] for i in range(layers - 1) for a in range(width) for b in range(width)]


def long_path_ops(seed: int = 5, length: int = 4000, back_edges: int = 6) -> list:
    """Path p0000 -> p0001 -> ...; at every third node i a diamond i -> d_i -> i+2 whose edges are added so that succ[i] lists
    i+1 first but pred[i+2] lists d_i first; a few long back edges."""
    rng = random.Random(seed)
    p = [f"p{i:04d}" for i in range(length)]
    ops = []
    for i in range(length - 1):
        ops.append(["e", p[i], p[i + 1], "next", 1.0, True, {}])
        if i % 3 == 0 and i + 2 < length:
            ops.append(["e", p[i], f"d{i:04d}", "side", 1.0, True, {}])
            ops.append(["e", f"d{i:04d}", p[i + 2], "side", 1.0, True, {}])
    for _ in range(back_edges):
        j = rng.randrange(length // 2, length)
        ops.append(["e", p[j], p[rng.randrange(0, j - length // 4)], "back", 1.0, True, {}])
    return ops


def long_path_pairs(ids: list[str], seed: int = 5, pairs: int = 160) -> list[list[int]]:
    """Far-apart path nodes, both directions (backwards only through the back edges, or not at all)."""
    rng = random.Random(seed + 1)
    path = [i for i, v in enumerate(ids) if v.startswith("p")]
    out = []
    while len(out) < pairs:
        a, b = rng.sample(range(len(path)), 2)
        if abs(a - b) >= 1000:
            out.append([path[a], path[b]])
    return out


def case_ops(params: dict) -> list:
    kind = params["kind"]
    if kind == "weights":
        return weights_ops(params["row"], params["seed"])
    if kind == "rows":
        return rows_ops(params["seed"], params["pool"], params["sink_in"])
    if kind == "chain":
        return chain_ops(params["width"], params["layers"])
    if kind == "long-path":
        return long_path_ops(params["seed"], params["length"], params["back_edges"])
    raise ValueError(kind)


def digraph(ops):
    """The reference NetworkXBackend's graph: nx.DiGraph, undirected edges added both ways, a re-added edge takes the new weight."""
    import networkx as nx

    g = nx.DiGraph()
    for op in ops:
        if op[0] == "n":
            g.add_node(op[1])
        else:
            g.add_edge(op[1], op[2], weight=op[4])
            if not op[5]:
                g.add_edge(op[2], op[1], weight=op[4])
    return g


def pagerank_and_iterations(g) -> tuple[list[float] | None, int]:
    """nx.pagerank and the power iterations it ran: the least max_iter that converges (convergence at iteration k does not depend
    on max_iter >= k, so a bisection finds it); (None, 0) when 100 iterations do not converge."""
    import networkx as nx

    def run(max_iter):
        try:
            return nx.pagerank(g, max_iter=max_iter)
        except nx.PowerIterationFailedConvergence:
            return None

    full = run(100)
    if full is None:
        return None, 0
    lo, hi = 1, 100
    while lo < hi:
        mid = (lo + hi) // 2
        if run(mid) is None:
            lo = mid + 1
        else:
            hi = mid
    assert run(lo) == full
    return [full[v] for v in g], lo


def score_digest(scores: list[float]) -> str:
    import numpy as np

    return hashlib.sha256(np.asarray(scores, dtype="<f8").tobytes()).hexdigest()


def main():
    import networkx as nx
    import numpy as np
    import scipy

    cases = []
    for label, row in WEIGHT_ROWS.items():
        params = {"kind": "weights", "seed": 7, "row": row}
        g = digraph(case_ops(params))
        pr, it = pagerank_and_iterations(g)
        cases.append({"label": f"weights:{label}", "params": params, "nodes": len(g), "pagerank": pr, "iterations": it})
        print(f"weights:{label}: {it} iterations", flush=True)

    params = {"kind": "rows", "seed": 11, "pool": 70_000, "sink_in": 20_000}
    g = digraph(case_ops(params))
    ids = list(g)
    pr, it = pagerank_and_iterations(g)
    assert it > 0
    index = {v: i for i, v in enumerate(ids)}
    rng = random.Random(12)
    probe = sorted({index[f"d{k}"] for k in ROW_DEGREES} | {index["sink"]} | set(rng.sample(range(len(ids)), 500)))
    cases.append({"label": "rows", "params": params, "nodes": len(ids), "iterations": it, "pagerank_sha256": score_digest(pr),
                  "pagerank_at": [[i, pr[i]] for i in probe]})
    print(f"rows: {len(ids)} nodes, {g.number_of_edges()} edges, {it} iterations", flush=True)

    params = {"kind": "chain", "width": 2, "layers": 1100}
    g = digraph(case_ops(params))
    pr, it = pagerank_and_iterations(g)
    bc = nx.betweenness_centrality(g)
    cases.append({"label": "chain", "params": params, "nodes": len(g), "pagerank": pr, "iterations": it, "betweenness": [bc[v] for v in g]})
    print(f"chain: {len(g)} nodes, {sum(math.isnan(x) for x in bc.values())} NaN betweenness scores", flush=True)

    params = {"kind": "long-path", "seed": 5, "length": 4000, "back_edges": 6}
    g = digraph(case_ops(params))
    ids = list(g)
    index = {v: i for i, v in enumerate(ids)}
    shortest = []
    for s, t in long_path_pairs(ids):
        try:
            p = [index[v] for v in nx.shortest_path(g, ids[s], ids[t])]
        except nx.NetworkXNoPath:
            p = None
        shortest.append([s, t, p])
    bfs = []
    for s in (0, 1, 2, index["p2000"], index["p3999"]):
        for d in (4, 6):
            tree = nx.bfs_tree(g, ids[s], depth_limit=d)
            bfs.append([s, d, [[index[v] for v in nx.shortest_path(g, ids[s], u)] for u in tree if u != ids[s]]])
    total = sum(len(p) for _, _, p in shortest if p)
    assert total > max(65_536, 8 * len(shortest))
    cases.append({"label": "long-path", "params": params, "nodes": len(ids), "shortest": shortest, "bfs": bfs})
    print(f"long-path: {len(ids)} nodes, {len(shortest)} pairs, {sum(p is None for _, _, p in shortest)} without a path, "
          f"{total} path nodes", flush=True)

    doc = {"versions": {"networkx": nx.__version__, "scipy": scipy.__version__, "numpy": np.__version__, "python": platform.python_version()},
           "host": {"machine": platform.machine(), "processor": platform.processor() or platform.machine(), "system": platform.system()},
           "cases": cases}
    OUT.write_bytes(gzip.compress(json.dumps(doc, separators=(",", ":"), sort_keys=True).encode(), mtime=0))
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
