#!/usr/bin/env python3
"""Generate tests/golden/context/networkx_backend.json.gz with the UNMODIFIED reference's ``NetworkXBackend``.

Runs only where the reference tree and networkx are importable (the tests read the fixture alone).  Every case is an op
sequence (``["n", id, kind, label, meta]`` / ``["e", s, t, kind, weight, directed, meta]``) replayed into the reference backend
— for the bridges, the calls the reference's ``from_unified_graph`` / ``from_context_graph`` made — with every protocol
method's answer: PageRank and betweenness of every node (exact floats, node order), ``bottleneck_nodes`` for top 5, 20 and n,
``bfs`` for several sources and depths, and ``shortest_path`` pairs including missing, equal and unreachable ones.

    python oracle/make_networkx_golden.py            # writes the fixture
    python oracle/make_networkx_golden.py --time     # instead times the reference on one CPU core (profiles/centrality_reference.json)
"""

from __future__ import annotations

import gzip
import json
import platform
import random
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import OUT, estate, mesh_inventory  # noqa: E402

import networkx as nx  # noqa: E402
import numpy as np  # noqa: E402
import scipy  # noqa: E402
from agent_bom import graph_backend as gb  # noqa: E402


class Recording(gb.NetworkXBackend):
    def __init__(self):
        super().__init__()
        self.ops = []

    def add_node(self, node_id, kind, label, **metadata):
        self.ops.append(["n", node_id, kind, label, dict(metadata)])
        super().add_node(node_id, kind, label, **metadata)

    def add_edge(self, source, target, kind, weight=1.0, *, directed=False, **metadata):
        self.ops.append(["e", source, target, kind, weight, directed, dict(metadata)])
        super().add_edge(source, target, kind, weight, directed=directed, **metadata)


def bridged(fn, *args):
    """Run a reference bridge with the recording backend; returns it."""
    rec = Recording()
    saved = gb.get_backend
    gb.get_backend = lambda backend="auto": rec
    try:
        fn(*args)
    finally:
        gb.get_backend = saved
    return rec


def replayed(ops):
    rec = Recording()
    for op in ops:
        if op[0] == "n":
            rec.add_node(op[1], op[2], op[3], **op[4])
        else:
            rec.add_edge(op[1], op[2], op[3], op[4], directed=op[5], **op[6])
    return rec


def record(label, b, rng, small):
    ids = list(b._graph)
    doc = {"label": label, "ops": b.ops, "node_count": b.node_count(), "edge_count": b.edge_count()}
    pr = b.centrality_scores()
    bc = nx.betweenness_centrality(b._graph)
    assert list(pr) == ids
    doc["pagerank"] = [pr[v] for v in ids]
    doc["betweenness"] = [bc[v] for v in ids]
    doc["node_ids"] = ids
    for key, top in (("bottleneck_5", 5), ("bottleneck_20", 20), ("bottleneck_n", len(ids))):
        doc[key] = [list(x) for x in b.bottleneck_nodes(top)]
    sources = ids[:2] + rng.sample(ids, min(4, len(ids))) + ["missing"] if ids else ["missing"]
    doc["bfs"] = [[s, d, b.bfs(s, d)] for s in sources for d in ((0, 1, 2, 4, 6) if small else (1, 4))]
    pairs = [[rng.choice(ids), rng.choice(ids)] for _ in range(40 if small else 60)] if ids else []
    pairs += [["missing", ids[0] if ids else "x"], [ids[0] if ids else "x", "missing"]] + ([[ids[0], ids[0]]] if ids else [])
    doc["shortest"] = [[s, t, b.shortest_path(s, t)] for s, t in pairs]
    if small:
        doc["to_dict"] = b.to_dict()
        doc["neighbors"] = {v: b.neighbors(v) for v in ids[:30]}
        doc["has_edge"] = [[s, t, b.has_edge(s, t)] for s, t in pairs[:30]]
    print(f"{label}: {len(ids)} nodes, {b._graph.number_of_edges()} edges", flush=True)
    return doc


def random_ops(seed):
    """Weighted op soup: implicit endpoints, re-added nodes and edges with new attributes, self loops, dangling nodes, and hubs whose
    rows are longer than 128 and than 1 024 entries."""
    rng = random.Random(seed)
    n = rng.randint(20, 400)
    names = [f"n{i:04d}" for i in rng.sample(range(10 * n), n)]
    ops = [["n", v, rng.choice(["agent", "server", "tool"]), v.upper(), {"tier": rng.randint(0, 3)} if rng.random() < 0.3 else {}] for v in names]
    for _ in range(rng.randint(n, 5 * n)):
        u = f"x{rng.randint(0, 5 * n)}" if rng.random() < 0.15 else rng.choice(names)
        v = rng.choice(names) if rng.random() < 0.9 else rng.choice(["hub", "sink"])
        ops.append(["e", u, v, rng.choice(["uses", "provides"]), rng.choice([1.0, 0.5, 0.3, 2.7, 1 / 3, 2]), rng.random() < 0.6, {"note": "x"} if rng.random() < 0.1 else {}])
        if rng.random() < 0.05:
            ops.append(["e", u, u, "self", rng.choice([1.0, 0.25]), True, {}])
        if rng.random() < 0.05:
            ops.append(["n", rng.choice(names), "agent", "re-added", {"again": True}])
    hub_len = 200 if seed % 2 else 1500
    for k in range(hub_len):
        ops.append(["e", "hub", rng.choice(names) if k < n else f"leaf{k}", "fan", rng.choice([0.1, 0.7, 1.3]), True, {}])
    for k in range(min(hub_len, 1100)):
        ops.append(["e", f"in{k % 300}", "sink", "fan", rng.choice([0.2, 1.0]), True, {}])
    for _ in range(n // 10):
        ops.append(["e", rng.choice(names), rng.choice(names), "uses", rng.choice([4.0, 0.125]), rng.random() < 0.5, {}])   # re-added pairs
    return ops


def bipartite_chain(width=20, layers=14):
    """Layered complete-bipartite chain: path counts reach width**(layers-1) > 2**53."""
    ops = []
    for i in range(layers - 1):
        for a in range(width):
            for b in range(width):
                ops.append(["e", f"L{i:02d}_{a:02d}", f"L{i + 1:02d}_{b:02d}", "next", 1.0, True, {}])
    return ops


def main():
    rng = random.Random(2145)
    cases = []
    cent = json.loads(gzip.decompress((OUT / "context" / "centrality.json.gz").read_bytes()))
    for d in cent["backends"]:
        cases.append(record(f"centrality:{d['label']}", replayed(d["ops"]), rng, True))
    mesh = mesh_inventory()
    ub = bridged(gb.from_unified_graph, mesh)
    cases.append(record("mesh:from_unified_graph", ub, rng, True))
    cg = {"nodes": [{"id": n["id"], "kind": n["kind"], "label": n["label"]} for n in ub.to_dict()["nodes"]], "edges": ub.to_dict()["edges"]}
    cases.append(record("mesh:from_context_graph", bridged(gb.from_context_graph, cg), rng, True))
    for seed in range(6):
        cases.append(record(f"random:{seed}", replayed(random_ops(seed)), rng, True))
    cases.append(record("bipartite-chain", replayed(bipartite_chain()), rng, False))
    cases.append(record("empty", replayed([]), rng, True))
    cases.append(record("single", replayed([["n", "a", "agent", "a", {}]]), rng, True))
    cases.append(record("pair", replayed([["e", "a", "b", "uses", 2.0, True, {}]]), rng, True))
    for agents in (40, 150):
        cases.append(record(f"estate:{agents}", bridged(gb.from_unified_graph, estate(agents)), rng, False))
    doc = {"versions": {"networkx": nx.__version__, "scipy": scipy.__version__, "numpy": np.__version__, "python": platform.python_version()},
           "host": {"machine": platform.machine(), "processor": platform.processor() or platform.machine(), "system": platform.system()},
           "cases": cases}
    path = OUT / "context" / "networkx_backend.json.gz"
    path.write_bytes(gzip.compress(json.dumps(doc, separators=(",", ":"), sort_keys=True).encode(), mtime=0))
    print(f"wrote {path} ({path.stat().st_size} bytes)")


def time_reference(budget_s: float = 120.0):
    """Wall time of the reference's centrality_scores / bottleneck_nodes (first call each) on generator estates through its
    from_unified_graph, smallest first, until one call exceeds the budget."""
    rows = []
    for agents in (40, 150, 1000):
        b = gb.from_unified_graph(estate(agents), backend="networkx")
        row = {"agents": agents, "nodes": b.node_count(), "directed_edges": b._graph.number_of_edges()}
        for name, fn in (("centrality_scores_s", b.centrality_scores), ("bottleneck_nodes_5_s", lambda: b.bottleneck_nodes(5))):
            t0 = time.perf_counter()
            fn()
            row[name] = time.perf_counter() - t0
        rows.append(row)
        print(row, flush=True)
        if row["bottleneck_nodes_5_s"] > budget_s / 10:
            break
    out = {"what": "reference NetworkXBackend, unmodified, one CPU core, seed 2145 generator estates",
           "versions": {"networkx": nx.__version__, "scipy": scipy.__version__, "numpy": np.__version__, "python": platform.python_version()},
           "host": {"machine": platform.machine(), "processor": platform.processor() or platform.machine()}, "estates": rows}
    path = Path(__file__).resolve().parents[1] / "profiles" / "centrality_reference.json"
    path.write_text(json.dumps(out, indent=1))
    print(f"wrote {path}")


if __name__ == "__main__":
    time_reference() if "--time" in sys.argv else main()
