"""B200Backend — drop-in for the reference's ``GraphBackend`` protocol (``/root/reference/src/agent_bom/graph_backend.py:23-38``).

Same methods, argument meaning and return shapes as ``InMemoryBackend`` (``:41-155``): nodes are attribute dicts,
edges live in a dict-of-dicts adjacency (``add_edge`` is undirected unless ``directed=True``; re-adding a pair
overwrites its attributes but keeps its place in the neighbour order), ``bfs`` returns one path per reached node in
discovery order, ``shortest_path`` the first-discoverer path, ``centrality_scores`` degree centrality and
``bottleneck_nodes`` the 50-source sampled score.  The traversals (``bfs``, ``shortest_path``, ``bottleneck_nodes``)
run on the GPU through the ordered walk engine; the adjacency is exported to a CSR lazily and re-exported after a
mutation.  ``get_backend`` / ``from_context_graph`` / ``from_unified_graph`` mirror ``:245-306``.

B200NetworkXBackend (name ``"b200-networkx"``) is the drop-in for the reference's other backend, ``NetworkXBackend``
(``:158-242``): an ``nx.DiGraph`` on the host, with PageRank, exact betweenness and NetworkX's bidirectional shortest paths
computed on the GPU.
"""

from __future__ import annotations

from collections import defaultdict
from typing import Protocol, runtime_checkable

import numpy as np

from . import _lib
from .graph import csr as csrmod
from .graph.schema import ENTITY_CODE_GHOST, enum_value

_SAMPLE = 50      # sources sampled by bottleneck_nodes (graph_backend.py:135)


@runtime_checkable
class GraphBackend(Protocol):
    """The reference's protocol (graph_backend.py:23-38), restated so callers can ``isinstance``-check a backend."""

    def add_node(self, node_id: str, kind: str, label: str, **metadata: object) -> None: ...
    def add_edge(self, source: str, target: str, kind: str, weight: float = 1.0, *, directed: bool = False, **metadata: object) -> None: ...
    def has_node(self, node_id: str) -> bool: ...
    def has_edge(self, source: str, target: str) -> bool: ...
    def neighbors(self, node_id: str) -> list[str]: ...
    def bfs(self, source: str, max_depth: int = 4) -> list[list[str]]: ...
    def shortest_path(self, source: str, target: str) -> list[str] | None: ...
    def node_count(self) -> int: ...
    def edge_count(self) -> int: ...
    def to_dict(self) -> dict: ...
    def centrality_scores(self) -> dict[str, float]: ...
    def bottleneck_nodes(self, top_n: int = 5) -> list[tuple[str, float]]: ...


class B200Backend:
    name = "b200"

    def __init__(self, device: int = 0):
        self._nodes: dict[str, dict] = {}
        self._adj: dict[str, dict[str, dict]] = defaultdict(dict)
        self._edge_count = 0
        self._device = device
        self._csr: csrmod.HostCSR | None = None
        self._dg = None

    # ── mutation ────────────────────────────────────────────────────────
    def _invalidate(self) -> None:
        self._csr = None
        if self._dg is not None:
            self._dg.close()
            self._dg = None

    def add_node(self, node_id: str, kind: str, label: str, **metadata: object) -> None:
        self._nodes[node_id] = {"kind": kind, "label": label, **metadata}
        self._invalidate()

    def add_edge(self, source: str, target: str, kind: str, weight: float = 1.0, *, directed: bool = False, **metadata: object) -> None:
        self._adj[source][target] = {"kind": kind, "weight": weight, **metadata}
        if not directed:
            self._adj[target][source] = {"kind": kind, "weight": weight, **metadata}
        self._edge_count += 1
        self._invalidate()

    # ── point queries (host) ────────────────────────────────────────────
    def has_node(self, node_id: str) -> bool:
        return node_id in self._nodes

    def has_edge(self, source: str, target: str) -> bool:
        return target in self._adj.get(source, {})

    def neighbors(self, node_id: str) -> list[str]:
        return list(self._adj.get(node_id, {}).keys())

    def node_count(self) -> int:
        return len(self._nodes)

    def edge_count(self) -> int:
        return self._edge_count

    def to_dict(self) -> dict:
        return {
            "nodes": [{"id": nid, **data} for nid, data in self._nodes.items()],
            "edges": [{"source": src, "target": tgt, **data} for src, targets in self._adj.items() for tgt, data in targets.items() if src < tgt],
            "stats": {"node_count": self.node_count(), "edge_count": self.edge_count()},
        }

    def centrality_scores(self) -> dict[str, float]:
        if not self._nodes:
            return {}
        max_possible = max(len(self._nodes) - 1, 1)
        return {nid: len(self._adj.get(nid, {})) / max_possible for nid in self._nodes}

    # ── device export ───────────────────────────────────────────────────
    @property
    def csr(self) -> csrmod.HostCSR:
        """Adjacency rows in neighbour (dict) order; ids without a node record become ghost rows after the real ones."""
        if self._csr is None:
            ids = list(self._nodes)
            index = {nid: i for i, nid in enumerate(ids)}
            n_real = len(ids)
            src: list[int] = []
            dst: list[int] = []
            for s, nbrs in self._adj.items():
                si = index.get(s)
                if si is None:
                    si = index[s] = len(ids)
                    ids.append(s)
                for t in nbrs:
                    ti = index.get(t)
                    if ti is None:
                        ti = index[t] = len(ids)
                        ids.append(t)
                    src.append(si)
                    dst.append(ti)
            node_type = np.zeros(len(ids), dtype=np.uint8)
            node_type[n_real:] = ENTITY_CODE_GHOST
            ne = len(src)
            c = csrmod.from_arrays(ids, node_type, np.asarray(src, dtype=np.int32), np.asarray(dst, dtype=np.int32), np.zeros(ne, dtype=np.uint8),
                                   np.full(ne, csrmod.EDGE_TRAVERSABLE, dtype=np.uint8), n_real=n_real)
            c.index = index
            self._csr = c
        return self._csr

    @property
    def device_graph(self):
        if self._dg is None:
            from .engine import DeviceGraph

            self._dg = DeviceGraph.upload(self.csr, self._device)
        return self._dg

    # ── traversals (GPU) ────────────────────────────────────────────────
    def bfs(self, source: str, max_depth: int = 4) -> list[list[str]]:
        """One path per node reached within ``max_depth`` hops, in discovery order (``:67-83``)."""
        if source not in self._nodes:
            return []
        c = self.csr
        res = self.device_graph.bfs_many(np.asarray([c.index[source]], dtype=np.int32), max_depth, False)
        ids = c.node_ids
        nodes, parent = res.slice(0).tolist(), res.aux(0, "parent").tolist()
        paths: list[list[str]] = []
        for i, u in enumerate(nodes):
            p = parent[i]                      # queue position of the first discoverer: 0 = the source, k > 0 = emitted entry k-1
            paths.append(([source] if p <= 0 else paths[p - 1]) + [ids[u]])
        return paths

    def shortest_path(self, source: str, target: str) -> list[str] | None:
        if source not in self._nodes or target not in self._nodes:
            return None
        if source == target:
            return [source]
        c = self.csr
        s, t = c.index[source], c.index[target]
        res = self.device_graph.shortest_path_many(np.asarray([s], dtype=np.int32), np.asarray([t], dtype=np.int32))
        if not (int(res.flags[0]) & _lib.QFLAG_TARGET_FOUND):
            return None
        nodes, parent = res.slice(0), res.aux(0, "parent")
        i = len(nodes) - 1
        while nodes[i] != t:
            i -= 1
        path = []
        while i >= 0:
            path.append(c.node_ids[int(nodes[i])])
            i = int(parent[i])
        return path[::-1]

    def bottleneck_nodes(self, top_n: int = 5) -> list[tuple[str, float]]:
        """Sampled betweenness approximation (``:127-155``): BFS from the first 50 nodes, +1 for every node strictly inside a
        first-discoverer path; normalised by the grand total, highest first, ties in node order."""
        if not self._nodes:
            return []
        c = self.csr
        sample = np.arange(min(_SAMPLE, c.n_real), dtype=np.int32)
        return rank_bottlenecks(c, self.device_graph.bottleneck_scores(sample), top_n)

    @classmethod
    def from_unified_graph(cls, graph, device: int = 0) -> "B200Backend":
        return from_unified_graph(graph, device=device)


class B200NetworkXBackend:
    """Drop-in for ``NetworkXBackend`` (graph_backend.py:158-242) with the host semantics of an ``nx.DiGraph``: ``add_edge``
    creates missing endpoints as attribute-less nodes; adding a node or an edge again merges its attributes into the existing
    entry, which keeps its position; ``edge_count`` is ``number_of_edges() // 2`` (the reference's count, also for directed-only
    graphs).  ``centrality_scores`` is ``nx.pagerank``, ``bottleneck_nodes`` exact ``nx.betweenness_centrality``, ``bfs`` /
    ``shortest_path`` use ``nx.shortest_path``'s bidirectional search — all on the GPU, bit for bit with networkx 3.6.1."""

    name = "b200-networkx"

    def __init__(self, device: int = 0):
        self._nodes: dict[str, dict] = {}
        self._succ: dict[str, dict[str, dict]] = {}
        self._edges: list[tuple[str, str]] = []     # first insertion order: rows of both CSR directions keep dict order
        self._device = device
        self._csr: csrmod.HostCSR | None = None
        self._weights: np.ndarray | None = None
        self._dg = None

    # ── mutation ────────────────────────────────────────────────────────
    def _invalidate(self) -> None:
        self._csr = self._weights = None
        if self._dg is not None:
            self._dg.close()
            self._dg = None

    def _ensure_node(self, node_id: str) -> dict:
        data = self._nodes.get(node_id)
        if data is None:
            data = self._nodes[node_id] = {}
            self._succ[node_id] = {}
            self._invalidate()
        return data

    def _put_edge(self, source: str, target: str, attrs: dict) -> None:
        self._ensure_node(source)
        self._ensure_node(target)
        row = self._succ[source]
        if target not in row:
            row[target] = {}
            self._edges.append((source, target))
        row[target].update(attrs)

    def add_node(self, node_id: str, kind: str, label: str, **metadata: object) -> None:
        self._ensure_node(node_id).update({"kind": kind, "label": label, **metadata})

    def add_edge(self, source: str, target: str, kind: str, weight: float = 1.0, *, directed: bool = False, **metadata: object) -> None:
        self._put_edge(source, target, {"kind": kind, "weight": weight, **metadata})
        if not directed:
            self._put_edge(target, source, {"kind": kind, "weight": weight, **metadata})
        self._invalidate()                  # a merged weight changes PageRank even when the topology does not

    # ── point queries (host) ────────────────────────────────────────────
    def has_node(self, node_id: str) -> bool:
        return node_id in self._nodes

    def has_edge(self, source: str, target: str) -> bool:
        return target in self._succ.get(source, {})

    def neighbors(self, node_id: str) -> list[str]:
        return list(self._succ.get(node_id, {}))

    def node_count(self) -> int:
        return len(self._nodes)

    def edge_count(self) -> int:
        return len(self._edges) // 2

    def to_dict(self) -> dict:
        seen: set[tuple[str, str]] = set()
        edges = []
        for src, targets in self._succ.items():
            for tgt, data in targets.items():
                key = (min(src, tgt), max(src, tgt))
                if key not in seen:
                    seen.add(key)
                    edges.append({"source": src, "target": tgt, **data})
        return {
            "nodes": [{"id": nid, **data} for nid, data in self._nodes.items()],
            "edges": edges,
            "stats": {"node_count": self.node_count(), "edge_count": self.edge_count()},
        }

    # ── device export ───────────────────────────────────────────────────
    @property
    def csr(self) -> csrmod.HostCSR:
        """The DiGraph in node order: forward rows = successors, reverse rows = predecessors, both in dict order."""
        if self._csr is None:
            ids = list(self._nodes)
            index = {nid: i for i, nid in enumerate(ids)}
            ne = len(self._edges)
            src = np.fromiter((index[s] for s, _ in self._edges), dtype=np.int32, count=ne)
            dst = np.fromiter((index[t] for _, t in self._edges), dtype=np.int32, count=ne)
            c = csrmod.from_arrays(ids, np.zeros(len(ids), dtype=np.uint8), src, dst, np.zeros(ne, dtype=np.uint8),
                                   np.full(ne, csrmod.EDGE_TRAVERSABLE, dtype=np.uint8))
            c.index = index
            self._csr = c
        return self._csr

    @property
    def weights(self) -> np.ndarray:
        """``weight`` of each forward adjacency entry as f64 (NetworkX reads ``d.get("weight", 1)``)."""
        if self._weights is None:
            c = self.csr
            by_edge = np.fromiter((float(self._succ[s][t].get("weight", 1)) for s, t in self._edges), dtype=np.float64, count=len(self._edges))
            self._weights = np.ascontiguousarray(by_edge[c.fwd_eid >> 1])
        return self._weights

    @property
    def device_graph(self):
        if self._dg is None:
            from .engine import DeviceGraph

            self._dg = DeviceGraph.upload(self.csr, self._device)
        return self._dg

    # ── analytics (GPU) ─────────────────────────────────────────────────
    def bfs(self, source: str, max_depth: int = 4) -> list[list[str]]:
        """``nx.shortest_path(G, source, v)`` for every node ``v`` of ``nx.bfs_tree(G, source, depth_limit=max_depth)`` but the
        source, in the tree's discovery order: one ordered walk for the tree, one batched bidirectional search for the paths."""
        if source not in self._nodes:
            return []
        c = self.csr
        s = c.index[source]
        tree = self.device_graph.bfs_many(np.asarray([s], dtype=np.int32), max_depth, False).slice(0)
        paths = self.device_graph.bidirectional_paths(np.full(tree.shape[0], s, dtype=np.int32), tree)
        ids = c.node_ids
        return [[ids[int(u)] for u in p] for p in paths]

    def shortest_path(self, source: str, target: str) -> list[str] | None:
        if source not in self._nodes or target not in self._nodes:
            return None
        if source == target:
            return [source]
        c = self.csr
        p = self.device_graph.bidirectional_paths(np.asarray([c.index[source]], dtype=np.int32), np.asarray([c.index[target]], dtype=np.int32))[0]
        return None if p is None else [c.node_ids[int(u)] for u in p]

    def centrality_scores(self) -> dict[str, float]:
        """``nx.pagerank(G)``: alpha 0.85, 100 iterations at most, tolerance 1e-6, edge weights."""
        if not self._nodes:
            return {}
        scores, _ = self.device_graph.pagerank(self.weights)
        return dict(zip(self.csr.node_ids, scores.tolist()))

    def bottleneck_nodes(self, top_n: int = 5) -> list[tuple[str, float]]:
        """Exact ``nx.betweenness_centrality(G)``, highest first, ties in node order."""
        if not self._nodes:
            return []
        scores = self.device_graph.betweenness()
        return sorted(zip(self.csr.node_ids, scores.tolist()), key=lambda x: x[1], reverse=True)[:top_n]

    @classmethod
    def from_unified_graph(cls, graph, device: int = 0) -> "B200NetworkXBackend":
        return from_unified_graph(graph, backend=cls.name, device=device)


def rank_bottlenecks(c: csrmod.HostCSR, scores: np.ndarray, top_n: int) -> list[tuple[str, float]]:
    """Normalise and rank raw device scores the way the reference does; a scored id without a node record is the
    reference's ``KeyError`` (its score table only holds recorded nodes)."""
    ghosts = np.flatnonzero(scores[c.n_real:])
    if ghosts.size:
        raise KeyError(c.node_ids[c.n_real + int(ghosts[0])])
    real = scores[: c.n_real].astype(np.float64)
    total = float(real.sum()) or 1.0
    order = np.argsort(-real, kind="stable")[:top_n]
    return [(c.node_ids[int(i)], float(real[int(i)]) / total) for i in order]


def get_backend(backend: str = "b200", **kwargs) -> B200Backend | B200NetworkXBackend:
    """``get_backend("b200")`` — the name a ``--graph-backend b200`` flag would pass (reference cli/options_surfaces.py:161-162;
    factory ``graph_backend.py:245-259``); ``"b200-networkx"`` gives the NetworkXBackend drop-in.  There is no CPU fallback
    here: other names are an error."""
    if backend in ("b200", "auto"):
        return B200Backend(**kwargs)
    if backend == B200NetworkXBackend.name:
        return B200NetworkXBackend(**kwargs)
    raise ValueError(f"unknown graph backend {backend!r}: this package only provides 'b200' and 'b200-networkx' (no CPU fallback)")


def from_context_graph(context_graph_data: dict, backend: str = "b200", **kwargs) -> B200Backend | B200NetworkXBackend:
    """Serialised context graph → backend (``:262-278``): undirected edges, kind / label / weight kept."""
    graph = get_backend(backend, **kwargs)
    for node in context_graph_data.get("nodes", []):
        graph.add_node(node_id=node["id"], kind=node.get("kind", ""), label=node.get("label", ""))
    for edge in context_graph_data.get("edges", []):
        graph.add_edge(source=edge["source"], target=edge["target"], kind=edge.get("kind", ""), weight=edge.get("weight", 1.0))
    return graph


def from_unified_graph(ug, backend: str = "b200", **kwargs) -> B200Backend | B200NetworkXBackend:
    """UnifiedGraph → backend (``:281-306``): directed edges one-way, bidirectional edges both ways."""
    graph = get_backend(backend, **kwargs)
    for node in ug.nodes.values():
        graph.add_node(node_id=node.id, kind=enum_value(node.entity_type), label=node.label, severity=node.severity, risk_score=node.risk_score)
    for edge in ug.edges:
        bidirectional = getattr(edge, "is_bidirectional", None)
        if bidirectional is None:
            bidirectional = getattr(edge, "direction", "directed") == "bidirectional"
        graph.add_edge(source=edge.source, target=edge.target, kind=enum_value(edge.relationship), weight=getattr(edge, "weight", 1.0), directed=not bidirectional)
    return graph
