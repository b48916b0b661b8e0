"""UnifiedGraph — host container of the typed exposure graph whose traversals run on the H100.

Same surface as the reference container
(``/root/reference/src/agent_bom/graph/container.py:90-538``): ``add_node`` /
``add_edge`` with the reference's merge and de-duplication rules, point queries
(``edges_from``, ``edges_to``, ``sources_of`` …) and the traversal methods
``impact_of``, ``bfs``, ``shortest_path``, ``reachable_from``,
``traverse_subgraph`` — plus batched ``*_many`` forms, which is how the device
is meant to be driven.

Every traversal is executed by the CUDA engine (``engine.DeviceGraph``) on a CSR
exported from this container; there is no host traversal code here.  The
device copy is a cache: it is (re)built lazily after any mutation.
"""

from __future__ import annotations

import time
from collections import defaultdict
from datetime import datetime, timezone
from typing import Any, Iterable

import numpy as np

from .. import _lib
from . import csr as csrmod
from .model import AttackPath, UnifiedEdge, UnifiedNode
from .schema import (
    ENTITY_CODE,
    ENTITY_VALUES,
    FINDING_CODES,
    REL_CODE,
    SEVERITY_RANK,
    EntityType,
    enum_value,
    rel_mask,
)

_EMPTY = (None, "", [], {})


def _now_iso() -> str:
    return datetime.now(timezone.utc).isoformat()


def reversed_edge(edge):
    """The reversed twin of a bidirectional edge, for our records or duck-typed reference records."""
    if hasattr(edge, "reversed_copy"):
        return edge.reversed_copy()
    kwargs = dict(source=edge.target, target=edge.source, relationship=edge.relationship, direction=edge.direction,
                  weight=getattr(edge, "weight", 1.0), traversable=edge.traversable, evidence=getattr(edge, "evidence", {}))
    return type(edge)(**kwargs)


class UnifiedGraph:
    def __init__(self, scan_id: str = "", tenant_id: str = "", created_at: str = "", *, device: int = 0):
        self.nodes: dict[str, Any] = {}
        self.edges: list[Any] = []
        self._edge_keys: set[tuple[str, str, str]] = set()
        self._edge_index: dict[tuple[str, str, str], int] = {}
        self.attack_paths: list[AttackPath] = []
        self.interaction_risks: list[Any] = []
        self.unhandled_sections: list[str] = []      # report sections the light builder did not model (graph/builder.py)
        self.scan_id, self.tenant_id = scan_id, tenant_id
        self.created_at = created_at or _now_iso()
        self.device = device
        self._csr: csrmod.HostCSR | None = None
        self._dg = None
        # per-graph caches of the ranked views (graph/exposure.py, graph/fix_first.py), dropped with the device graph
        self._rank_inputs = None
        self._focus_index = None
        self._edge_lookup = None
        self._clusters = None              # semantic-cluster key table (graph/clusters.py)
        self._delta = None                 # snapshot-diff tables (graph/delta.py)

    # ── construction from foreign graphs ────────────────────────────────
    @classmethod
    def from_graph(cls, graph, *, device: int = 0) -> "UnifiedGraph":
        """Adopt any UnifiedGraph-shaped object (e.g. the reference's) without copying node / edge records."""
        g = cls(scan_id=getattr(graph, "scan_id", ""), tenant_id=getattr(graph, "tenant_id", ""), created_at=getattr(graph, "created_at", ""), device=device)
        g.nodes = graph.nodes if isinstance(graph.nodes, dict) else dict(graph.nodes)
        g.edges = graph.edges
        for i, e in enumerate(g.edges):
            key = (e.source, e.target, enum_value(e.relationship))
            g._edge_keys.add(key)
            g._edge_index.setdefault(key, i)
        g.attack_paths = list(getattr(graph, "attack_paths", []) or [])
        g.interaction_risks = list(getattr(graph, "interaction_risks", []) or [])
        return g

    # ── mutation (reference container.py:116-198) ───────────────────────
    def _invalidate(self) -> None:
        self._csr = None
        self._rank_inputs = self._focus_index = self._edge_lookup = self._clusters = self._delta = None
        if self._dg is not None:
            self._dg.close()
            self._dg = None

    def add_node(self, node) -> None:
        """Add or merge: attributes update, higher severity / risk win, tags and sources are unioned."""
        existing = self.nodes.get(node.id)
        if existing is None:
            self.nodes[node.id] = node
            self._invalidate()
            return
        self._rank_inputs = self._clusters = self._delta = None     # a merge can raise severity / risk and change attributes, which they read
        existing.last_seen = getattr(node, "last_seen", "") or _now_iso()
        existing.attributes.update(node.attributes)
        if SEVERITY_RANK.get(node.severity, 0) > SEVERITY_RANK.get(existing.severity, 0):
            existing.severity = node.severity
            if hasattr(existing, "severity_id"):
                existing.severity_id = getattr(node, "severity_id", existing.severity_id)
        if node.risk_score > existing.risk_score:
            existing.risk_score = node.risk_score
        for field in ("data_sources", "compliance_tags"):
            have = getattr(existing, field)
            seen = set(have)
            for item in getattr(node, field):
                if item not in seen:
                    have.append(item)
                    seen.add(item)

    def add_edge(self, edge) -> None:
        """O(1) de-duplication on (source, target, relationship); a repeated edge only merges its evidence."""
        key = (edge.source, edge.target, enum_value(edge.relationship))
        if key in self._edge_keys:
            evidence = getattr(edge, "evidence", None)
            if evidence:
                stored = self.edges[self._edge_index[key]]
                for k, v in evidence.items():
                    if v in _EMPTY:
                        continue
                    if k not in stored.evidence or stored.evidence[k] in _EMPTY:
                        stored.evidence[k] = v
            return
        self._edge_keys.add(key)
        self._edge_index[key] = len(self.edges)
        self.edges.append(edge)
        self._invalidate()

    # ── device cache ────────────────────────────────────────────────────
    @property
    def csr(self) -> csrmod.HostCSR:
        if self._csr is None:
            self._csr = csrmod.from_unified_graph(self)
        return self._csr

    @property
    def device_graph(self):
        if self._dg is None:
            from ..engine import DeviceGraph

            self._dg = DeviceGraph.upload(self.csr, self.device)
        return self._dg

    def _idx(self, node_id: str) -> int:
        """Index of a node that has a record (ghost endpoints are not valid sources), else -1."""
        i = self.csr.idx(node_id)
        return i if 0 <= i < self.csr.n_real else -1

    # ── point queries (host CSR rows) ───────────────────────────────────
    def get_node(self, node_id: str):
        return self.nodes.get(node_id)

    def has_node(self, node_id: str) -> bool:
        return node_id in self.nodes

    def nodes_by_type(self, entity_type) -> list:
        want = enum_value(entity_type)
        return [n for n in self.nodes.values() if enum_value(n.entity_type) == want]

    def _row_edges(self, node_id: str, forward: bool) -> list:
        c = self.csr
        u = c.idx(node_id)
        if u < 0:
            return []
        off, eid = (c.fwd_off, c.fwd_eid) if forward else (c.rev_off, c.rev_eid)
        out = []
        for e2 in eid[int(off[u]): int(off[u + 1])].tolist():
            edge = self.edges[e2 >> 1]
            out.append(reversed_edge(edge) if e2 & 1 else edge)
        return out

    def edges_from(self, node_id: str) -> list:
        """``adjacency[node_id]`` in list order (reversed twins of bidirectional edges included)."""
        return self._row_edges(node_id, True)

    def edges_to(self, node_id: str) -> list:
        """``reverse_adjacency[node_id]`` in list order."""
        return self._row_edges(node_id, False)

    def neighbors(self, node_id: str) -> list[str]:
        return [e.target for e in self.edges_from(node_id)]

    def sources_of(self, node_id: str) -> list[str]:
        return [e.source for e in self.edges_to(node_id)]

    def has_edge(self, source: str, target: str) -> bool:
        return any(e.target == target for e in self.edges_from(source))

    @property
    def adjacency(self) -> dict[str, list]:
        return {nid: lst for nid in self.csr.node_ids if (lst := self.edges_from(nid))}

    @property
    def reverse_adjacency(self) -> dict[str, list]:
        return {nid: lst for nid in self.csr.node_ids if (lst := self.edges_to(nid))}

    def finding_ids(self) -> list[str]:
        return [n.id for n in self.nodes.values() if ENTITY_CODE.get(enum_value(n.entity_type)) in FINDING_CODES]

    # ── impact_of (reference container.py:230-279) ──────────────────────
    def _impact_dict(self, node_id: str, res, q: int) -> dict:
        ids = self.csr.node_ids
        reached = res.slice(q)
        by_type = res.hist_dict(q)
        if (self.csr.node_type[reached] == csrmod.ENTITY_CODE_OTHER).any():   # entity kinds outside the enum are tallied on the host
            for i in reached[self.csr.node_type[reached] == csrmod.ENTITY_CODE_OTHER].tolist():
                k = enum_value(self.nodes[ids[i]].entity_type)
                by_type[k] = by_type.get(k, 0) + 1
        return {"node_id": node_id, "affected_nodes": sorted(ids[i] for i in reached.tolist()), "affected_by_type": by_type,
                "affected_count": int(res.count[q]), "max_depth_reached": int(res.maxd[q])}

    def impact_of(self, node_id: str, max_depth: int = 4) -> dict:
        return self.impact_of_many([node_id], max_depth)[0]

    def impact_of_many(self, node_ids: Iterable[str], max_depth: int = 4) -> list[dict]:
        """Blast radius of every listed node in ONE device batch (reverse BFS, all relationships, traversable ignored)."""
        node_ids = list(node_ids)
        idx = np.asarray([self._idx(n) for n in node_ids], dtype=np.int32)
        res = self.device_graph.impact_many(idx, max_depth)
        out = []
        for q, nid in enumerate(node_ids):
            if idx[q] < 0:
                out.append({"node_id": nid, "affected_nodes": [], "affected_by_type": {}, "affected_count": 0, "max_depth_reached": 0})
            else:
                out.append(self._impact_dict(nid, res, q))
        return out

    # ── bfs (reference container.py:367-391) ────────────────────────────
    def bfs(self, source: str, max_depth: int = 4, traversable_only: bool = True) -> list[list[str]]:
        return self.bfs_many([source], max_depth, traversable_only)[0]

    def bfs_many(self, sources: Iterable[str], max_depth: int = 4, traversable_only: bool = True) -> list[list[list[str]]]:
        """Per source: one path per reached node, in discovery order, via first-discoverer parents."""
        sources = list(sources)
        idx = np.asarray([self._idx(s) for s in sources], dtype=np.int32)
        res = self.device_graph.bfs_many(idx, max_depth, traversable_only)
        ids = self.csr.node_ids
        out = []
        for q, s in enumerate(sources):
            paths: list[list[str]] = []
            if idx[q] >= 0:
                nodes, parent = res.slice(q).tolist(), res.aux(q, "parent").tolist()
                for i, u in enumerate(nodes):
                    p = parent[i]            # position in the full queue: 0 is the source, k>0 is emitted entry k-1
                    paths.append(([s] if p <= 0 else paths[p - 1]) + [ids[u]])
            out.append(paths)
        return out

    # ── shortest_path (reference container.py:393-409) ──────────────────
    def shortest_path(self, source: str, target: str) -> list[str] | None:
        s, t = self._idx(source), self._idx(target)
        if s < 0 or t < 0:
            return None
        if s == t:
            return [source]
        res = self.device_graph.shortest_path_many(np.asarray([s], dtype=np.int32), np.asarray([t], dtype=np.int32))
        if not (int(res.flags[0]) & _lib.QFLAG_TARGET_FOUND):
            return None
        nodes, parent = res.slice(0), res.aux(0, "parent")
        i = len(nodes) - 1
        while nodes[i] != t:
            i -= 1
        path = []
        while i >= 0:
            path.append(self.csr.node_ids[int(nodes[i])])
            i = int(parent[i])
        return path[::-1]

    # ── reachable_from (reference container.py:411-436) ─────────────────
    def reachable_from(self, source: str, max_depth: int = 6, *, traversable_only: bool = False, include_source: bool = True) -> set[str]:
        s = self._idx(source)
        if s < 0:
            return set()
        res = self.device_graph.reachable_many(np.asarray([s], dtype=np.int32), max_depth, traversable_only)
        ids = self.csr.node_ids
        out = {ids[i] for i in res.slice(0).tolist()}
        if include_source:
            out.add(source)
        return out

    # ── traverse_subgraph (reference container.py:438-538) ──────────────
    def traverse_subgraph(self, roots: list[str], *, direction: str = "forward", max_depth: int = 4, max_nodes: int = 500, max_edges: int = 10_000,
                          deadline_monotonic: float | None = None, traversable_only: bool = False, relationship_types=None, static_only: bool = False,
                          dynamic_only: bool = False, include_roots: bool = True) -> tuple["UnifiedGraph", dict[str, int], bool]:
        sub = UnifiedGraph(scan_id=self.scan_id, tenant_id=self.tenant_id, created_at=self.created_at, device=self.device)
        if not roots:
            return sub, {}, False
        valid_roots = [r for r in roots if r in self.nodes]
        if deadline_monotonic is not None and time.monotonic() >= deadline_monotonic:
            # the reference checks the deadline before the first pop: only the seeded roots survive
            if include_roots:
                for r in valid_roots:
                    sub.add_node(self.nodes[r])
            return sub, {r: 0 for r in valid_roots}, True
        dir_code = {"forward": _lib.DIR_FORWARD, "reverse": _lib.DIR_REVERSE, "both": _lib.DIR_BOTH}.get(direction)
        if dir_code is None:
            # the reference silently yields no candidates for an unknown direction
            if include_roots:
                for r in valid_roots:
                    sub.add_node(self.nodes[r])
            return sub, {r: 0 for r in valid_roots}, False
        mask = rel_mask(relationship_types) if relationship_types else 0     # 0 = no relationship filter for the spec constructor
        dg = self.device_graph
        spec = dg.spec_traverse(dir_code, max_depth, max_nodes, max_edges, traversable_only, mask, static_only, dynamic_only, include_roots)
        if relationship_types and mask == 0:
            spec.rel_mask = 0                                                 # a filter that names no known relationship admits nothing
        root_idx = np.asarray([self.csr.idx(r) if r in self.nodes else -1 for r in roots], dtype=np.int32)
        res = dg.walk(spec, root_idx, np.asarray([0, len(root_idx)], dtype=np.int64))
        ids = self.csr.node_ids
        nodes, depth = res.slice(0).tolist(), res.aux(0, "depth").tolist()
        depth_by_node: dict[str, int] = {}
        for u, d in zip(nodes, depth):
            depth_by_node[ids[u]] = d
        visited = {ids[u] for u in nodes[len(valid_roots):]}
        if include_roots:
            visited.update(valid_roots)
        for nid in visited:
            node = self.nodes.get(nid)
            if node is not None:
                sub.add_node(node)
        seen_e2: set[int] = set()
        for e2 in res.edge_slice(0).tolist():
            if e2 in seen_e2:
                continue
            seen_e2.add(e2)
            edge = self.edges[e2 >> 1]
            if e2 & 1:
                edge = reversed_edge(edge)
            if edge.source in sub.nodes and edge.target in sub.nodes:
                sub.add_edge(edge)
        truncated = bool(int(res.flags[0]) & _lib.QFLAG_TRUNCATED)
        if deadline_monotonic is not None and time.monotonic() >= deadline_monotonic:
            truncated = True
        return sub, depth_by_node, truncated

    # ── centrality (reference container.py:540-567) ─────────────────────
    def degree_centrality(self) -> dict[str, float]:
        if not self.nodes:
            return {}
        c = self.csr
        max_possible = max(len(self.nodes) - 1, 1)
        deg = np.diff(c.fwd_off.astype(np.int64))
        return {nid: int(deg[i]) / max_possible for i, nid in enumerate(self.nodes)}

    def bottleneck_nodes(self, top_n: int = 5) -> list[tuple[str, float]]:
        """BFS from the first 50 nodes over the forward adjacency (every entry, any depth); each node strictly inside a
        first-discoverer path scores +1; scores are normalised by their sum and ranked, ties in node order."""
        if not self.nodes:
            return []
        from ..backend import rank_bottlenecks

        c = self.csr
        sample = np.arange(min(50, c.n_real), dtype=np.int32)
        return rank_bottlenecks(c, self.device_graph.bottleneck_scores(sample), top_n)

    # ── OCSF export (reference container.py:628-654) ────────────────────
    def iter_ocsf_events(self, product_version: str = "0.0.0", *, enrich_neighbors: bool = True, batch_size: int = 65536):
        """Finding nodes as OCSF events, in ``nodes`` order; with ``enrich_neighbors`` each carries its ``graph_context``
        (typed in-neighbours, blast radius and its type histogram), computed on the device one batch of findings at a time."""
        from .ocsf import iter_ocsf_events

        return iter_ocsf_events(self, product_version, enrich_neighbors=enrich_neighbors, batch_size=batch_size)

    def to_ocsf_events(self, product_version: str = "0.0.0", *, enrich_neighbors: bool = True) -> list[dict[str, Any]]:
        return list(self.iter_ocsf_events(product_version, enrich_neighbors=enrich_neighbors))

    # ── serialisation ───────────────────────────────────────────────────
    def to_dict(self) -> dict[str, Any]:
        def nd(n):
            return n.to_dict() if hasattr(n, "to_dict") else {"id": n.id, "entity_type": enum_value(n.entity_type), "label": n.label}

        return {"scan_id": self.scan_id, "tenant_id": self.tenant_id, "created_at": self.created_at, "nodes": [nd(n) for n in self.nodes.values()],
                "edges": [e.to_dict() for e in self.edges], "attack_paths": [p.to_dict() for p in self.attack_paths]}

    @classmethod
    def from_dict(cls, data: dict[str, Any]) -> "UnifiedGraph":
        from .schema import NodeStatus, RelationshipType

        g = cls(scan_id=data.get("scan_id", ""), tenant_id=data.get("tenant_id", ""), created_at=data.get("created_at", ""))
        for n in data.get("nodes", []):
            et = n.get("entity_type", "")
            g.add_node(UnifiedNode(id=n["id"], entity_type=EntityType(et) if et in ENTITY_VALUES else et, label=n.get("label", n["id"]),
                                   status=NodeStatus(n.get("status", "active")), risk_score=n.get("risk_score", 0.0), severity=n.get("severity", ""),
                                   attributes=n.get("attributes", {}), compliance_tags=n.get("compliance_tags", []), data_sources=n.get("data_sources", [])))
        for e in data.get("edges", []):
            rel = e.get("relationship", "")
            g.add_edge(UnifiedEdge(source=e["source"], target=e["target"], relationship=RelationshipType(rel) if rel in REL_CODE else rel,
                                   direction=e.get("direction", "directed"), weight=e.get("weight", 1.0), traversable=e.get("traversable", True),
                                   evidence=e.get("evidence", {})))
        g.attack_paths = [AttackPath.from_dict(p) for p in data.get("attack_paths", [])]
        return g

    def stats(self) -> dict[str, Any]:
        by_type: dict[str, int] = defaultdict(int)
        for n in self.nodes.values():
            by_type[enum_value(n.entity_type)] += 1
        by_rel: dict[str, int] = defaultdict(int)
        for e in self.edges:
            by_rel[enum_value(e.relationship)] += 1
        return {"total_nodes": len(self.nodes), "total_edges": len(self.edges), "node_types": dict(by_type), "relationship_types": dict(by_rel)}
