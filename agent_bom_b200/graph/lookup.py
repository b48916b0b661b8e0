"""Node records, drilldown edge rows and snapshot statistics served from the snapshot cache.

The reference's SQLite store answers ``edges_for_node_ids``, ``node_context`` and ``snapshot_stats``
(``/root/reference/src/agent_bom/api/graph_store.py:889-948, 1139-1240, 1315-1344``) with queries that read every edge row of the
scan.  Here the cached device graph decides which rows and in which order (``csrc/lookup.cuh``), and SQLite is asked only for the
records of those rows, by primary key:

- ``edges_for_node_ids``: the device's incident original edges of the id set, in edge-id order.  Edge ids follow load order, which is
  rowid order, the order the reference's index scan yields;
- ``node_context``: the node's incident original edges sorted on the device by (source rank, target rank, relationship rank), which
  is ``ORDER BY source_id, target_id, relationship`` under SQLite's BINARY collation;
- ``snapshot_stats`` (unfiltered): the device's histogram of node types, severities and relationships, computed once per graph,
  plus the cached attack paths and interaction risks;
- ``nodes_by_ids``: the ids the cache holds as nodes, in id order (the primary-key index's order).

A snapshot loaded topology-first (graph/snapshot.py) leaves out the stored edge rows whose other endpoint is not a node.  One query
per scan, cached with the graph, finds them with their rowid positions, and they are merged into the answers where SQLite would
return them.
"""

from __future__ import annotations

import heapq
import sqlite3
import threading
from collections import Counter
from typing import Any

import numpy as np

from . import csr as csrmod
from .container import UnifiedGraph
from .csr import EDGE_BIDIRECTIONAL, EDGE_TRAVERSABLE, ENTITY_CODE_OTHER
from .delta import CODE_OTHER, SEVERITY_CODES, _edge_key, _holds_unloaded_edges, real_records, relationship_slots, severity_codes
from .schema import ENTITY_CODE_GHOST, ENTITY_VALUES, REL_CODE, REL_CODE_OTHER, RelationshipType, enum_value
from .snapshot import _EDGE_LAZY_COLUMNS, _NODE_LAZY_COLUMNS, SnapshotEdge, SnapshotNode, edge_columns, node_columns

SEVERITY_NAMES = {code: name for name, code in SEVERITY_CODES.items()}
_CHUNK = 300
_lock = threading.Lock()


def connect(db_path) -> sqlite3.Connection:
    return sqlite3.connect(f"file:{db_path}?mode=ro", uri=True, timeout=10)


class LookupTable:
    """Per-graph state of the lookups: the relationship slots uploaded once, the statistics, the stored rows the loader left out and,
    when a walk needs them, a graph that holds those rows too.  ``lock`` guards the once-per-graph steps of this graph only."""

    def __init__(self, graph):
        csr = graph.csr
        recs = real_records(graph)
        self.erel, self.rel_names = relationship_slots(graph)
        self.severity = severity_codes(recs)
        self.other_severity = Counter(recs[i].severity for i in np.flatnonzero(self.severity == CODE_OTHER).tolist())
        self.other_types = Counter(enum_value(recs[i].entity_type) for i in np.flatnonzero(csr.node_type[:csr.n_real] == ENTITY_CODE_OTHER).tolist())
        self.lock = threading.Lock()
        self.counts: dict[str, np.ndarray] | None = None
        self.unloaded: list[tuple[int, tuple[str, str, str]]] | None = None
        self.unloaded_flags: list[int] = []
        self.unloaded_by_id: dict[str, list[int]] = {}
        self._full_graph: UnifiedGraph | None = None

    def ensure_device(self, graph) -> None:
        with self.lock:
            if self.counts is None:
                self.counts = graph.device_graph.build_lookup_table(graph.csr.n_real, self.severity, self.erel)

    def ensure_unloaded(self, graph, conn, tenant: str) -> None:
        """Stored rows of the scan whose endpoints are not both nodes, each with the number of loaded edges stored before it."""
        with self.lock:
            if self.unloaded is not None:
                return
            rows: list[tuple[int, tuple[str, str, str]]] = []
            flags: list[int] = []
            if _holds_unloaded_edges(graph):
                q = ("SELECT pos, source_id, target_id, relationship, direction, traversable FROM (SELECT row_number() OVER (ORDER BY e.rowid) - 1 "
                     "AS pos, e.source_id, e.target_id, e.relationship, e.direction, e.traversable, (NOT EXISTS (SELECT 1 FROM graph_nodes s WHERE "
                     "s.id = e.source_id AND s.scan_id = e.scan_id AND s.tenant_id = e.tenant_id) OR NOT EXISTS (SELECT 1 FROM graph_nodes t WHERE "
                     "t.id = e.target_id AND t.scan_id = e.scan_id AND t.tenant_id = e.tenant_id)) AS gone FROM graph_edges e WHERE e.tenant_id = ? "
                     "AND e.scan_id = ?) WHERE gone ORDER BY pos")
                for k, (pos, s, t, r, direction, trav) in enumerate(conn.execute(q, (tenant, graph.scan_id))):
                    rows.append((pos - k, (s, t, r)))
                    flags.append((EDGE_TRAVERSABLE if trav else 0) | (EDGE_BIDIRECTIONAL if direction == "bidirectional" else 0))
            by_id: dict[str, list[int]] = {}
            for i, (_, (s, t, _r)) in enumerate(rows):
                by_id.setdefault(s, []).append(i)
                if t != s:
                    by_id.setdefault(t, []).append(i)
            self.unloaded_by_id, self.unloaded_flags, self.unloaded = by_id, flags, rows

    def full_graph(self, graph) -> UnifiedGraph:
        """``graph`` plus the stored rows it leaves out, their endpoints that are not nodes as ghost nodes: what the SQLite store's
        walk and the reference engine on the saved graph see.  Built on first use, and only for a graph that leaves rows out."""
        with self.lock:
            if self._full_graph is None:
                csr = graph.csr
                ids = list(csr.node_ids)
                index = dict(csr.index) if csr.index is not None else {nid: i for i, nid in enumerate(ids)}
                src, dst, rel = [], [], []
                for _, (s, t, r) in self.unloaded:
                    for x in (s, t):
                        if x not in index:
                            index[x] = len(ids)
                            ids.append(x)
                    src.append(index[s])
                    dst.append(index[t])
                    rel.append(REL_CODE.get(r, REL_CODE_OTHER))
                types = np.concatenate([csr.node_type, np.full(len(ids) - csr.n_nodes, ENTITY_CODE_GHOST, np.uint8)])
                full = csrmod.from_arrays(ids, types, np.concatenate([csr.src, np.asarray(src, np.int32)]), np.concatenate([csr.dst, np.asarray(dst, np.int32)]),
                                          np.concatenate([csr.rel, np.asarray(rel, np.uint8)]), np.concatenate([csr.flags, np.asarray(self.unloaded_flags, np.uint8)]),
                                          n_real=csr.n_real)
                full.index = index
                g = UnifiedGraph(scan_id=graph.scan_id, tenant_id=graph.tenant_id, created_at=graph.created_at, device=graph.device)
                g.nodes = graph.nodes
                g._csr = full
                self._full_graph = g
            return self._full_graph

    def stats(self, graph) -> dict[str, Any]:
        c = self.counts
        types = Counter(self.other_types)
        for code in np.flatnonzero(c["type"]).tolist():
            if code < len(ENTITY_VALUES):
                types[ENTITY_VALUES[code]] += int(c["type"][code])
        sev = Counter(self.other_severity)
        for code in np.flatnonzero(c["severity"]).tolist():
            if code != CODE_OTHER and SEVERITY_NAMES[code]:
                sev[SEVERITY_NAMES[code]] += int(c["severity"][code])
        rel = {self.rel_names[s]: int(c["relationship"][s]) for s in np.flatnonzero(c["relationship"]).tolist()}
        paths = [float(p.composite_risk or 0.0) for p in graph.attack_paths]
        risks = [float(r.risk_score or 0.0) for r in graph.interaction_risks]
        return {"total_nodes": int(graph.csr.n_real), "total_edges": int(c["relationship"].sum()), "node_types": dict(sorted(types.items())),
                "severity_counts": dict(sorted(sev.items())), "relationship_types": dict(sorted(rel.items())), "attack_path_count": len(paths),
                "interaction_risk_count": len(risks), "max_attack_path_risk": max(paths, default=0.0), "highest_interaction_risk": max(risks, default=0.0)}


def lookup_table(graph) -> LookupTable:
    t = graph._lookup
    if t is None:
        with _lock:                       # only to give the graph its own lock: building one graph's table never waits on another's
            glock = graph.__dict__.setdefault("_lookup_lock", threading.Lock())
        with glock:
            t = graph._lookup
            if t is None:
                t = graph._lookup = LookupTable(graph)
    return t


# ── keyed hydration: the only statements a warm lookup sends to SQLite ──
def node_records(conn, tenant: str, scan: str, ids: list[str]) -> dict[str, SnapshotNode]:
    out: dict[str, SnapshotNode] = {}
    cols = ", ".join(_NODE_LAZY_COLUMNS)
    for a in range(0, len(ids), _CHUNK):
        chunk = ids[a: a + _CHUNK]
        q = (f"SELECT id, entity_type, label, status, risk_score, severity, {cols} FROM graph_nodes WHERE tenant_id = ? AND scan_id = ? "
             f"AND id IN ({','.join('?' * len(chunk))})")
        for row in conn.execute(q, [tenant, scan, *chunk]):
            node = SnapshotNode(None, row[0], row[1], row[2], row[3], row[4], row[5] or "")
            node._full = node_columns(row[6:])
            out[row[0]] = node
    return out


def edge_records(conn, tenant: str, scan: str, keys: list[tuple[str, str, str]]) -> dict[tuple[str, str, str], SnapshotEdge]:
    out: dict[tuple[str, str, str], SnapshotEdge] = {}
    cols = ", ".join(_EDGE_LAZY_COLUMNS)
    for a in range(0, len(keys), _CHUNK):
        chunk = keys[a: a + _CHUNK]
        q = (f"SELECT source_id, target_id, relationship, direction, weight, traversable, {cols} FROM graph_edges WHERE tenant_id = ? AND "
             f"scan_id = ? AND (source_id, target_id, relationship) IN (VALUES {','.join(['(?,?,?)'] * len(chunk))})")
        params: list[Any] = [tenant, scan]
        for k in chunk:
            params.extend(k)
        for row in conn.execute(q, params):
            try:
                rel = RelationshipType(row[2])
            except ValueError:
                rel = row[2]
            edge = SnapshotEdge(None, row[0], row[1], rel, row[3], row[4], bool(row[5]))
            edge._full = edge_columns(row[6:], scan)
            out[(row[0], row[1], row[2])] = edge
    return out


# ── the lookups ──
def nodes_by_ids(graph, db_path, tenant: str, node_ids) -> list[SnapshotNode]:
    """Records of the ids that are nodes of ``graph``, in id order."""
    ids = sorted(nid for nid in set(node_ids) if graph.has_node(nid))
    if not ids:
        return []
    conn = connect(db_path)
    try:
        recs = node_records(conn, tenant, graph.scan_id, ids)
    finally:
        conn.close()
    return [recs[nid] for nid in ids if nid in recs]


def _edges_in_order(graph, conn, tenant: str, keys: list[tuple[str, str, str]]) -> list[SnapshotEdge]:
    recs = edge_records(conn, tenant, graph.scan_id, keys)
    return [recs[k] for k in keys if k in recs]


def edges_for_node_ids(graph, db_path, tenant: str, node_ids) -> list[SnapshotEdge]:
    """Stored edge rows with an endpoint in ``node_ids``, in rowid order.  Unlike the reference's query, which binds two parameters
    per id and fails past SQLite's variable limit (about 16 000 ids), any number of ids is answered."""
    ids = set(node_ids)
    if not ids:
        return []
    csr = graph.csr
    idx = np.unique(np.asarray([i for i in (csr.idx(nid) for nid in ids) if i >= 0], np.int32))
    table = lookup_table(graph)
    conn = connect(db_path)
    try:
        table.ensure_unloaded(graph, conn, tenant)
        loaded = graph.device_graph.incident_edges(idx).tolist() if idx.size else []
        extra = sorted({i for nid in ids for i in table.unloaded_by_id.get(nid, ())})
        keys: list[tuple[str, str, str]] = []
        j = 0
        for e in loaded:
            while j < len(extra) and table.unloaded[extra[j]][0] <= e:
                keys.append(table.unloaded[extra[j]][1])
                j += 1
            keys.append(_edge_key(graph, e))
        keys.extend(table.unloaded[i][1] for i in extra[j:])
        return _edges_in_order(graph, conn, tenant, keys)
    finally:
        conn.close()


def node_context_edges(graph, db_path, tenant: str, node_id: str) -> list[SnapshotEdge]:
    """Stored edge rows with ``node_id`` as an endpoint, in (source_id, target_id, relationship) order."""
    table = lookup_table(graph)
    conn = connect(db_path)
    try:
        table.ensure_device(graph)
        table.ensure_unloaded(graph, conn, tenant)
        keys = [_edge_key(graph, e) for e in graph.device_graph.context_edges(graph.csr.idx(node_id)).tolist()]
        extra = sorted(table.unloaded[i][1] for i in table.unloaded_by_id.get(node_id, ()))
        if extra:
            keys = list(heapq.merge(keys, extra))
        return _edges_in_order(graph, conn, tenant, keys)
    finally:
        conn.close()


def node_impact(graph, db_path, tenant: str, node_id: str) -> dict[str, Any]:
    """``impact_of(node_id)`` over every stored row of the snapshot.  The device walk of ``graph`` is exact unless the node or a node
    it reaches is an endpoint of a row the loader left out; then the walk runs on the graph that holds those rows too."""
    impact = graph.impact_of(node_id)
    table = lookup_table(graph)
    conn = connect(db_path)
    try:
        table.ensure_unloaded(graph, conn, tenant)
    finally:
        conn.close()
    by_id = table.unloaded_by_id
    if by_id and (node_id in by_id or any(n in by_id for n in impact["affected_nodes"])):
        impact = table.full_graph(graph).impact_of(node_id)
    return impact


def snapshot_stats(graph) -> dict[str, Any]:
    """The unfiltered ``snapshot_stats`` body of ``graph``; the device histogram is computed once per graph."""
    table = lookup_table(graph)
    table.ensure_device(graph)
    return table.stats(graph)


EMPTY_STATS = {"total_nodes": 0, "total_edges": 0, "node_types": {}, "severity_counts": {}, "relationship_types": {}, "attack_path_count": 0,
               "interaction_risk_count": 0, "max_attack_path_risk": 0.0, "highest_interaction_risk": 0.0}
