"""Topology-first loader for persisted graph snapshots (SURVEY.md §8 row f1).

The reference rebuilds a full ``UnifiedGraph`` from SQLite by constructing one
``UnifiedNode`` / ``UnifiedEdge`` per row and JSON-decoding seven text columns per
row (``/root/reference/src/agent_bom/db/graph_store.py:558-668``; tables ``:52-160``).
The traversal engine needs none of that: it needs the node list in row order, the
entity type, and the ``(source, target, relationship, direction, traversable)``
stream in row order.  ``load_snapshot`` therefore scans exactly those columns with
the reference's own ``WHERE tenant_id = ? AND scan_id = ?`` predicates (same query
plan, so the same row order — adjacency order is what fixes BFS discovery order),
builds the CSR straight from arrays, and keeps node / edge *records* thin: the
columns the exposure ranking needs (label, risk, severity) are resident, the JSON
columns are fetched per node only when a caller actually asks for them (the ≤500
nodes of a ``traverse_subgraph`` answer, not the 10 M of the estate).

Kept from the reference: tenant normalisation (``:169-172``), latest-snapshot
resolution (``:309-322,349-364``), edges whose endpoints are not both present are
dropped (``:611-612``), materialised ``attack_paths`` / ``interaction_risks`` rows
are loaded as they are (``:633-666``) because materialised paths win over derived
ones (``api/routes/graph.py:695-696``).
"""

from __future__ import annotations

import json
import sqlite3
import uuid
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any

import numpy as np

from . import csr as csrmod
from .container import UnifiedGraph
from .model import AttackPath
from .csr import EDGE_BIDIRECTIONAL, EDGE_TRAVERSABLE, ENTITY_CODE_OTHER
from .schema import ENTITY_CODE, REL_CODE, REL_CODE_OTHER, RELATIONSHIP_VALUES, EntityType, NodeStatus, RelationshipType

DEFAULT_GRAPH_TENANT_ID = "default"
#: namespace of the reference's deterministic ids (canonical_ids.py:12) — a wire constant, needed for identical ``canonical_id`` values
_ID_NAMESPACE = uuid.UUID("7f3e4b2a-9c1d-5f8e-a0b4-12c3d4e5f6a7")


def _canonical_id(*parts: str) -> str:
    """UUIDv5 over the lower-cased, stripped, non-empty parts joined by ':' (canonical_ids.py:24-33,80-85)."""
    return str(uuid.uuid5(_ID_NAMESPACE, ":".join(t.lower().strip() for t in (str(p) for p in parts if p is not None) if t)))


def normalize_graph_tenant_id(tenant_id: str | None) -> str:
    """Blank tenants live in the ``default`` bucket (reference db/graph_store.py:169-172)."""
    return (tenant_id or "").strip() or DEFAULT_GRAPH_TENANT_ID


def latest_snapshot_id(conn: sqlite3.Connection, *, tenant_id: str = "") -> str:
    row = conn.execute("SELECT scan_id FROM graph_snapshots WHERE tenant_id = ? ORDER BY created_at DESC, scan_id DESC LIMIT 1",
                       (normalize_graph_tenant_id(tenant_id),)).fetchone()
    return str(row[0]) if row else ""


def resolve_snapshot(conn: sqlite3.Connection, *, tenant_id: str = "", scan_id: str = "") -> tuple[str, str]:
    """``(scan_id, created_at)`` of the requested or newest snapshot, ``("", "")`` when there is none (:349-364)."""
    tenant = normalize_graph_tenant_id(tenant_id)
    effective = scan_id or latest_snapshot_id(conn, tenant_id=tenant)
    if not effective:
        return "", ""
    row = conn.execute("SELECT created_at FROM graph_snapshots WHERE scan_id = ? AND tenant_id = ?", (effective, tenant)).fetchone()
    return effective, (str(row[0]) if row else "")


@dataclass(slots=True)
class InteractionRisk:
    """Row of ``interaction_risks`` (reference graph/container.py:60-78)."""

    pattern: str
    agents: list[str] = field(default_factory=list)
    risk_score: float = 0.0
    description: str = ""
    owasp_agentic_tag: str | None = None

    def to_dict(self) -> dict[str, Any]:
        return {"pattern": self.pattern, "agents": self.agents, "risk_score": self.risk_score, "description": self.description,
                "owasp_agentic_tag": self.owasp_agentic_tag}


_NODE_JSON_COLUMNS = ("attributes", "compliance_tags", "data_sources", "dimensions")
_NODE_LAZY_COLUMNS = ("category_uid", "class_uid", "type_uid", "severity_id", "first_seen", "last_seen") + _NODE_JSON_COLUMNS


def _entity(value: str):
    try:
        return EntityType(value)
    except ValueError:
        return value


class SnapshotNode:
    """A node record whose scalar columns are resident and whose JSON columns are read on first use."""

    __slots__ = ("id", "entity_type", "label", "status", "risk_score", "severity", "_graph", "_full")

    def __init__(self, graph: "SnapshotGraph", node_id: str, entity_type: str, label: str, status: str, risk_score: float, severity: str):
        self.id, self.label, self.risk_score, self.severity = node_id, label, risk_score, severity
        self.entity_type = _entity(entity_type)
        try:
            self.status = NodeStatus(status)
        except ValueError:
            self.status = status
        self._graph = graph
        self._full: dict[str, Any] | None = None

    def _hydrate(self) -> dict[str, Any]:
        if self._full is None:
            self._graph.hydrate_nodes([self.id])
            if self._full is None:      # row vanished under us: behave like an empty record
                self._full = {c: ({} if c in ("attributes", "dimensions") else [] if c in _NODE_JSON_COLUMNS else 0 if c.endswith("_uid") or c == "severity_id" else "")
                              for c in _NODE_LAZY_COLUMNS}
        return self._full

    def __getattr__(self, name: str):
        if name in _NODE_LAZY_COLUMNS:
            return self._hydrate()[name]
        raise AttributeError(name)

    @property
    def canonical_id(self) -> str:
        """Stable cross-scan identity (graph/node.py:124-131): an explicit attribute wins, else a UUIDv5 of (kind, id)."""
        attrs = self._hydrate()["attributes"]
        candidate = attrs.get("canonical_id") or attrs.get("stable_id")
        if isinstance(candidate, str) and candidate.strip():
            return candidate
        return _canonical_id("graph_node", getattr(self.entity_type, "value", str(self.entity_type)), self.id)

    def to_dict(self) -> dict[str, Any]:
        """Same keys as the reference's ``UnifiedNode.to_dict`` (graph/node.py:133-152)."""
        full = self._hydrate()
        d = {"id": self.id, "canonical_id": self.canonical_id, "entity_type": getattr(self.entity_type, "value", self.entity_type), "label": self.label,
             "category_uid": full["category_uid"], "class_uid": full["class_uid"], "type_uid": full["type_uid"],
             "status": getattr(self.status, "value", self.status), "risk_score": self.risk_score, "severity": self.severity,
             "severity_id": full["severity_id"], "first_seen": full["first_seen"], "last_seen": full["last_seen"],
             "attributes": full["attributes"], "compliance_tags": full["compliance_tags"], "data_sources": full["data_sources"],
             "dimensions": full["dimensions"]}
        return d


def node_columns(values) -> dict[str, Any]:
    """The lazy columns of a node row (``_NODE_LAZY_COLUMNS`` order), JSON decoded as the reference's ``_node_from_row`` does."""
    full = dict(zip(_NODE_LAZY_COLUMNS, values))
    for c in _NODE_JSON_COLUMNS:
        full[c] = json.loads(full[c]) if full[c] else ({} if c in ("attributes", "dimensions") else [])
    return full


_EDGE_LAZY_COLUMNS = ("first_seen", "last_seen", "valid_from", "valid_to", "confidence", "provenance", "source_scan_id", "source_run_id", "evidence", "activity_id")


def edge_columns(values, scan_id: str) -> dict[str, Any]:
    """The lazy columns of an edge row (``_EDGE_LAZY_COLUMNS`` order) as the reference's ``_edge_from_row`` reads them."""
    first_seen, last_seen, valid_from, valid_to, confidence, provenance, src_scan, src_run, evidence, activity = values
    return {"first_seen": first_seen, "last_seen": last_seen, "valid_from": valid_from or first_seen, "valid_to": valid_to,
            "confidence": confidence, "provenance": json.loads(provenance or "{}"), "source_scan_id": src_scan or scan_id,
            "source_run_id": src_run or "", "evidence": json.loads(evidence or "{}"), "activity_id": activity}


class SnapshotEdge:
    """Edge record synthesised from the edge arrays; evidence / provenance / timestamps are read on first use."""

    __slots__ = ("source", "target", "relationship", "direction", "weight", "traversable", "_graph", "_row", "_full")

    def __init__(self, graph: "SnapshotGraph", source: str, target: str, relationship, direction: str, weight: float, traversable: bool, row=None):
        self.source, self.target, self.relationship = source, target, relationship
        self.direction, self.weight, self.traversable = direction, weight, traversable
        self._graph, self._full = graph, None
        # primary key of the stored row (a reversed twin keeps the original's)
        self._row = row if row is not None else (source, target, getattr(relationship, "value", relationship))

    @property
    def is_bidirectional(self) -> bool:
        return self.direction == "bidirectional"

    @property
    def id(self) -> str:
        return f"{getattr(self.relationship, 'value', self.relationship)}:{self.source}:{self.target}"

    def _hydrate(self) -> dict[str, Any]:
        if self._full is None:
            self._graph.hydrate_edges([self])
        return self._full

    def __getattr__(self, name: str):
        if name in ("evidence", "provenance", "confidence", "first_seen", "last_seen", "valid_from", "valid_to", "source_scan_id", "source_run_id", "activity_id"):
            return self._hydrate()[name]
        raise AttributeError(name)

    def reversed_copy(self) -> "SnapshotEdge":
        twin = SnapshotEdge(self._graph, self.target, self.source, self.relationship, self.direction, self.weight, self.traversable, row=self._row)
        twin._full = self._full
        return twin

    @property
    def canonical_id(self) -> str:
        return _canonical_id("graph_edge", getattr(self.relationship, "value", str(self.relationship)), self.source, self.target)

    def to_dict(self) -> dict[str, Any]:
        """Same keys as the reference's ``UnifiedEdge.to_dict`` (graph/edge.py:73-95)."""
        full = self._hydrate()
        return {"id": self.id, "canonical_id": self.canonical_id, "source": self.source, "target": self.target, "source_id": self.source,
                "target_id": self.target, "relationship": getattr(self.relationship, "value", self.relationship),
                "direction": self.direction, "weight": self.weight, "traversable": self.traversable, "first_seen": full["first_seen"],
                "last_seen": full["last_seen"], "valid_from": full["valid_from"], "valid_to": full["valid_to"], "confidence": full["confidence"],
                "provenance": full["provenance"], "source_scan_id": full["source_scan_id"], "source_run_id": full["source_run_id"],
                "evidence": full["evidence"], "activity_id": full["activity_id"]}


class _EdgeList:
    """``graph.edges`` over the edge arrays: records are made when indexed, never all at once."""

    def __init__(self, graph: "SnapshotGraph"):
        self._g = graph

    def __len__(self) -> int:
        return int(self._g._e_src.shape[0])

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        g = self._g
        if i < 0:
            i += len(self)
        ids = g.csr.node_ids
        code = int(g._e_rel[i])
        rel_name = g._e_other.get(i) if code == REL_CODE_OTHER else RELATIONSHIP_VALUES[code]
        try:
            rel = RelationshipType(rel_name)
        except ValueError:
            rel = rel_name
        fl = int(g._e_flags[i])
        return SnapshotEdge(g, ids[int(g._e_src[i])], ids[int(g._e_dst[i])], rel, "bidirectional" if fl & EDGE_BIDIRECTIONAL else "directed",
                            float(g._e_weight[i]), bool(fl & EDGE_TRAVERSABLE))

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    def append(self, _edge) -> None:
        raise TypeError("a snapshot graph is immutable; build a UnifiedGraph to add edges")


class SnapshotGraph(UnifiedGraph):
    """One persisted snapshot, loaded topology-first.  Read-only: snapshots are immutable per scan (:368-372)."""

    def __init__(self, db_path: str | Path, scan_id: str = "", tenant_id: str = "", created_at: str = "", *, device: int = 0):
        super().__init__(scan_id=scan_id, tenant_id=tenant_id, created_at=created_at or " ", device=device)
        self.created_at = created_at
        self.db_path = str(db_path)
        self._e_src = self._e_dst = np.zeros(0, dtype=np.int32)
        self._e_rel = self._e_flags = np.zeros(0, dtype=np.uint8)
        self._e_weight = np.zeros(0, dtype=np.float32)
        self._e_other: dict[int, str] = {}
        self.edges = _EdgeList(self)

    # the CSR is built once by the loader and never invalidated by mutation
    def add_node(self, node) -> None:
        raise TypeError("a snapshot graph is immutable; build a UnifiedGraph to add nodes")

    def add_edge(self, edge) -> None:
        raise TypeError("a snapshot graph is immutable; build a UnifiedGraph to add edges")

    def _connect(self) -> sqlite3.Connection:
        conn = sqlite3.connect(f"file:{self.db_path}?mode=ro", uri=True, timeout=10)
        return conn

    def hydrate_nodes(self, node_ids) -> None:
        """Read the wide columns of the given nodes in one query per 500 ids."""
        want = [nid for nid in node_ids if nid in self.nodes and self.nodes[nid]._full is None]
        if not want:
            return
        tenant = normalize_graph_tenant_id(self.tenant_id)
        conn = self._connect()
        try:
            for a in range(0, len(want), 500):
                chunk = want[a: a + 500]
                q = (f"SELECT id, {', '.join(_NODE_LAZY_COLUMNS)} FROM graph_nodes WHERE tenant_id = ? AND scan_id = ? "
                     f"AND id IN ({','.join('?' * len(chunk))})")
                for row in conn.execute(q, [tenant, self.scan_id, *chunk]):
                    self.nodes[row[0]]._full = node_columns(row[1:])
        finally:
            conn.close()

    def hydrate_edges(self, edges) -> None:
        """Read the wide columns of the given edge records, 250 rows per query."""
        want = [e for e in edges if isinstance(e, SnapshotEdge) and e._full is None]
        if not want:
            return
        tenant = normalize_graph_tenant_id(self.tenant_id)
        by_row: dict[tuple[str, str, str], list[SnapshotEdge]] = {}
        for e in want:
            by_row.setdefault(e._row, []).append(e)
        keys = list(by_row)
        conn = self._connect()
        try:
            for a in range(0, len(keys), 250):
                chunk = keys[a: a + 250]
                q = (f"SELECT source_id, target_id, relationship, {', '.join(_EDGE_LAZY_COLUMNS)} FROM graph_edges WHERE tenant_id = ? AND scan_id = ? "
                     f"AND (source_id, target_id, relationship) IN (VALUES {','.join(['(?,?,?)'] * len(chunk))})")
                params = [tenant, self.scan_id]
                for k in chunk:
                    params.extend(k)
                for row in conn.execute(q, params):
                    full = edge_columns(row[3:], self.scan_id)
                    for e in by_row.get((row[0], row[1], row[2]), ()):
                        e._full = full
        finally:
            conn.close()
        for e in want:
            if e._full is None:        # row vanished under us
                e._full = {"first_seen": "", "last_seen": "", "valid_from": "", "valid_to": None, "confidence": 1.0, "provenance": {},
                           "source_scan_id": self.scan_id, "source_run_id": "", "evidence": {}, "activity_id": 1}

    def traverse_subgraph(self, roots, **kwargs):
        sub, depths, truncated = super().traverse_subgraph(roots, **kwargs)
        self.hydrate_nodes(list(sub.nodes))            # a few queries for the whole answer instead of one per record
        self.hydrate_edges(sub.edges)
        return sub, depths, truncated


def load_snapshot(db: str | Path | sqlite3.Connection, *, tenant_id: str = "", scan_id: str = "", device: int = 0) -> SnapshotGraph:
    """Load one snapshot topology-first.  ``db`` is a path (or an open connection to a file database)."""
    if isinstance(db, sqlite3.Connection):
        conn, own = db, False
        path = next((row[2] for row in conn.execute("PRAGMA database_list") if row[1] == "main"), "")
    else:
        path, own = str(db), True
        conn = sqlite3.connect(f"file:{path}?mode=ro", uri=True, timeout=10)
    try:
        tenant = normalize_graph_tenant_id(tenant_id)
        effective, created_at = resolve_snapshot(conn, tenant_id=tenant, scan_id=scan_id)
        graph = SnapshotGraph(path, scan_id=effective, tenant_id=tenant, created_at=created_at, device=device)
        if not effective:
            graph._csr = csrmod.from_arrays([], np.zeros(0, np.uint8), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(0, np.uint8), n_real=0)
            return graph
        conn.row_factory = None
        ids: list[str] = []
        types: list[int] = []
        index: dict[str, int] = {}
        nodes = graph.nodes
        for nid, etype, label, status, risk, sev in conn.execute(
                "SELECT id, entity_type, label, status, risk_score, severity FROM graph_nodes WHERE tenant_id = ? AND scan_id = ?", (tenant, effective)):
            index[nid] = len(ids)
            ids.append(nid)
            types.append(ENTITY_CODE.get(etype, ENTITY_CODE_OTHER))
            nodes[nid] = SnapshotNode(graph, nid, etype, label, status, risk, sev or "")
        src: list[int] = []
        dst: list[int] = []
        rel: list[int] = []
        flags: list[int] = []
        weight: list[float] = []
        other: dict[int, str] = {}
        get = index.get
        for s, t, r, direction, w, trav in conn.execute(
                "SELECT source_id, target_id, relationship, direction, weight, traversable FROM graph_edges WHERE tenant_id = ? AND scan_id = ?", (tenant, effective)):
            si, ti = get(s), get(t)
            if si is None or ti is None:
                continue
            code = REL_CODE.get(r, REL_CODE_OTHER)
            if code == REL_CODE_OTHER:
                other[len(src)] = r
            src.append(si)
            dst.append(ti)
            rel.append(code)
            flags.append((EDGE_TRAVERSABLE if trav else 0) | (EDGE_BIDIRECTIONAL if direction == "bidirectional" else 0))
            weight.append(w if w is not None else 1.0)
        graph._e_src, graph._e_dst = np.asarray(src, dtype=np.int32), np.asarray(dst, dtype=np.int32)
        graph._e_rel, graph._e_flags = np.asarray(rel, dtype=np.uint8), np.asarray(flags, dtype=np.uint8)
        graph._e_weight, graph._e_other = np.asarray(weight, dtype=np.float32), other
        csr = csrmod.from_arrays(ids, np.asarray(types, dtype=np.uint8), graph._e_src, graph._e_dst, graph._e_rel, graph._e_flags, n_real=len(ids))
        csr.index = index
        graph._csr = csr
        for row in conn.execute("SELECT source_node, target_node, path_nodes, path_edges, composite_risk, summary, credential_exposure, tool_exposure, vuln_ids "
                                "FROM attack_paths WHERE tenant_id = ? AND scan_id = ?", (tenant, effective)):
            graph.attack_paths.append(AttackPath(source=row[0], target=row[1], hops=json.loads(row[2]), edges=json.loads(row[3]), composite_risk=row[4],
                                                 summary=row[5] or "", credential_exposure=json.loads(row[6]), tool_exposure=json.loads(row[7]),
                                                 vuln_ids=json.loads(row[8])))
        for row in conn.execute("SELECT pattern, agents, risk_score, description, owasp_agentic_tag FROM interaction_risks WHERE tenant_id = ? AND scan_id = ?",
                                (tenant, effective)):
            graph.interaction_risks.append(InteractionRisk(pattern=row[0], agents=json.loads(row[1]), risk_score=row[2], description=row[3], owasp_agentic_tag=row[4]))
        return graph
    finally:
        if own:
            conn.close()
