"""Scan-to-scan snapshot diff (``GET /v1/graph/diff``) with the set arithmetic on the device.

The reference's ``diff_snapshots`` (``/root/reference/src/agent_bom/db/graph_store.py:671-738``) builds a metadata dict for every
node row and a ``(source, target, relationship)`` tuple for every edge row of both scans, and ``changed_edges_between_scans``
(``:799-842``) a full row dict for every edge row.  Here both snapshots are device graphs (``csrc/delta.cuh``):

- each graph gets its diff tables once (id bytes, sorted-order permutation, label bytes, status / severity codes, risk, per-edge
  relationship slot and flags), freed with the device graph;
- the device matches the two id sets, compares matched nodes and sorts and set-differences the edge keys, and returns only the
  added / removed / changed indices, already in the reference's ``sorted()`` order;
- the columns the topology-first loader does not hold (node ``severity_id``; edge ``weight``, ``direction`` string,
  ``confidence``, ``provenance``, ``evidence``, ``activity_id``) are compared by one SQL join per table over the primary key.
  Its candidates, and every pair the device leaves to the host, are decided by the reference's own row rules, so different
  JSON text that decodes to equal values is not a change;
- edge rows whose endpoints are not both nodes of their scan are stored but not loaded as graph edges; one SQL query per scan
  finds them and they are merged into the answer on the host;
- dicts are built only for the rows returned.

``changed_edges_between_scans`` reuses the same device diff and edge correction, plus the shared edge pairs the device already
matched (``abb_delta_shared_host``), and returns full rows for the added, removed and unchanged keys.
"""

from __future__ import annotations

import json
import sqlite3
import threading
from typing import Any

import numpy as np

from .schema import REL_CODE_OTHER, RELATIONSHIP_VALUES, enum_value

SEVERITY_CODES = {s: i for i, s in enumerate(("", "critical", "high", "medium", "low", "info", "informational", "none", "unknown"))}
STATUS_CODES = {s: i for i, s in enumerate(("", "active", "inactive", "vulnerable", "remediated"))}
CODE_OTHER = 255
REL_SLOTS = 64

_lock = threading.Lock()


def _risk(value) -> float:
    """The risk the store reads back: NULL and NaN (stored as NULL) read as 0.0."""
    r = float(value or 0.0)
    return 0.0 if r != r else r


def _text(value) -> str:
    return enum_value(value) if value is not None else ""


def _pack(strings) -> tuple[bytes, np.ndarray]:
    enc = [s.encode("utf-8", "surrogatepass") for s in strings]
    off = np.zeros(len(enc) + 1, np.int64)
    if enc:
        np.cumsum([len(b) for b in enc], out=off[1:])
    return b"".join(enc), off


def real_records(graph) -> list:
    """The node records of the graph's real nodes, in index order."""
    nodes = graph.nodes
    return [nodes[nid] for nid in graph.csr.node_ids[:graph.csr.n_real]]


def severity_codes(recs) -> np.ndarray:
    """``SEVERITY_CODES`` of each record's severity string; ``CODE_OTHER`` for a string outside the table."""
    return np.fromiter((SEVERITY_CODES.get(r.severity or "", CODE_OTHER) for r in recs), np.uint8, len(recs))


def relationship_slots(graph) -> tuple[np.ndarray, list[str]]:
    """Per original edge the slot of its relationship string, and the graph's distinct relationship strings in sorted order (the
    slot is the string's rank).  More than ``REL_SLOTS`` strings is an error."""
    codes = np.asarray(graph.csr.rel, np.int64)
    other = {int(i): enum_value(graph.edges[int(i)].relationship) for i in np.flatnonzero(codes == REL_CODE_OTHER)}
    names = sorted({RELATIONSHIP_VALUES[c] for c in np.unique(codes).tolist() if c != REL_CODE_OTHER} | set(other.values()))
    if len(names) > REL_SLOTS:
        raise ValueError(f"{len(names)} distinct relationships exceed the {REL_SLOTS} relationship slots")
    slot = {s: i for i, s in enumerate(names)}
    code_slot = np.zeros(32, np.uint8)
    for c, v in enumerate(RELATIONSHIP_VALUES):
        code_slot[c] = slot.get(v, 0)
    erel = code_slot[codes] if codes.size else np.zeros(0, np.uint8)
    for i, v in other.items():
        erel[i] = slot[v]
    return erel, names


class DeltaTable:
    """Host half of a graph's diff tables: the relationship strings of its slots, and the per-graph arrays uploaded once."""

    def __init__(self, graph):
        csr = graph.csr
        n_real = csr.n_real
        recs = real_records(graph)
        self.ids_bytes, self.id_off = _pack(csr.node_ids)
        self.perm = np.argsort(csr.node_rank, kind="stable").astype(np.int32)
        self.label_bytes, self.label_off = _pack([_text(r.label) for r in recs])
        self.status = np.fromiter((STATUS_CODES.get(_text(r.status), CODE_OTHER) for r in recs), np.uint8, n_real)
        self.severity = severity_codes(recs)
        self.risk = np.fromiter((_risk(r.risk_score) for r in recs), np.float64, n_real)
        self.erel, self.rel_names = relationship_slots(graph)
        self.eflag = np.ascontiguousarray(csr.flags, np.uint8)
        self.uploaded = False

    def ensure_device(self, graph) -> None:
        if not self.uploaded:
            csr = graph.csr
            graph.device_graph.build_delta_table(csr.n_real, self.ids_bytes, self.id_off, self.perm, self.label_bytes, self.label_off, self.status,
                                                 self.severity, self.risk, self.erel, self.eflag)
            self.uploaded = True


def delta_table(graph) -> DeltaTable:
    t = getattr(graph, "_delta", None)
    if t is None:
        with _lock:
            t = getattr(graph, "_delta", None)
            if t is None:
                t = graph._delta = DeltaTable(graph)
    return t


def device_diff(old, new, shared: bool = False) -> dict[str, np.ndarray]:
    """The device's answer for ``old`` -> ``new`` (``DeviceGraph.diff``), with the relationship slots of both graphs ranked together;
    ``shared`` adds the edge pairs whose key both graphs hold."""
    to, tn = delta_table(old), delta_table(new)
    union = sorted(set(to.rel_names) | set(tn.rel_names))
    if len(union) > REL_SLOTS:
        raise ValueError(f"{len(union)} distinct relationships exceed the diff's {REL_SLOTS}")
    rank = {s: i for i, s in enumerate(union)}
    with _lock:
        to.ensure_device(old)
        tn.ensure_device(new)
    relmaps = [rank[s] for s in to.rel_names], [rank[s] for s in tn.rel_names]
    if shared:
        return new.device_graph.diff(old.device_graph, *relmaps, shared=True)
    return new.device_graph.diff(old.device_graph, *relmaps)


# ── reference row rules (db/graph_store.py:680-689, 741-773), restated ──
def node_metadata(row) -> dict[str, Any]:
    return {"id": row["id"], "entity_type": row["entity_type"], "label": row["label"], "severity": row["severity"] or "",
            "severity_id": int(row["severity_id"] or 0), "risk_score": float(row["risk_score"] or 0.0), "status": row["status"] or ""}


def edge_history_row(row) -> dict[str, Any]:
    return {"source_id": row["source_id"], "target_id": row["target_id"], "relationship": row["relationship"], "direction": row["direction"],
            "weight": float(row["weight"] or 0.0), "traversable": bool(row["traversable"]), "first_seen": row["first_seen"], "last_seen": row["last_seen"],
            "valid_from": row["valid_from"] or row["first_seen"], "valid_to": row["valid_to"],
            "confidence": float(row["confidence"] if row["confidence"] is not None else 1.0), "provenance": json.loads(row["provenance"] or "{}"),
            "source_scan_id": row["source_scan_id"] or row["scan_id"], "source_run_id": row["source_run_id"] or "",
            "evidence": json.loads(row["evidence"] or "{}"), "activity_id": int(row["activity_id"] or 1), "scan_id": row["scan_id"], "tenant_id": row["tenant_id"]}


def edge_fingerprint(edge: dict[str, Any]) -> dict[str, Any]:
    return {k: edge[k] for k in ("direction", "weight", "traversable", "confidence", "provenance", "evidence", "activity_id")}


_NODE_COLS = "id, entity_type, label, status, severity, severity_id, risk_score"
_CHUNK = 300


def _node_rows(conn, tenant: str, scan: str, ids: list[str]) -> dict[str, dict[str, Any]]:
    out: dict[str, dict[str, Any]] = {}
    for a in range(0, len(ids), _CHUNK):
        chunk = ids[a: a + _CHUNK]
        q = f"SELECT {_NODE_COLS} FROM graph_nodes WHERE scan_id = ? AND tenant_id = ? AND id IN ({','.join('?' * len(chunk))})"
        for row in conn.execute(q, [scan, tenant, *chunk]):
            out[row["id"]] = node_metadata(row)
    return out


def _edge_rows(conn, tenant: str, scan: str, keys: list[tuple[str, str, str]]) -> dict[tuple[str, str, str], dict[str, Any]]:
    out: dict[tuple[str, str, str], dict[str, Any]] = {}
    for a in range(0, len(keys), _CHUNK):
        chunk = keys[a: a + _CHUNK]
        q = ("SELECT * FROM graph_edges WHERE scan_id = ? AND tenant_id = ? AND (source_id, target_id, relationship) IN "
             f"(VALUES {','.join(['(?,?,?)'] * len(chunk))})")
        params: list[Any] = [scan, tenant]
        for k in chunk:
            params.extend(k)
        for row in conn.execute(q, params):
            out[(row["source_id"], row["target_id"], row["relationship"])] = edge_history_row(row)
    return out


def rich_node_candidates(conn, tenant: str, old_scan: str, new_scan: str) -> list[str]:
    """Shared node ids whose ``severity_id`` column differs (the one node column the loader does not hold)."""
    return [r[0] for r in conn.execute(
        "SELECT n.id FROM graph_nodes o JOIN graph_nodes n ON n.id = o.id AND n.scan_id = ? AND n.tenant_id = o.tenant_id "
        "WHERE o.scan_id = ? AND o.tenant_id = ? AND o.severity_id IS NOT n.severity_id", (new_scan, old_scan, tenant))]


def rich_edge_candidates(conn, tenant: str, old_scan: str, new_scan: str) -> list[tuple[str, str, str]]:
    """Shared edge keys whose stored text or number differs in a column the device does not compare."""
    return [tuple(r) for r in conn.execute(
        "SELECT n.source_id, n.target_id, n.relationship FROM graph_edges o JOIN graph_edges n ON n.source_id = o.source_id AND "
        "n.target_id = o.target_id AND n.relationship = o.relationship AND n.scan_id = ? AND n.tenant_id = o.tenant_id "
        "WHERE o.scan_id = ? AND o.tenant_id = ? AND (o.weight IS NOT n.weight OR o.direction IS NOT n.direction OR "
        "o.confidence IS NOT n.confidence OR o.provenance IS NOT n.provenance OR o.evidence IS NOT n.evidence OR "
        "o.activity_id IS NOT n.activity_id)", (new_scan, old_scan, tenant))]


def unloaded_edge_keys(conn, tenant: str, scan: str) -> set[tuple[str, str, str]]:
    """Stored edge rows of a scan whose endpoints are not both nodes of it: the topology-first loader drops them."""
    return {tuple(r) for r in conn.execute(
        "SELECT e.source_id, e.target_id, e.relationship FROM graph_edges e WHERE e.scan_id = ? AND e.tenant_id = ? AND ("
        "NOT EXISTS (SELECT 1 FROM graph_nodes s WHERE s.id = e.source_id AND s.scan_id = e.scan_id AND s.tenant_id = e.tenant_id) OR "
        "NOT EXISTS (SELECT 1 FROM graph_nodes t WHERE t.id = e.target_id AND t.scan_id = e.scan_id AND t.tenant_id = e.tenant_id))",
        (scan, tenant))}


def _edge_key(graph, e: int) -> tuple[str, str, str]:
    csr = graph.csr
    code = int(csr.rel[e])
    rel = RELATIONSHIP_VALUES[code] if code != REL_CODE_OTHER else enum_value(graph.edges[e].relationship)
    return csr.node_ids[int(csr.src[e])], csr.node_ids[int(csr.dst[e])], rel


def _holds_unloaded_edges(graph) -> bool:
    """A snapshot graph loaded topology-first (graph/snapshot.py) has no edge whose endpoint lacks a node row."""
    from .snapshot import SnapshotGraph

    return isinstance(graph, SnapshotGraph)


def _edge_sql(conn, tenant: str, old, new, old_scan: str, new_scan: str, nodeless: bool = False):
    """The SQL half of the edge comparison: shared keys with a differing stored column, and each scan's rows the loader dropped.
    ``nodeless``: a graph without nodes stands for a named scan whose stored edge rows (if any) all lack their endpoints."""
    def unloaded(g, scan):
        if _holds_unloaded_edges(g) or (nodeless and scan and not g.nodes):
            return unloaded_edge_keys(conn, tenant, scan)
        return set()

    return rich_edge_candidates(conn, tenant, old_scan, new_scan), unloaded(old, old_scan), unloaded(new, new_scan)


def _edge_changes(conn, tenant: str, old, new, old_scan: str, new_scan: str, d: dict[str, np.ndarray], sql) -> dict[str, Any]:
    """The edge half of a diff: ``added`` / ``removed`` keys and ``changed`` {before, after} rows in key order, from the device's
    lists corrected by the stored rows the loaded graphs do not hold; with ``d["shared_new"]`` also the ``unchanged`` keys (every key
    both scans store, minus the changed ones)."""
    rich_edges, go, gn = sql
    e_add = [_edge_key(new, e) for e in d["edges_added"].tolist()]
    e_rem = [_edge_key(old, e) for e in d["edges_removed"].tolist()]
    e_chg = {_edge_key(new, e) for e in d["echanged_new"].tolist()}
    shared_unloaded: list[tuple[str, str, str]] = []
    if go or gn:
        in_old = set(_edge_rows(conn, tenant, old_scan, sorted(gn)))
        in_new = set(_edge_rows(conn, tenant, new_scan, sorted(go)))
        shared_unloaded = sorted((gn & in_old) | (go & in_new))
        e_add = sorted([k for k in e_add if k not in go] + [k for k in gn if k not in in_old])
        e_rem = sorted([k for k in e_rem if k not in gn] + [k for k in go if k not in in_new])
    check_e = sorted((set(rich_edges) | set(shared_unloaded) | e_chg))
    before = _edge_rows(conn, tenant, old_scan, check_e)
    after = _edge_rows(conn, tenant, new_scan, check_e)
    changed_keys = [k for k in check_e if k in before and k in after and (k in e_chg or edge_fingerprint(before[k]) != edge_fingerprint(after[k]))]
    out = {"added": e_add, "removed": e_rem, "changed": [{"before": before[k], "after": after[k]} for k in changed_keys]}
    if "shared_new" in d:
        gone = set(changed_keys)
        shared = {_edge_key(new, e) for e in d["shared_new"].tolist()} | set(shared_unloaded)
        out["unchanged"] = sorted(k for k in shared if k not in gone)
    return out


def snapshot_diff(old, new, *, db_path=None, tenant_id: str | None = None, timings: dict | None = None) -> dict[str, Any]:
    """The body of the reference ``diff_snapshots(old.scan_id, new.scan_id)`` for two snapshots persisted in ``db_path`` (default: the
    graphs' own database), with ``old`` and ``new`` as their device graphs.  ``timings`` (optional) receives the seconds of each stage."""
    import time

    from .snapshot import normalize_graph_tenant_id

    db_path = db_path or getattr(new, "db_path", None) or getattr(old, "db_path", None)
    if not db_path:
        raise ValueError("snapshot_diff compares persisted snapshots: pass db_path")
    tenant = normalize_graph_tenant_id(new.tenant_id if tenant_id is None else tenant_id)
    old_scan, new_scan = old.scan_id or "", new.scan_id or ""
    t = {}
    t0 = time.perf_counter()
    d = device_diff(old, new)
    t["device_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    conn = sqlite3.connect(f"file:{db_path}?mode=ro", uri=True, timeout=10)
    conn.row_factory = sqlite3.Row
    try:
        rich_nodes = rich_node_candidates(conn, tenant, old_scan, new_scan)
        sql = _edge_sql(conn, tenant, old, new, old_scan, new_scan)
        t["sql_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        oids, nids = old.csr.node_ids, new.csr.node_ids
        # nodes: added / removed rows straight from the device's id-ordered indices
        added_ids = [nids[i] for i in d["nodes_added"].tolist()]
        removed_ids = [oids[i] for i in d["nodes_removed"].tolist()]
        new_rows = _node_rows(conn, tenant, new_scan, added_ids)
        old_rows = _node_rows(conn, tenant, old_scan, removed_ids)
        changed = {nids[i] for i, f in zip(d["changed_new"].tolist(), d["changed_flag"].tolist()) if f == 1}
        check = [nids[i] for i, f in zip(d["changed_new"].tolist(), d["changed_flag"].tolist()) if f == 2]
        check += [nid for nid in rich_nodes if nid not in changed]
        if check:
            a, b = _node_rows(conn, tenant, old_scan, check), _node_rows(conn, tenant, new_scan, check)
            changed.update(nid for nid in check if nid in a and nid in b and a[nid] != b[nid])
        # edges: device lists in key order, corrected by the stored rows the loaded graphs do not hold
        edges = _edge_changes(conn, tenant, old, new, old_scan, new_scan, d, sql)
        body = {
            "nodes_added": [new_rows[nid] for nid in added_ids],
            "nodes_removed": [old_rows[nid] for nid in removed_ids],
            "nodes_changed": sorted(changed),
            "edges_added": edges["added"],
            "edges_removed": edges["removed"],
            "edges_changed": edges["changed"],
        }
        t["response_s"] = time.perf_counter() - t0
    finally:
        conn.close()
    if timings is not None:
        timings.update(t)
    return body


_FULL_SCAN = 2000      # above this many keys one pass over the scan's rows beats keyed lookups


def _rows_of(conn, tenant: str, scan: str, keys: list[tuple[str, str, str]]) -> dict[tuple[str, str, str], dict[str, Any]]:
    """Full history rows of ``keys`` in one scan: keyed lookups for a few, one pass over the scan's rows for many."""
    if len(keys) <= _FULL_SCAN:
        return _edge_rows(conn, tenant, scan, keys)
    want = set(keys)
    out: dict[tuple[str, str, str], dict[str, Any]] = {}
    for row in conn.execute("SELECT * FROM graph_edges WHERE scan_id = ? AND tenant_id = ?", (scan, tenant)):
        k = (row["source_id"], row["target_id"], row["relationship"])
        if k in want:
            out[k] = edge_history_row(row)
    return out


def changed_edges_between_scans(old, new, *, db_path=None, tenant_id: str | None = None, timings: dict | None = None) -> dict[str, Any]:
    """The body of the reference ``changed_edges_between_scans(old.scan_id, new.scan_id)`` (db/graph_store.py:799-841) for two
    snapshots persisted in ``db_path``, with ``old`` and ``new`` as their device graphs.  The key sets come from the device diff (its
    shared pairs give the unchanged edges) corrected as ``snapshot_diff`` corrects them; ``edges_changed`` is exactly the diff's.
    Rows are built only for the keys returned.  ``timings`` (optional) receives the seconds of each stage."""
    import time

    from .snapshot import normalize_graph_tenant_id

    db_path = db_path or getattr(new, "db_path", None) or getattr(old, "db_path", None)
    if not db_path:
        raise ValueError("changed_edges_between_scans compares persisted snapshots: pass db_path")
    tenant = normalize_graph_tenant_id(new.tenant_id if tenant_id is None else tenant_id)
    old_scan, new_scan = old.scan_id or "", new.scan_id or ""
    t = {}
    t0 = time.perf_counter()
    d = device_diff(old, new, shared=True)
    t["device_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    conn = sqlite3.connect(f"file:{db_path}?mode=ro", uri=True, timeout=10)
    conn.row_factory = sqlite3.Row
    try:
        conn.execute("BEGIN")          # one read transaction: every row below comes from one state of the database
        sql = _edge_sql(conn, tenant, old, new, old_scan, new_scan, nodeless=True)
        t["sql_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        edges = _edge_changes(conn, tenant, old, new, old_scan, new_scan, d, sql)
        new_rows = _rows_of(conn, tenant, new_scan, sorted(set(edges["added"]) | set(edges["unchanged"])))
        old_rows = _rows_of(conn, tenant, old_scan, edges["removed"])
        conn.rollback()
        body = {
            "scan_id_old": old_scan,
            "scan_id_new": new_scan,
            "edges_added": [new_rows[k] for k in edges["added"]],
            "edges_removed": [old_rows[k] for k in edges["removed"]],
            "edges_changed": edges["changed"],
            "edges_unchanged": [new_rows[k] for k in edges["unchanged"]],
            "summary": {"added": len(edges["added"]), "removed": len(edges["removed"]), "changed": len(edges["changed"]),
                        "unchanged": len(edges["unchanged"])},
        }
        t["response_s"] = time.perf_counter() - t0
    finally:
        conn.close()
    if timings is not None:
        timings.update(t)
    return body
