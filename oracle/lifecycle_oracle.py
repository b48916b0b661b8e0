"""CPU restatements of the two edge lifecycle reads, used only to check the device path.

- ``active_edges_at(conn, at, tenant_id)`` and ``changed_edges_between_scans(conn, old, new, tenant_id)`` answer from plain Python
  over every stored row: timestamps compared as Python strings (code-point order, which is SQLite's ``BINARY`` order of UTF-8 text),
  versions ranked by ``(created_at, scan_id)``, keys sorted as string tuples.  tests/test_lifecycle.py checks them against the
  reference's goldens (oracle/make_lifecycle_golden.py), and the device is checked against them on seeded random histories.
- ``HistoryOracle`` answers ``engine.EdgeHistory.active`` from the coded rows, and ``SharedDeltaOracle`` adds the shared edge pairs
  to ``DeltaOracle.diff``, so the host pipelines run without a GPU.
"""

from __future__ import annotations

import json
from typing import Any

import numpy as np
from oracle.delta_oracle import DeltaOracle


def _tenant(tenant_id) -> str:
    return (tenant_id or "").strip() or "default"


def history_row(row: dict[str, Any]) -> dict[str, Any]:
    """The stored row as the edge lifecycle reads return it: empty valid_from reads as first_seen, NULL numbers and JSON as their
    column defaults."""
    def num(v, default):
        return float(default if v is None else v)

    return {
        "source_id": row["source_id"], "target_id": row["target_id"], "relationship": row["relationship"], "direction": row["direction"],
        "weight": num(row["weight"] or None, 0.0), "traversable": row["traversable"] not in (0, None), "first_seen": row["first_seen"],
        "last_seen": row["last_seen"], "valid_from": row["valid_from"] if row["valid_from"] else row["first_seen"], "valid_to": row["valid_to"],
        "confidence": num(row["confidence"], 1.0), "provenance": json.loads(row["provenance"]) if row["provenance"] else {},
        "source_scan_id": row["source_scan_id"] if row["source_scan_id"] else row["scan_id"], "source_run_id": row["source_run_id"] or "",
        "evidence": json.loads(row["evidence"]) if row["evidence"] else {}, "activity_id": int(row["activity_id"]) if row["activity_id"] else 1,
        "scan_id": row["scan_id"], "tenant_id": row["tenant_id"],
    }


def _rows(conn, sql: str, params) -> list[dict[str, Any]]:
    cur = conn.execute(sql, params)
    names = [d[0] for d in cur.description]
    return [dict(zip(names, r)) for r in cur.fetchall()]


def active_edges_at(conn, at: str, tenant_id: str = "") -> list[dict[str, Any]]:
    tenant = _tenant(tenant_id)
    created = {r["scan_id"]: r["created_at"] for r in _rows(conn, "SELECT scan_id, created_at FROM graph_snapshots WHERE tenant_id = ?", (tenant,))}
    best: dict[tuple[str, str, str], tuple[tuple[str, str], dict]] = {}
    for row in _rows(conn, "SELECT * FROM graph_edges WHERE tenant_id = ?", (tenant,)):
        if row["scan_id"] not in created:
            continue
        version = (created[row["scan_id"]], row["scan_id"])
        vf = row["valid_from"] if row["valid_from"] else row["first_seen"]
        vt = row["valid_to"]
        if not (version[0] <= at and vf is not None and vf <= at and (vt is None or vt == "" or vt > at)):
            continue
        key = (row["source_id"], row["target_id"], row["relationship"])
        if key not in best or best[key][0] < version:
            best[key] = (version, row)
    return [history_row(best[k][1]) for k in sorted(best)]


_FINGERPRINT = ("direction", "weight", "traversable", "confidence", "provenance", "evidence", "activity_id")


def changed_edges_between_scans(conn, old: str, new: str, tenant_id: str = "") -> dict[str, Any]:
    tenant = _tenant(tenant_id)

    def scan(s):
        rows = _rows(conn, "SELECT * FROM graph_edges WHERE tenant_id = ? AND scan_id = ?", (tenant, s))
        return {(r["source_id"], r["target_id"], r["relationship"]): history_row(r) for r in rows}

    a, b = scan(old), scan(new)
    changed, unchanged = [], []
    for k in sorted(a.keys() & b.keys()):
        same = all(a[k][f] == b[k][f] for f in _FINGERPRINT)
        (unchanged.append(b[k]) if same else changed.append({"before": a[k], "after": b[k]}))
    added = [b[k] for k in sorted(b.keys() - a.keys())]
    removed = [a[k] for k in sorted(a.keys() - b.keys())]
    return {"scan_id_old": old, "scan_id_new": new, "edges_added": added, "edges_removed": removed, "edges_changed": changed,
            "edges_unchanged": unchanged, "summary": {"added": len(added), "removed": len(removed), "changed": len(changed), "unchanged": len(unchanged)}}


class HistoryOracle:
    """``engine.EdgeHistory`` on the CPU: rows grouped by key (stable), the last active version of each key."""

    def __init__(self, src, tgt, rel, created, valid_from, valid_to, n_ids, n_rels, *, device=0, id_limit=None):
        limit = (1 << 27) if id_limit is None else id_limit
        if n_ids > limit:
            raise ValueError(f"{n_ids} distinct edge endpoint ids exceed the history key's limit of {limit}")
        keys = list(zip(np.asarray(src).tolist(), np.asarray(tgt).tolist(), np.asarray(rel).tolist()))
        order = sorted(range(len(keys)), key=lambda i: keys[i])
        self.segments: list[list[int]] = []
        for i in order:
            if self.segments and keys[self.segments[-1][0]] == keys[i]:
                self.segments[-1].append(i)
            else:
                self.segments.append([i])
        self.cr, self.vf, self.vt = (np.asarray(c).tolist() for c in (created, valid_from, valid_to))

    def active(self, r: int, timing=None) -> np.ndarray:
        out = []
        for seg in self.segments:
            for i in reversed(seg):
                if self.cr[i] < r and self.vf[i] < r and self.vt[i] >= r:
                    out.append(i)
                    break
        return np.asarray(out, np.int32)


class SharedDeltaOracle(DeltaOracle):
    """``DeltaOracle`` whose ``diff(shared=True)`` also returns the edge pairs whose key both graphs hold, in key order."""

    def diff(self, old, relmap_old, relmap_new, shared: bool = False):
        out = super().diff(old, relmap_old, relmap_new)
        if shared:
            a, b = self.t, old.t
            union = sorted(set(a["ids"]) | set(b["ids"]))
            urank = {s: i for i, s in enumerate(union)}

            def keys(t, c, relmap):
                return {(urank[t["ids"][int(s)]], urank[t["ids"][int(d)]], int(relmap[int(r)])): e
                        for e, (s, d, r) in enumerate(zip(c.src.tolist(), c.dst.tolist(), t["erel"].tolist()))}

            ka, kb = keys(a, self.csr, relmap_new), keys(b, old.csr, relmap_old)
            both = sorted(ka.keys() & kb.keys())
            out["shared_new"] = np.asarray([ka[k] for k in both], np.int32)
            out["shared_old"] = np.asarray([kb[k] for k in both], np.int32)
        return out
