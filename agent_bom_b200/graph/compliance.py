"""Compliance posture served from the snapshot cache.

The reference's SQLite store answers ``compliance_summary`` (reference ``api/graph_store.py:950-1031``, ``GET /v1/graph/compliance``)
per request: it reads every tagged node of the scan, ``json.loads`` each row and loops in Python over every (node, tag) pair,
de-duplicating member nodes with a list scan, so a framework that tags k nodes costs O(k^2).  Here each cached graph gets a
compliance table once: the host reads the tagged rows with the reference's own query and interns them, the device rolls every
(row, tag) pair up per framework (``csrc/compliance.cuh``), and the host turns the table into the full answer, every framework
included.  A request then selects the framework its filter names; it sends no SQL beyond latest-scan resolution.

- Rows: ``json_array_length(compliance_tags) > 0`` in id order, the reference's SQL, so malformed JSON raises SQLite's error.
- Interning: ``json.loads`` once per distinct ``compliance_tags`` text; the framework rule (:999) once per distinct tag, in the
  order the reference first meets it, so a non-string tag raises what the reference raises.  Tags and frameworks are coded in
  sorted order, so the device's (framework, tag) order is the answer's.
- ``by_severity`` / ``by_entity_type`` keep first-appearance order: the device gives each (framework, key) run its first row.
"""

from __future__ import annotations

import json
import threading
from typing import Any

import numpy as np

from .lookup import connect

ROWS_SQL = ("SELECT id, entity_type, severity, compliance_tags FROM graph_nodes "
            "WHERE tenant_id = ? AND scan_id = ? AND json_array_length(compliance_tags) > 0 ORDER BY id ASC")
_lock = threading.Lock()


def framework_of(tag) -> str:
    """The reference's framework of a tag (:999), verbatim: Python's full case mapping included, and a non-string tag raises."""
    return tag.split("-")[0].upper() if "-" in tag else tag.upper()


def empty_summary(scan_id: str) -> dict[str, Any]:
    return {"scan_id": scan_id, "framework_count": 0, "total_tagged_findings": 0, "frameworks": {}}


class ComplianceInputs:
    """The tagged rows of one scan, interned: per row (id order) a text, severity and entity-type code; per distinct text its tag
    codes; per tag its framework code.  ``tags`` and ``frameworks`` are sorted, and codes are positions in them."""

    def __init__(self, rows):
        self.ids: list[str] = []
        texts: dict[str, int] = {}
        text_tags: list[list[int]] = []
        tag_ix: dict[str, int] = {}          # first-appearance codes, remapped to sorted order below
        tag_fw: list[str] = []
        sev_ix: dict[Any, int] = {}
        type_ix: dict[Any, int] = {}
        row_text, row_sev, row_type = [], [], []
        for node_id, entity_type, severity, raw in rows:
            t = texts.get(raw)
            if t is None:
                codes = []
                for tag in json.loads(raw):
                    c = tag_ix.get(tag) if isinstance(tag, str) else None
                    if c is None:
                        fw = framework_of(tag)
                        c = tag_ix[tag] = len(tag_fw)
                        tag_fw.append(fw)
                    codes.append(c)
                t = texts[raw] = len(text_tags)
                text_tags.append(codes)
            self.ids.append(node_id)
            row_text.append(t)
            row_sev.append(sev_ix.setdefault(severity or "unknown", len(sev_ix)))
            row_type.append(type_ix.setdefault(entity_type, len(type_ix)))
        self.tags = sorted(tag_ix)
        self.frameworks = sorted(set(tag_fw))
        fw_rank = {f: k for k, f in enumerate(self.frameworks)}
        rank = np.empty(len(tag_fw), np.int32)              # first-appearance code -> sorted code
        rank[np.fromiter((tag_ix[t] for t in self.tags), np.int64, len(self.tags))] = np.arange(len(self.tags), dtype=np.int32)
        self.tag_fw = np.fromiter((fw_rank[tag_fw[tag_ix[t]]] for t in self.tags), np.int32, len(self.tags))
        self.text_off = np.zeros(len(text_tags) + 1, np.int64)
        self.text_off[1:] = np.cumsum([len(c) for c in text_tags])
        flat = np.fromiter((c for codes in text_tags for c in codes), np.int64, int(self.text_off[-1]))
        self.text_tags = rank[flat] if flat.size else np.zeros(0, np.int32)
        self.row_text = np.asarray(row_text, np.int32)
        self.row_sev = np.asarray(row_sev, np.int32)
        self.row_type = np.asarray(row_type, np.int32)
        self.severities = list(sev_ix)
        self.types = list(type_ix)


def _counts(runs: np.ndarray, names: list, n_fw: int) -> list[dict]:
    """Per framework, ``{name: pairs}`` of its runs in first-row order."""
    order = np.lexsort((runs[3], runs[0]))
    fw, code, cnt = runs[0][order].tolist(), runs[1][order].tolist(), runs[2][order].tolist()
    out: list[dict] = [{} for _ in range(n_fw)]
    for f, c, k in zip(fw, code, cnt):
        out[f][names[c]] = k
    return out


def summarize(inputs: ComplianceInputs, table: dict[str, np.ndarray]) -> dict[str, dict[str, Any]]:
    """Every framework's entry, in sorted name order, from the device table."""
    n_fw = len(inputs.frameworks)
    by_sev = _counts(table["sev"], inputs.severities, n_fw)
    by_type = _counts(table["type"], inputs.types, n_fw)
    tags: list[list[str]] = [[] for _ in range(n_fw)]
    for f, c in zip(table["tag"][0].tolist(), table["tag"][1].tolist()):
        tags[f].append(inputs.tags[c])
    total = np.zeros(n_fw, np.int64)
    np.add.at(total, table["sev"][0], table["sev"][2])
    node_count = table["node_count"].tolist()
    rows = table["node_rows"].tolist()
    out: dict[str, dict[str, Any]] = {}
    at = 0
    for f, name in enumerate(inputs.frameworks):
        k = min(node_count[f], 100)
        out[name] = {"total_findings": int(total[f]), "by_severity": by_sev[f], "by_entity_type": by_type[f], "tags": tags[f],
                     "node_count": node_count[f], "node_ids": [inputs.ids[r] for r in rows[at: at + k]]}
        at += k
    return out


class ComplianceSummary:
    """Every framework of one graph's scan; a request selects from it."""

    def __init__(self, graph, db_path, tenant: str):
        conn = connect(db_path)
        try:
            rows = conn.execute(ROWS_SQL, (tenant, graph.scan_id)).fetchall()
        finally:
            conn.close()
        inputs = ComplianceInputs(rows)
        if inputs.ids:
            table = graph.device_graph.compliance_table(inputs.row_text, inputs.row_sev, inputs.row_type, inputs.text_off, inputs.text_tags,
                                                        inputs.tag_fw, len(inputs.frameworks), len(inputs.severities), len(inputs.types))
            self.frameworks = summarize(inputs, table)
        else:
            self.frameworks = {}
        self.total = sum(v["total_findings"] for v in self.frameworks.values())

    def select(self, scan_id: str, framework: str) -> dict[str, Any]:
        """The reference's body for ``framework`` (``""``: all).  The framework entries are shared by every call: read-only."""
        if not framework:
            frameworks, total = dict(self.frameworks), self.total
        else:
            entry = self.frameworks.get(framework.upper())
            frameworks = {} if entry is None else {framework.upper(): entry}
            total = 0 if entry is None else entry["total_findings"]
        return {"scan_id": scan_id, "framework_count": len(frameworks), "total_tagged_findings": total, "frameworks": frameworks}


def compliance_summary(graph, db_path, tenant: str, framework: str = "") -> dict[str, Any]:
    """``compliance_summary`` over ``graph`` (the resolved scan): built once per graph under the graph's own lock, so a first
    call on one graph never waits on another's; a build that raises caches nothing."""
    s = graph._compliance
    if s is None:
        with _lock:
            glock = graph.__dict__.setdefault("_compliance_lock", threading.Lock())
        with glock:
            s = graph._compliance
            if s is None:
                s = graph._compliance = ComplianceSummary(graph, db_path, tenant)
    return s.select(graph.scan_id, framework)
