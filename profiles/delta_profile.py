#!/usr/bin/env python3
"""Cost of the device snapshot diff (``graph/delta.py``) on columnar estates saved to SQLite.

    python profiles/delta_profile.py [--out DIR] [--sizes M1,M2] [--reps 3]

Per size the old snapshot is the ``agent_bom_b200.estate`` estate and the new one the same generator with 2 % more agents and
the first 1 % of agents left out, so most ids and edges are shared.  Both are written to one SQLite file with the store's
columns (one row per node and edge) and loaded topology-first.  Reported separately: the diff tables (host build and upload),
the match and edge-diff call (wall, and its kernels by name under torch.profiler in a separate call), the SQL rich-column pass,
building the response, the whole ``snapshot_diff`` (median of --reps after one warm call) and one ``compute_delta_alerts``.  The card's name and power limit
are read in the same run.  Writes DIR/delta_profile.json after every size (DIR defaults to a temporary directory).
"""

from __future__ import annotations

import argparse
import json
import sqlite3
import statistics
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from clusters_profile import kernel_table  # noqa: E402
from paths_profile import gpu_info  # noqa: E402

AGENTS = {"M1": 2_000, "M2": 20_700}
NOW = "2026-01-01T00:00:00+00:00"

DDL = [
    "CREATE TABLE graph_nodes (id TEXT NOT NULL, entity_type TEXT NOT NULL, label TEXT NOT NULL, category_uid INTEGER DEFAULT 0, "
    "class_uid INTEGER DEFAULT 0, type_uid INTEGER DEFAULT 0, status TEXT DEFAULT 'active', risk_score REAL DEFAULT 0.0, severity TEXT DEFAULT '', "
    "severity_id INTEGER DEFAULT 0, first_seen TEXT NOT NULL, last_seen TEXT NOT NULL, attributes TEXT DEFAULT '{}', compliance_tags TEXT DEFAULT '[]', "
    "data_sources TEXT DEFAULT '[]', dimensions TEXT DEFAULT '{}', scan_id TEXT NOT NULL, tenant_id TEXT NOT NULL DEFAULT 'default', "
    "PRIMARY KEY (id, scan_id, tenant_id))",
    "CREATE TABLE graph_edges (source_id TEXT NOT NULL, target_id TEXT NOT NULL, relationship TEXT NOT NULL, direction TEXT DEFAULT 'directed', "
    "weight REAL DEFAULT 1.0, traversable INTEGER DEFAULT 1, first_seen TEXT NOT NULL, last_seen TEXT NOT NULL, valid_from TEXT DEFAULT '', "
    "valid_to TEXT DEFAULT NULL, confidence REAL DEFAULT 1.0, provenance TEXT DEFAULT '{}', source_scan_id TEXT DEFAULT '', source_run_id TEXT DEFAULT '', "
    "evidence TEXT DEFAULT '{}', activity_id INTEGER DEFAULT 1, scan_id TEXT NOT NULL, tenant_id TEXT NOT NULL DEFAULT 'default', "
    "PRIMARY KEY (source_id, target_id, relationship, scan_id, tenant_id))",
    "CREATE INDEX idx_gn_tenant_scan ON graph_nodes(tenant_id, scan_id)",
    "CREATE INDEX idx_ge_tenant_scan ON graph_edges(tenant_id, scan_id)",
    "CREATE TABLE graph_snapshots (scan_id TEXT NOT NULL, tenant_id TEXT NOT NULL DEFAULT 'default', created_at TEXT NOT NULL, node_count INTEGER DEFAULT 0, "
    "edge_count INTEGER DEFAULT 0, risk_summary TEXT DEFAULT '{}', PRIMARY KEY (scan_id, tenant_id))",
    "CREATE TABLE attack_paths (source_node TEXT, target_node TEXT, hop_count INTEGER, composite_risk REAL, summary TEXT, path_nodes TEXT, path_edges TEXT, "
    "credential_exposure TEXT, tool_exposure TEXT, vuln_ids TEXT, scan_id TEXT, tenant_id TEXT, computed_at TEXT)",
    "CREATE TABLE interaction_risks (pattern TEXT, agents TEXT, risk_score REAL, description TEXT, owasp_agentic_tag TEXT, scan_id TEXT, tenant_id TEXT)",
]


def save(conn, g, scan: str, skip_agents: int) -> None:
    """Write one columnar graph as a snapshot, leaving out its first ``skip_agents`` agents and their edges."""
    from agent_bom_b200.graph.schema import ENTITY_VALUES, RELATIONSHIP_VALUES

    cols = g._cols
    ids, labels, sev, risk = cols.ids, cols.labels, cols.severity, cols.risk
    types = bytes(cols.types)
    skip = set([ids[i] for i in range(len(ids)) if types[i] == 0][:skip_agents])
    conn.executemany("INSERT INTO graph_nodes (id, entity_type, label, risk_score, severity, first_seen, last_seen, scan_id, tenant_id) VALUES (?,?,?,?,?,?,?,?,?)",
                     ((ids[i], ENTITY_VALUES[types[i]] if types[i] < len(ENTITY_VALUES) else "other", labels[i], risk[i], sev[i], NOW, NOW, scan, "default")
                      for i in range(len(ids)) if ids[i] not in skip))
    all_ids = g.csr.node_ids
    csr = g.csr
    rels = list(RELATIONSHIP_VALUES) + ["other"]
    conn.executemany("INSERT INTO graph_edges (source_id, target_id, relationship, direction, weight, traversable, first_seen, last_seen, evidence, scan_id, tenant_id) "
                     "VALUES (?,?,?,?,?,?,?,?,?,?,?)",
                     ((all_ids[s], all_ids[t], rels[r], "bidirectional" if f & 2 else "directed", float(w), f & 1, NOW, NOW, '{"v": 1}', scan, "default")
                      for s, t, r, f, w in zip(csr.src.tolist(), csr.dst.tolist(), csr.rel.tolist(), csr.flags.tolist(), g._e_weight.tolist())
                      if all_ids[s] not in skip and all_ids[t] not in skip))
    conn.execute("INSERT INTO graph_snapshots VALUES (?, 'default', ?, 0, 0, '{}')", (scan, NOW if scan == "old" else "2026-01-02T00:00:00+00:00"))
    conn.commit()


def profile_size(size: str, reps: int, work: Path) -> dict:
    import torch

    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report, delta
    from agent_bom_b200.graph.snapshot import load_snapshot

    agents = AGENTS[size]
    db = work / f"delta_{size}.sqlite"
    db.unlink(missing_ok=True)
    conn = sqlite3.connect(str(db))
    for stmt in DDL:
        conn.execute(stmt)
    t0 = time.perf_counter()
    for scan, n, skip in (("old", agents, 0), ("new", int(agents * 1.02), agents // 100)):
        est = estate.generate(n, 2145, estate.BENCH_KNOBS, exact_rank=False)
        save(conn, build_unified_graph_from_report(est.report_json(), columnar=True), scan, skip)
    conn.close()
    rec = {"agents_old": agents, "agents_new": int(agents * 1.02), "write_sqlite_s": round(time.perf_counter() - t0, 1)}
    t0 = time.perf_counter()
    old, new = load_snapshot(db, scan_id="old"), load_snapshot(db, scan_id="new")
    rec["load_s"] = round(time.perf_counter() - t0, 2)
    rec.update(nodes_old=len(old.nodes), edges_old=len(old.edges), nodes_new=len(new.nodes), edges_new=len(new.edges))
    _ = old.device_graph, new.device_graph
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    to, tn = delta.delta_table(old), delta.delta_table(new)
    rec["table_host_s"] = round(time.perf_counter() - t0, 3)
    t0 = time.perf_counter()
    to.ensure_device(old)
    tn.ensure_device(new)
    rec["table_upload_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
    rec["table_device_bytes"] = old.device_graph.delta_table_bytes() + new.device_graph.delta_table_bytes()
    delta.device_diff(old, new)                      # warm: module load, cub algorithm selection
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = delta.device_diff(old, new)
        ts.append(time.perf_counter() - t0)
    rec["match_and_edge_diff_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "reps": reps}
    rec["kernels_ms"] = kernel_table(lambda: delta.device_diff(old, new))
    rec["device_counts"] = {k: int(v.size) for k, v in d.items()}
    runs = []
    for _ in range(reps):
        t = {}
        t0 = time.perf_counter()
        body = delta.snapshot_diff(old, new, timings=t)
        t["total_s"] = time.perf_counter() - t0
        runs.append(t)
    rec["snapshot_diff_s"] = {k: round(statistics.median(r[k] for r in runs), 3) for k in runs[0]}
    rec["answer"] = {k: len(v) for k, v in body.items()}
    from agent_bom_b200.graph import compute_delta_alerts

    t0 = time.perf_counter()
    alerts = compute_delta_alerts(old, new)
    rec["compute_delta_alerts_s"] = round(time.perf_counter() - t0, 3)
    rec["alerts"] = len(alerts)
    db.unlink(missing_ok=True)
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="M1,M2")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="delta_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    doc = {"device": gpu_info(), "sizes": {}}
    work = Path(tempfile.mkdtemp(prefix="delta_db_"))
    for size in a.sizes.split(","):
        doc["sizes"][size] = profile_size(size, a.reps, work)
        (out / "delta_profile.json").write_text(json.dumps(doc, indent=1))
        print(size, json.dumps(doc["sizes"][size]), flush=True)
    print(f"-> {out / 'delta_profile.json'}")


if __name__ == "__main__":
    main()
