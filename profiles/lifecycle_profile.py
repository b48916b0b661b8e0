#!/usr/bin/env python3
"""Cost of the edge lifecycle reads (``graph/lifecycle.py``, ``graph/delta.py``) on the M1 columnar estate saved as S perturbed snapshots.

    python profiles/lifecycle_profile.py [--out DIR] [--snapshots 2,8] [--reps 5]

Snapshot s is the 2 000-agent estate (even s) or its 2 % larger copy (odd s) with a different run of agents left out; each save
closes ``valid_to`` on the previous snapshot's edges it drops, as the SQLite store's save does.  Reported separately per S: the
history build (SQL pass, host interning, upload and device sort), the per-call device time (CUDA events over repeated calls), the
hydration of the winners' rows, and end-to-end ``active_edges_at`` (warm) and ``changed_edges_between_scans`` (first -> last
snapshot).  The card's name and power limit are read in the same run.  Writes DIR/lifecycle_profile.json.
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

from delta_profile import DDL, save  # noqa: E402
from paths_profile import gpu_info  # noqa: E402

AGENTS = 2_000


def stamp(s: int) -> str:
    return f"2026-01-{s + 1:02d}T00:00:00+00:00"


def write_history(db: Path, snapshots: int, graphs) -> float:
    conn = sqlite3.connect(str(db))
    for stmt in DDL:
        conn.execute(stmt)
    t0 = time.perf_counter()
    for s in range(snapshots):
        scan = f"s{s}"
        save(conn, graphs[s % 2], scan, (s * 37) % (AGENTS // 10))
        conn.execute("UPDATE graph_snapshots SET created_at = ? WHERE scan_id = ?", (stamp(s), scan))
        conn.execute("UPDATE graph_edges SET first_seen = ?, last_seen = ? WHERE scan_id = ?", (stamp(s), stamp(s), scan))
        if s:
            conn.execute("UPDATE graph_edges SET valid_to = COALESCE(valid_to, ?) WHERE scan_id = ? AND NOT EXISTS (SELECT 1 FROM graph_edges n "
                         "WHERE n.source_id = graph_edges.source_id AND n.target_id = graph_edges.target_id AND n.relationship = graph_edges.relationship "
                         "AND n.scan_id = ? AND n.tenant_id = graph_edges.tenant_id)", (stamp(s), f"s{s - 1}", scan))
        conn.commit()
        print(f"  wrote snapshot {scan} ({time.perf_counter() - t0:.0f} s)", flush=True)
    conn.close()
    return time.perf_counter() - t0


def profile(snapshots: int, reps: int, graphs, work: Path) -> dict:
    from agent_bom_b200.graph import delta, lifecycle
    from agent_bom_b200.graph.snapshot import load_snapshot

    db = work / f"lifecycle_{snapshots}.sqlite"
    db.unlink(missing_ok=True)
    rec: dict = {"snapshots": snapshots, "write_sqlite_s": round(write_history(db, snapshots, graphs), 1)}
    conn = sqlite3.connect(str(db))
    rec["edge_rows"] = conn.execute("SELECT COUNT(*) FROM graph_edges").fetchone()[0]
    rec["closed_rows"] = conn.execute("SELECT COUNT(*) FROM graph_edges WHERE valid_to IS NOT NULL").fetchone()[0]
    conn.close()
    after, middle = "2027-01-01T00:00:00+00:00", stamp(snapshots // 2)
    cache = lifecycle.HistoryCache(1)
    t = {}
    t0 = time.perf_counter()
    body = lifecycle.active_edges_at(cache, db, after, timings=t)
    t["total_s"] = time.perf_counter() - t0
    print(f"  history built: {t}", flush=True)
    rec["cold_active_edges_at_s"] = {k: round(v, 4) for k, v in t.items()}
    hist = next(iter(cache._entries.values()))
    rec["history"] = {"rows": hist.n_rows, "keys": hist.table.n_keys, "ids": len(hist.ids), "relationships": len(hist.rels),
                      "timestamps": len(hist.stamps), "device_bytes": hist.table.nbytes}
    for name, at in (("after", after), ("middle", middle)):
        r = lifecycle.timestamp_rank(hist.stamps, at)
        hist.table.active(r)
        dev, call = [], []
        for _ in range(max(reps, 20)):
            d = {}
            t0 = time.perf_counter()
            hist.table.active(r, d)
            call.append(time.perf_counter() - t0)
            dev.append(d["device_ms"])
        runs = []
        for _ in range(reps):
            t = {}
            t0 = time.perf_counter()
            body = lifecycle.active_edges_at(cache, db, at, timings=t)
            t["total_s"] = time.perf_counter() - t0
            runs.append(t)
        rec[f"active_{name}"] = {"edges": len(body), "device_ms_median": round(statistics.median(dev), 4), "device_ms_min": round(min(dev), 4),
                                 "call_with_readback_ms_median": round(statistics.median(call) * 1e3, 3),
                                 "warm_s": {k: round(statistics.median(x[k] for x in runs), 4) for k in ("fingerprint_s", "call_s", "hydrate_s", "total_s")}}
    print(f"  active_edges_at: {rec['active_after']}", flush=True)
    t0 = time.perf_counter()
    old, new = load_snapshot(db, scan_id="s0"), load_snapshot(db, scan_id=f"s{snapshots - 1}")
    rec["load_snapshots_s"] = round(time.perf_counter() - t0, 2)
    delta.changed_edges_between_scans(old, new)
    runs = []
    for _ in range(reps):
        t = {}
        t0 = time.perf_counter()
        ch = delta.changed_edges_between_scans(old, new, timings=t)
        t["total_s"] = time.perf_counter() - t0
        runs.append(t)
    rec["changed_edges_between_scans_s"] = {k: round(statistics.median(x[k] for x in runs), 4) for k in runs[0]}
    rec["changes"] = ch["summary"]
    db.unlink(missing_ok=True)
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--snapshots", default="2,8")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report

    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="lifecycle_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    doc = {"device": gpu_info(), "estate": f"M1 ({AGENTS} agents, columnar)", "sizes": {}}
    graphs = [build_unified_graph_from_report(estate.generate(n, 2145, estate.BENCH_KNOBS, exact_rank=False).report_json(), columnar=True)
              for n in (AGENTS, int(AGENTS * 1.02))]
    print("estates built", flush=True)
    work = Path(tempfile.mkdtemp(prefix="lifecycle_db_"))
    for s in (int(x) for x in a.snapshots.split(",")):
        doc["sizes"][f"S{s}"] = profile(s, a.reps, graphs, work)
        (out / "lifecycle_profile.json").write_text(json.dumps(doc, indent=1))
        print(f"S{s}", json.dumps(doc["sizes"][f"S{s}"]), flush=True)
    print(f"-> {out / 'lifecycle_profile.json'}")


if __name__ == "__main__":
    main()
