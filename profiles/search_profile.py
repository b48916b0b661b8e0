#!/usr/bin/env python3
"""Cost of node search and node pages (``graph/search.py``) through ``B200GraphStore`` on the M1 columnar estate saved to SQLite.

    python profiles/search_profile.py [--out DIR] [--sizes M1] [--reps 5]
    python profiles/search_profile.py --reference [--out DIR] [--reps 3] [--timeout 300]
                                        # the same calls on the unmodified SQLite store (needs the reference)

The estate is written with the store's columns as in delta_profile.py, plus one ``graph_node_search`` FTS5 row per node with the
reference schema.  Its ``search_text`` is id, label, entity type and severity joined and lowered, followed by ``{}`` twice: the
estate's nodes carry no tags, sources, attributes or dimensions, so only the dimensions JSON differs from what ``save_graph``
writes.  Recorded: the table build (host time on the first call, device bytes, kernels), and warm calls (median of --reps after
one warm call): a broad FTS query, a narrow one, a LIKE query, the second page of the broad query by cursor and the first agent
page of ``page_nodes``.  Kernel time of each call is taken under torch.profiler in a separate call.  The card's name and power
limit are read in the same run.  Writes DIR/search_profile.json (``--reference``: DIR/search_reference.json).
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
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from delta_profile import AGENTS, DDL, save  # noqa: E402

FTS_DDL = ("CREATE VIRTUAL TABLE IF NOT EXISTS graph_node_search USING fts5(tenant_id UNINDEXED, scan_id UNINDEXED, node_id UNINDEXED, "
           "entity_type, severity, compliance_tags, data_sources, search_text)")


def write_db(size: str, work: Path) -> tuple[Path, dict]:
    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report

    db = work / f"search_{size}.sqlite"
    db.unlink(missing_ok=True)
    conn = sqlite3.connect(str(db))
    for stmt in DDL:
        conn.execute(stmt)
    conn.execute(FTS_DDL)
    t0 = time.perf_counter()
    est = estate.generate(AGENTS[size], 2145, estate.BENCH_KNOBS, exact_rank=False)
    g = build_unified_graph_from_report(est.report_json(), columnar=True)
    save(conn, g, "old", 0)
    rows = conn.execute("SELECT id, entity_type, label, severity FROM graph_nodes WHERE scan_id = 'old'").fetchall()
    conn.executemany("INSERT INTO graph_node_search VALUES ('default', 'old', ?, ?, ?, '', '', ?)",
                     ((i, t, (s or "").lower(), " ".join(p for p in (i, lbl, t, s or "", "{}", "{}") if p).lower()) for i, t, lbl, s in rows))
    conn.execute("INSERT INTO graph_snapshots (scan_id, tenant_id, created_at, node_count, edge_count) SELECT 'old', 'default', '2026-01-01', 0, 0 "
                 "WHERE NOT EXISTS (SELECT 1 FROM graph_snapshots WHERE scan_id = 'old')")
    conn.commit()
    text_bytes = conn.execute("SELECT SUM(LENGTH(CAST(search_text AS BLOB))) FROM graph_node_search").fetchone()[0]
    conn.close()
    return db, {"agents": AGENTS[size], "nodes": len(rows), "index_text_bytes": int(text_bytes), "write_sqlite_s": round(time.perf_counter() - t0, 1)}


def timed(fn, reps: int) -> dict:
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": round(statistics.median(ts) * 1e3, 2), "min_ms": round(min(ts) * 1e3, 2), "reps": reps}


def calls(store) -> dict:
    def page2():
        _, _, nxt = store.search_nodes(scan_id="old", query="agent", limit=50)
        return store.search_nodes(scan_id="old", query="agent", limit=50, cursor=nxt)

    return {"fts_broad": lambda: store.search_nodes(scan_id="old", query="agent", limit=50),
            "fts_narrow": lambda: store.search_nodes(scan_id="old", query="agent-000123", limit=50),
            "like": lambda: store.search_nodes(scan_id="old", query="::", limit=50),
            "fts_broad_cursor_page2": page2,
            "agents_page": lambda: store.page_nodes(scan_id="old", entity_types={"agent"}, limit=50)}


def profile_size(size: str, reps: int, work: Path) -> dict:
    import torch
    from clusters_profile import kernel_table

    from agent_bom_b200.store import B200GraphStore

    db, rec = write_db(size, work)
    store = B200GraphStore(SimpleNamespace(_db_path=str(db), load_graph=lambda **_: None))
    g = store._graph("", "old")
    _ = g.device_graph
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    build_kernels = kernel_table(lambda: store.search_nodes(scan_id="old", query="agent", limit=50))
    rec["first_call_table_s"] = round(time.perf_counter() - t0, 3)      # reads, device table and fold probes, once per graph (profiled)
    rec["table_build_kernels_ms"] = build_kernels
    rec["search_table_bytes"] = g.device_graph.search_table_bytes()
    rec["search_table_bytes_per_node"] = round(rec["search_table_bytes"] / max(rec["nodes"], 1), 1)
    rec["wall"], rec["kernels_ms"] = {}, {}
    for name, fn in calls(store).items():
        rec["wall"][name] = timed(fn, reps)
        rec["kernels_ms"][name] = kernel_table(fn)
    c = calls(store)
    rec["totals"] = {k: (c[k]()[1] if k != "agents_page" else c[k]()[3]) for k in c}
    db.unlink(missing_ok=True)
    return rec


def _reference_call(db: str, name: str, reps: int, out) -> None:
    import oracle.make_golden  # noqa: F401  (puts the reference on the path)
    from agent_bom.api.graph_store import SQLiteGraphStore

    fn = calls(SQLiteGraphStore(db))[name]
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.put(time.perf_counter() - t0)


def reference_size(size: str, reps: int, work: Path, timeout_s: float) -> dict:
    """Each call in a child process of its own, ``reps`` times without a warm-up call, stopped after ``timeout_s``."""
    import multiprocessing as mp

    db, rec = write_db(size, work)
    ctx = mp.get_context("fork")
    rec["wall"] = {}
    for name in calls(None):
        q = ctx.Queue()
        p = ctx.Process(target=_reference_call, args=(str(db), name, reps, q))
        p.start()
        p.join(timeout_s)
        done = []
        while not q.empty():
            done.append(q.get())
        if p.is_alive():
            p.terminate()
            p.join()
            rec["wall"][name] = {"did_not_finish_within_s": timeout_s, "finished_reps": len(done)}
        else:
            rec["wall"][name] = {"median_ms": round(statistics.median(done) * 1e3, 2), "min_ms": round(min(done) * 1e3, 2), "reps": len(done)}
        print(name, rec["wall"][name], flush=True)
    db.unlink(missing_ok=True)
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="M1")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--timeout", type=float, default=300.0, help="--reference: seconds allowed per call")
    a = ap.parse_args()
    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="search_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    work = Path(tempfile.mkdtemp(prefix="search_db_"))
    if a.reference:
        import os
        import platform

        doc = {"store": "unmodified reference SQLiteGraphStore, one CPU process per call", "host": {"machine": platform.machine(),
               "cpu_count": os.cpu_count()}, "sizes": {}}
        name = "search_reference.json"
    else:
        from paths_profile import gpu_info

        doc = {"device": gpu_info(), "sizes": {}}
        name = "search_profile.json"
    for size in a.sizes.split(","):
        doc["sizes"][size] = reference_size(size, a.reps, work, a.timeout) if a.reference else profile_size(size, a.reps, work)
        (out / name).write_text(json.dumps(doc, indent=1))
        print(size, json.dumps(doc["sizes"][size]), flush=True)
    print(f"-> {out / name}")


if __name__ == "__main__":
    main()
