#!/usr/bin/env python3
"""Cost of warm record lookups (``graph/lookup.py``) through ``B200GraphStore`` on the M1 columnar estate saved to SQLite.

    python profiles/lookup_profile.py [--out DIR] [--sizes M1] [--reps 5]
    python profiles/lookup_profile.py --reference [--out DIR] [--reps 3] [--timeout 300]
                                        # the same calls on the unmodified SQLite store (needs the reference)

The estate is written with the store's columns as in delta_profile.py and loaded topology-first.  Timed calls (median of --reps
after one warm call): the drilldown (``bfs_paths`` + ``nodes_by_ids`` + ``edges_for_node_ids`` for the heaviest agent),
``node_context`` of a median-degree and of the highest-degree node, and ``snapshot_stats``.  Kernel time of each device call is
taken under torch.profiler in a separate call.  The card's name and power limit are read in the same run.  Writes
DIR/lookup_profile.json (``--reference``: DIR/lookup_reference.json).
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


def write_db(size: str, work: Path) -> tuple[Path, dict]:
    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report

    db = work / f"lookup_{size}.sqlite"
    db.unlink(missing_ok=True)
    conn = sqlite3.connect(str(db))
    for stmt in DDL:
        conn.execute(stmt)
    t0 = time.perf_counter()
    est = estate.generate(AGENTS[size], 2145, estate.BENCH_KNOBS, exact_rank=False)
    g = build_unified_graph_from_report(est.report_json(), columnar=True)
    save(conn, g, "old", 0)
    conn.close()
    csr = g.csr
    deg: dict[int, int] = {}
    for s, t in zip(csr.src.tolist(), csr.dst.tolist()):
        deg[s] = deg.get(s, 0) + 1
        if t != s:
            deg[t] = deg.get(t, 0) + 1
    ids = csr.node_ids
    order = sorted(deg, key=lambda i: (deg[i], ids[i]))
    agents = [i for i in range(csr.n_real) if csr.node_type[i] == 0]
    picks = {"highest_degree": ids[order[-1]], "median_degree": ids[order[len(order) // 2]],
             "heaviest_agent": ids[max(agents, key=lambda i: (deg.get(i, 0), ids[i]))]}
    return db, {"agents": AGENTS[size], "write_sqlite_s": round(time.perf_counter() - t0, 1), "degree": {k: deg[csr.idx(v)] for k, v in picks.items()}, **picks}


def timed(fn, reps: int) -> dict:
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": round(statistics.median(ts) * 1e3, 2), "min_ms": round(min(ts) * 1e3, 2), "reps": reps}


def calls(store, picks) -> dict:
    heavy = picks["heaviest_agent"]

    def drilldown():
        _paths, reach = store.bfs_paths(scan_id="old", source=heavy)
        ids = {heavy} | reach
        store.nodes_by_ids(scan_id="old", node_ids=ids)
        return store.edges_for_node_ids(scan_id="old", node_ids=ids)

    return {"drilldown": drilldown, "node_context_median": lambda: store.node_context(scan_id="old", node_id=picks["median_degree"]),
            "node_context_highest": lambda: store.node_context(scan_id="old", node_id=picks["highest_degree"]),
            "snapshot_stats": lambda: store.snapshot_stats(scan_id="old")}


def profile_size(size: str, reps: int, work: Path) -> dict:
    import torch
    from clusters_profile import kernel_table

    from agent_bom_b200.store import B200GraphStore

    db, rec = write_db(size, work)
    store = B200GraphStore(SimpleNamespace(_db_path=str(db), load_graph=lambda **_: None))
    t0 = time.perf_counter()
    g = store._graph("", "old")
    _ = g.device_graph
    torch.cuda.synchronize()
    rec.update(load_s=round(time.perf_counter() - t0, 2), nodes=len(g.nodes), edges=len(g.edges))
    t0 = time.perf_counter()
    store.snapshot_stats(scan_id="old")
    store.edges_for_node_ids(scan_id="old", node_ids={rec["median_degree"]})
    rec["first_call_tables_s"] = round(time.perf_counter() - t0, 2)      # the lookup table, the statistics and the left-out rows, once per graph
    rec["lookup_table_bytes"] = g.device_graph.lookup_table_bytes()
    rec["wall"] = {}
    rec["kernels_ms"] = {}
    for name, fn in calls(store, rec).items():
        rec["wall"][name] = timed(fn, reps)
        rec["kernels_ms"][name] = kernel_table(fn)
    rec["answer_rows"] = {"drilldown_edges": len(calls(store, rec)["drilldown"]()),
                          "context_highest": len(store.node_context(scan_id="old", node_id=rec["highest_degree"])["edges_out"])}
    db.unlink(missing_ok=True)
    return rec


def _reference_call(db: str, picks: dict, name: str, reps: int, out) -> None:
    import oracle.make_golden  # noqa: F401  (puts the reference on the path)
    from agent_bom.api.graph_store import SQLiteGraphStore

    fn = calls(SQLiteGraphStore(db), picks)[name]
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
        out.put(ts[-1])


def reference_size(size: str, reps: int, work: Path, timeout_s: float) -> dict:
    """Each call in a child process of its own, ``reps`` times without a warm-up call (the reference holds no cache between calls),
    stopped after ``timeout_s``: a call that does not finish is recorded as a lower bound."""
    import multiprocessing as mp

    db, rec = write_db(size, work)
    ctx = mp.get_context("fork")
    rec["wall"] = {}
    for name in ("snapshot_stats", "node_context_median", "node_context_highest", "drilldown"):
        q = ctx.Queue()
        p = ctx.Process(target=_reference_call, args=(str(db), rec, name, reps, q))
        t0 = time.perf_counter()
        p.start()
        p.join(timeout_s)
        done = []
        while not q.empty():
            done.append(q.get())
        if p.is_alive():
            p.terminate()
            p.join()
            rec["wall"][name] = {"did_not_finish_within_s": timeout_s, "finished_reps": len(done),
                                 "finished_ms": [round(t * 1e3, 1) for t in done]}
        else:
            rec["wall"][name] = {"median_ms": round(statistics.median(done) * 1e3, 2), "min_ms": round(min(done) * 1e3, 2), "reps": len(done)}
        rec["wall"][name]["elapsed_s"] = round(time.perf_counter() - t0, 1)
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
    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="lookup_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    work = Path(tempfile.mkdtemp(prefix="lookup_db_"))
    if a.reference:
        import os
        import platform

        doc = {"store": "unmodified reference SQLiteGraphStore, one CPU process per call", "host": {"machine": platform.machine(),
               "cpu_count": os.cpu_count()}, "sizes": {}}
        name = "lookup_reference.json"
    else:
        from paths_profile import gpu_info

        doc = {"device": gpu_info(), "sizes": {}}
        name = "lookup_profile.json"
    for size in a.sizes.split(","):
        doc["sizes"][size] = reference_size(size, a.reps, work, a.timeout) if a.reference else profile_size(size, a.reps, work)
        (out / name).write_text(json.dumps(doc, indent=1))
        print(size, json.dumps(doc["sizes"][size]), flush=True)
    print(f"-> {out / name}")


if __name__ == "__main__":
    main()
