#!/usr/bin/env python3
"""Cost of the semantic-cluster view on columnar estates (``Estate.report_json()`` through the columnar builder).

    python profiles/clusters_profile.py [--out DIR] [--reps 5] [--sizes M2,L]

Per size: the host key-table build (wall), the device build (``abb_clusters_build_host``: wall, and its kernels by name under
torch.profiler in a separate call), a warm ``semantic_clusters_view`` with the defaults (median of --reps after one warm-up) and
the bytes its fetch copies back.  The card's name and power limit are read in the same run.  Writes DIR/clusters_profile.json
after every size (DIR defaults to a directory under the system's temporary directory).
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from paths_profile import device_activities, gpu_info, kernel_name  # noqa: E402

AGENTS = {"M2": 20_700, "L": 215_000}


def kernel_table(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out: dict[str, float] = {}
    for e in device_activities(prof):
        k = kernel_name(e)
        out[k] = out.get(k, 0.0) + e["dur"] / 1000.0
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def profile_size(size: str, reps: int) -> dict:
    import torch

    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report, semantic_clusters_view
    from agent_bom_b200.graph import clusters as cl

    t0 = time.perf_counter()
    est = estate.generate(AGENTS[size], 2145, estate.BENCH_KNOBS, exact_rank=False)
    g = build_unified_graph_from_report(est.report_json(), columnar=True)
    rec = {"agents": AGENTS[size], "nodes": len(g.nodes), "edges": len(g.edges), "build_graph_s": round(time.perf_counter() - t0, 3)}
    t0 = time.perf_counter()
    dg = g.device_graph
    torch.cuda.synchronize()
    rec["upload_s"] = round(time.perf_counter() - t0, 3)
    t0 = time.perf_counter()
    table = cl.cluster_table(g)
    rec["key_table_s"] = round(time.perf_counter() - t0, 3)
    rec["clusters"] = table.n_clusters
    args = (table.n_clusters, table.codes, table.level, table.risk, table.etype)
    dg.build_clusters(*args)                        # warm: module load, cub algorithm selection
    t0 = time.perf_counter()
    s = dg.build_clusters(*args)
    rec["device_build_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    rec["device_build_kernels_ms"] = kernel_table(lambda: dg.build_clusters(*args))
    rec["rel_pairs"] = int(s["rel_nnz"].sum())
    rec["largest_cluster"] = int(s["count"].max()) if len(s["count"]) else 0
    t0 = time.perf_counter()
    body = semantic_clusters_view(g)                # first view: device tables + ranking order
    rec["first_view_s"] = round(time.perf_counter() - t0, 3)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        body = semantic_clusters_view(g)
        ts.append(time.perf_counter() - t0)
    sel_members = sum(c["count"] for c in body["clusters"])
    sel_pairs = sum(len(c["relationship_counts"]) for c in body["clusters"])
    rec["warm_view_s"] = {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "reps": reps}
    rec["view"] = {"clusters": len(body["clusters"]), "member_ids": sel_members, "fetch_d2h_bytes": sel_members * 4 + sel_pairs * 9}
    rec["view_fetch_kernels_ms"] = kernel_table(lambda: semantic_clusters_view(g))
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "abb_clusters_profile"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="M2,L")
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    rec = {**gpu_info(), "sizes": {}}
    for size in args.sizes.split(","):
        rec["sizes"][size] = profile_size(size, args.reps)
        print(json.dumps({size: rec["sizes"][size]}), flush=True)
        (out / "clusters_profile.json").write_text(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
