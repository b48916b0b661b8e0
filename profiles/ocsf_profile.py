#!/usr/bin/env python3
"""Cost of the OCSF export's graph context on the device, and of the host event assembly around it.

    python profiles/ocsf_profile.py [--out DIR] [--reps 7] [--skip-l]

Per estate (M2: 20.7 K agents, L: 215 K agents; bench knobs, every finding one query):
  - ``DeviceGraph.finding_context`` wall time: the median of --reps synchronous calls after two warm-up calls;
  - the impact walk's kernel time and the context kernels' time as the call reports them (CUDA events; the context kernels run on
    a second stream next to the walk);
  - bytes copied device-to-host by the call against ``impact_many`` for the same findings.
M2 only: the host side of ``UnifiedGraph.iter_ocsf_events`` (enriched) on the labelled graph (``Estate.report_json()`` through
the columnar builder): events per second end to end, and the share spent inside ``finding_context``.
Writes DIR/ocsf_profile.json and .md (DIR defaults to a directory under the system's temporary directory).
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from paths_profile import gpu_info  # noqa: E402

AGENTS = {"M2": 20_700, "L": 215_000}


def device_case(label: str, reps: int) -> dict:
    from agent_bom_b200 import estate
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    est = estate.generate(AGENTS[label], 2145, estate.BENCH_KNOBS, exact_rank=False)
    host = csrmod.from_arrays(None, est.node_type, est.src, est.dst, est.rel, est.flags, node_rank=est.node_rank)
    dg = DeviceGraph.upload(host)
    f = np.ascontiguousarray(est.findings, dtype=np.int32)
    for _ in range(2):
        ctx = dg.finding_context(f)
    ts, walk_ms, ctx_ms = [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ctx = dg.finding_context(f)
        ts.append(time.perf_counter() - t0)
        walk_ms.append(ctx.kernel_ms)
        ctx_ms.append(ctx.context_ms)
    imp = dg.impact_many(f)
    imp = dg.impact_many(f)
    rec = {"estate": label, "agents": AGENTS[label], "nodes": int(host.n_nodes), "entries": int(host.n_entries), "findings": int(f.size),
           "finding_context_median_ms": round(statistics.median(ts) * 1e3, 2), "walk_kernel_ms_median": round(statistics.median(walk_ms), 2),
           "context_kernel_ms_median": round(statistics.median(ctx_ms), 3), "sources": int(ctx.source_nodes.size),
           "d2h_bytes_finding_context": int(ctx.d2h_bytes), "d2h_bytes_impact_many": int(imp.d2h_bytes),
           "blast_radius_mean": round(float(ctx.count.mean()), 2), "blast_radius_max": int(ctx.count.max()), "reps": reps}
    if label == "M2":
        rec["host_assembly"] = host_assembly(est)
    dg.close()
    return rec


def host_assembly(est) -> dict:
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import build_unified_graph_from_report

    t0 = time.perf_counter()
    g = build_unified_graph_from_report(est.report_json(), columnar=True)
    build_s = time.perf_counter() - t0
    list(g.iter_ocsf_events())                      # upload + warm-up
    spent = [0.0]
    inner = DeviceGraph.finding_context

    def timed(self, *a, **kw):
        t = time.perf_counter()
        try:
            return inner(self, *a, **kw)
        finally:
            spent[0] += time.perf_counter() - t

    DeviceGraph.finding_context = timed
    try:
        t0 = time.perf_counter()
        n = sum(1 for _ in g.iter_ocsf_events())
        total_s = time.perf_counter() - t0
    finally:
        DeviceGraph.finding_context = inner
    return {"columnar_build_s": round(build_s, 2), "events": n, "iter_ocsf_events_s": round(total_s, 3), "events_per_s": round(n / total_s),
            "finding_context_s": round(spent[0], 4), "host_share": round(1 - spent[0] / total_s, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "abb_ocsf_profile"))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--skip-l", action="store_true")
    a = ap.parse_args()
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    rec = {"device": gpu_info(), "cases": []}
    for label in ("M2",) if a.skip_l else ("M2", "L"):
        rec["cases"].append(device_case(label, a.reps))
        print(json.dumps(rec["cases"][-1]), flush=True)
    (out / "ocsf_profile.json").write_text(json.dumps(rec, indent=1) + "\n")
    dev = rec["device"]
    lines = [f"# OCSF graph context on {dev.get('gpu')} ({dev.get('power_limit_w')} W power limit)", "",
             "| estate | findings | finding_context (median) | walk kernels | context kernels | d2h finding_context | d2h impact_many |",
             "|---|---:|---:|---:|---:|---:|---:|"]
    for c in rec["cases"]:
        lines.append(f"| {c['estate']} | {c['findings']:,} | {c['finding_context_median_ms']} ms | {c['walk_kernel_ms_median']} ms | "
                     f"{c['context_kernel_ms_median']} ms | {c['d2h_bytes_finding_context']:,} B | {c['d2h_bytes_impact_many']:,} B |")
    for c in rec["cases"]:
        if "host_assembly" in c:
            h = c["host_assembly"]
            lines += ["", f"Host assembly at {c['estate']} (`iter_ocsf_events`, enriched, columnar graph): {h['events']:,} events in {h['iter_ocsf_events_s']} s "
                          f"({h['events_per_s']:,} events/s); {h['finding_context_s']} s of it inside `finding_context`, so {h['host_share'] * 100:.1f} % is "
                          "building Python dicts on the host."]
    (out / "ocsf_profile.md").write_text("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
