#!/usr/bin/env python3
"""Per-stage times of the context-graph report (``build_context_graph`` + ``context_graph_report``, every agent's paths).

    python profiles/context_report_profile.py [--out DIR] [--agents 1000,4000,16000] [--reps 3]
    python profiles/context_report_profile.py --reference [--out DIR] [--agents 1000]

The fleet (``oracle/context_report_oracle.fleet``): per agent one private and two shared MCP servers, the shared names drawn
so that each is used by about agents / 20 agents, two tools per server (one execute-capable), a credential on 30 % of servers
(``GITHUB_TOKEN`` on all of them, so its clique spans most agents) and agents / 2 critical / high / medium vulnerabilities.
When a size's edge count would exceed ``--max-edges`` (the graph is Python objects) it is recorded as not measured.

Stages: builder loops, device scorer (``effective_reach.annotate_graph``), the per-graph encoding (``lateral._arrays_for``
and its enrichment tables; cached per graph, so a second report on the same graph skips it), the search kernel and the
enrichment kernels (device ms from CUDA events), the host path assembly, interaction risks and serialisation
(``json.dumps`` of the body).  Wall times are best of ``--reps`` reports on one graph, the first (cold) report separately.
The card name and power limit are read in the same run.  Writes DIR/h100_context_report_profile.json.

``--reference`` runs the unmodified reference chain on the CPU (build, ``find_lateral_paths`` per agent, risks,
``to_serializable``) and writes DIR/context_report_reference.json; it is the only mode that imports the reference.
"""

from __future__ import annotations

import argparse
import json
import platform
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle.context_report_oracle import fleet  # noqa: E402


def fleet_for(agents: int):
    return fleet(agents, 2145, clique=max(2, agents // 20), cred_share=1.0)


def expected_edges(agents_data) -> int:
    """Edges the builder will make, counted from the report lists (so an oversized graph is skipped before it is built)."""
    from collections import defaultdict

    srv, cred = defaultdict(set), defaultdict(set)
    n = 0
    for a in agents_data:
        for s in a["mcp_servers"]:
            srv[s["name"]].add(a["name"])
            n += 1 + len(s["tools"]) + sum(1 for k in s["env"] if k != "HOME")
            for k in s["env"]:
                if k != "HOME":
                    cred[k].add(a["name"])
    return n + sum(len(v) * (len(v) - 1) // 2 for v in srv.values()) + sum(len(v) * (len(v) - 1) // 2 for v in cred.values())


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def profile_size(agents: int, reps: int, max_edges: int) -> dict:
    from agent_bom_b200 import context_report as cr
    from agent_bom_b200 import lateral

    agents_data, blast, classify, is_cred = fleet_for(agents)
    want = expected_edges(agents_data)
    if want > max_edges:
        return {"agents": agents, "expected_edges": want, "status": f"not measured: more than {max_edges} edges as Python objects"}
    t = {}
    g = cr.build_context_graph(agents_data, blast, classify_tool=classify, is_credential_key=is_cred, timings=t)
    rec = {"agents": agents, "nodes": len(g.nodes), "edges": len(g.edges), "adjacency_entries": sum(map(len, g.adjacency.values())),
           "builder_loops_s": round(t["build"], 3), "device_scorer_s": round(t["score"], 3)}
    t0 = time.perf_counter()
    arr = lateral._arrays_for(g)
    t1 = time.perf_counter()
    arr.enrichment(g)
    rec["encoding_s"] = {"search_arrays": round(t1 - t0, 3), "enrichment_tables": round(time.perf_counter() - t1, 3)}

    def one():
        tm = {}
        t0 = time.perf_counter()
        body = cr.context_graph_report(g, max_depth=4, timings=tm)
        t1 = time.perf_counter()
        text = json.dumps(body)
        tm["serialise"] = tm["serialise"] + time.perf_counter() - t1
        tm["report_wall"] = time.perf_counter() - t0
        return tm, len(text), body["stats"]

    runs = [one() for _ in range(reps + 1)]
    cold, warm = runs[0], runs[1:]
    stages = ("search", "search_device_ms", "enrich", "enrich_device_ms", "assemble", "risks", "serialise", "report_wall")
    rec["cold_report"] = {k: round(cold[0][k], 4) for k in stages}
    rec["warm_report_best"] = {k: round(min(r[0][k] for r in warm), 4) for k in stages}
    rec["paths"] = cold[0]["paths"]
    rec["body_json_bytes"] = cold[1]
    rec["stats"] = cold[2]
    rec["units"] = "seconds, except *_device_ms (CUDA events around the kernels of one call)"
    return rec


def reference_size(agents: int) -> dict:
    import oracle.make_golden  # noqa: F401  (puts the reference on the path)
    from agent_bom.context_graph import NodeKind, build_context_graph, compute_interaction_risks, find_lateral_paths, to_serializable

    agents_data, blast, _c, _k = fleet_for(agents)
    t0 = time.perf_counter()
    g = build_context_graph(agents_data, blast)
    t1 = time.perf_counter()
    paths = []
    for nid, node in g.nodes.items():
        if node.kind == NodeKind.AGENT:
            paths.extend(find_lateral_paths(g, nid))
    t2 = time.perf_counter()
    risks = compute_interaction_risks(g)
    t3 = time.perf_counter()
    json.dumps(to_serializable(g, paths, risks))
    t4 = time.perf_counter()
    return {"agents": agents, "nodes": len(g.nodes), "edges": len(g.edges), "build_context_graph_s": round(t1 - t0, 2),
            "find_lateral_paths_all_agents_s": round(t2 - t1, 2), "compute_interaction_risks_s": round(t3 - t2, 3),
            "to_serializable_and_json_s": round(t4 - t3, 3), "route_total_s": round(t4 - t0, 2), "paths": len(paths)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles"))
    ap.add_argument("--agents", default="1000,4000,16000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-edges", type=int, default=8_000_000)
    ap.add_argument("--reference", action="store_true")
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    sizes = [int(x) for x in args.agents.split(",")]
    if args.reference:
        doc = {"what": "unmodified reference context-graph chain as the REST route runs it, on the CPU of a build host without a GPU; "
                       "not a like-for-like comparison with the GPU numbers",
               "host": {"machine": platform.machine(), "processor": platform.processor()}, "sizes": {}}
        for n in sizes:
            doc["sizes"][str(n)] = reference_size(n)
            print(n, json.dumps(doc["sizes"][str(n)]), flush=True)
            (out / "context_report_reference.json").write_text(json.dumps(doc, indent=1) + "\n")
        return
    doc = {"card": card(), "fleet": "profiles/context_report_profile.py fleet_for (seed 2145)", "sizes": {}}
    for n in sizes:
        doc["sizes"][str(n)] = profile_size(n, args.reps, args.max_edges)
        print(n, json.dumps(doc["sizes"][str(n)]), flush=True)
        (out / "h100_context_report_profile.json").write_text(json.dumps(doc, indent=1) + "\n")


if __name__ == "__main__":
    main()
