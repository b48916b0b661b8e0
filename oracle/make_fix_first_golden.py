#!/usr/bin/env python3
"""Generate tests/golden/fix_first/views.json.gz with the UNMODIFIED reference's fix-first route.

Runs only where the reference tree is importable (the GPU tests read the fixture alone).  The reference's own
``get_fix_first_graph_view`` coroutine (api/routes/graph.py:1110-1166) is awaited with a stub request and a store that returns
the graph, so the whole response is pinned: cards, ``summary`` and ``focus``.  Per graph the fixture also holds every derived
(or persisted) path and, per focus, the reference predicate's verdict on each of them (``_path_matches_focus``, :448-476).

    python oracle/make_fix_first_golden.py            # writes the fixture
    python oracle/make_fix_first_golden.py --time     # instead times the reference route on a small estate (profiles/)

Kept apart from oracle/make_golden.py so the fixtures that script writes are untouched; graph builders are shared with it.
"""

from __future__ import annotations

import asyncio
import gzip
import json
import sqlite3
import sys
import tempfile
import time
from collections import Counter
from pathlib import Path
from types import SimpleNamespace

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import AG, MIS, OUT, PKG, REF, SRV, VULN, CRED, TOOL, R, estate, kat_derived, kat_probe, mesh_inventory, mk  # noqa: E402

import agent_bom.api.routes.graph as route  # noqa: E402
from agent_bom.api.routes.graph import _derived_attack_paths, _path_matches_focus  # noqa: E402
from agent_bom.graph import AttackPath, EntityType  # noqa: E402

from agent_bom_b200.graph.schema import enum_value  # noqa: E402

AGENT_TYPES = {"agent", "user", "group", "service_account"}
NOTHING = "CVE-0000-MATCHES-NOTHING"


def kat_focus():
    """Focus edge cases: empty / padded / mixed-case labels, user, group and service-account principals, a package and a
    vulnerability sharing a label, misconfigurations, a server no principal uses, ghost endpoints."""
    E = EntityType
    return mk(
        [("agent:mixed", AG, "", 0, "  Agent-Mixed "), ("user:u", E.USER, "", 0, "Dana.User"), ("sa:ci", E.SERVICE_ACCOUNT, "", 0, "ci-bot"),
         ("group:ops", E.GROUP, "", 0, "Ops-Team"), ("agent:blank", AG, "", 0, "   "), ("agent:nolabel", AG, "", 0, ""),
         ("server:a", SRV, "", 0, "Srv-A"), ("server:b", SRV, "", 0, " srv-b"), ("server:lonely", SRV, "", 0, "Lonely"),
         ("pkg:shared", PKG, "", 0, "shared-name"), ("pkg:nolabel", PKG, "", 0, ""), ("pkg:left", PKG, "", 0, "Left-Pad "),
         ("vuln:shared", VULN, "high", 0.0, "Shared-Name"), ("CVE-2031-EMPTY", VULN, "critical", 0.0, ""), ("vuln:padded", VULN, "medium", 6.5, "  CVE-2031-0002  "),
         ("vuln:idonly", VULN, "low", 0.0, "Named-Finding"), ("mis:open-port", MIS, "high", 0.0, "Open-Port"), ("mis:blank", MIS, "low", 0.0, ""),
         ("cred:K", CRED, "", 0, "API_KEY"), ("tool:sh", TOOL, "", 0, "run_shell"), ("tool:r", TOOL, "", 0, "read")],
        [("agent:mixed", "server:a", R.USES), ("user:u", "server:a", R.USES), ("sa:ci", "server:b", R.USES), ("agent:blank", "server:b", R.USES),
         ("agent:nolabel", "server:a", R.USES), ("group:ops", "server:a", R.USES),
         ("server:a", "pkg:shared", R.DEPENDS_ON), ("server:a", "pkg:nolabel", R.DEPENDS_ON), ("server:b", "pkg:left", R.DEPENDS_ON),
         ("server:b", "group:ops", R.DEPENDS_ON), ("server:lonely", "pkg:left", R.DEPENDS_ON),
         ("pkg:shared", "vuln:shared", R.VULNERABLE_TO), ("pkg:nolabel", "CVE-2031-EMPTY", R.VULNERABLE_TO), ("pkg:left", "vuln:padded", R.VULNERABLE_TO),
         ("pkg:left", "CVE-2031-EMPTY", R.VULNERABLE_TO), ("group:ops", "vuln:idonly", R.VULNERABLE_TO), ("server:lonely", "mis:open-port", R.VULNERABLE_TO),
         ("server:a", "mis:blank", R.VULNERABLE_TO), ("server:b", "mis:open-port", R.VULNERABLE_TO),
         ("server:a", "cred:K", R.EXPOSES_CRED), ("server:a", "tool:sh", R.PROVIDES_TOOL), ("server:b", "tool:r", R.PROVIDES_TOOL),
         ("ghost:pkg", "vuln:shared", R.VULNERABLE_TO), ("server:a", "ghost:cred", R.EXPOSES_CRED), ("ghost:agent", "server:b", R.USES)],
    )


class Store:
    def __init__(self, graph):
        self.graph = graph

    def latest_snapshot_id(self, *, tenant_id=""):
        return self.graph.scan_id or "latest"

    def load_graph(self, *, scan_id="", tenant_id="", **_kw):
        return self.graph


def reference_view(graph, **focus):
    route._get_graph_store = lambda: Store(graph)
    request = SimpleNamespace(state=SimpleNamespace(tenant_id=graph.tenant_id or "default"))
    return asyncio.run(route.get_fix_first_graph_view(request, scan_id=graph.scan_id or None, **focus))


def labels_on_paths(g, paths, types):
    """How many paths carry each `label or id` of a hop with one of the types (hops without a record are skipped)."""
    count = Counter()
    for p in paths:
        seen = set()
        for h in p.hops:
            n = g.nodes.get(h)
            if n is not None and enum_value(n.entity_type) in types:
                seen.add(n.label or n.id)
        count.update(seen)
    return count


def heavy_and_rare(count: Counter) -> tuple[str, str]:
    usable = sorted((k for k in count if k.strip()), key=lambda k: (-count[k], k))
    if not usable:
        return "", ""
    return usable[0], usable[-1]


def focus_cases(g, paths):
    cves = labels_on_paths(g, paths, {"vulnerability", "misconfiguration"})
    for p in paths:
        cves.update({v for v in p.vuln_ids if v.strip()})
    cve_h, cve_r = heavy_and_rare(cves)
    pkg_h, pkg_r = heavy_and_rare(labels_on_paths(g, paths, {"package"}))
    ag_h, ag_r = heavy_and_rare(labels_on_paths(g, paths, AGENT_TYPES))
    # the pairs and the triple come from one path so they match something
    combo = {"cve": cve_h, "package": pkg_h, "agent": ag_h}
    for p in paths[len(paths) // 3:] + paths[: len(paths) // 3]:
        pk = [g.nodes[h].label or h for h in p.hops if h in g.nodes and enum_value(g.nodes[h].entity_type) == "package"]
        ag = [g.nodes[h].label or h for h in p.hops if h in g.nodes and enum_value(g.nodes[h].entity_type) in AGENT_TYPES]
        if pk and ag and p.vuln_ids and p.vuln_ids[0].strip():
            combo = {"cve": p.vuln_ids[0], "package": pk[0], "agent": ag[0]}
            break
    cases = [{}, {"limit": 1}, {"limit": 25}]
    for key, (h, r) in (("cve", (cve_h, cve_r)), ("package", (pkg_h, pkg_r)), ("agent", (ag_h, ag_r))):
        if h:
            cases += [{key: h}, {key: r}, {key: h, "limit": 25}, {key: f"  {h.upper()}\t"}, {key: f" {r.swapcase()} "}]
    for a, b in (("cve", "package"), ("cve", "agent"), ("package", "agent")):
        if combo[a] and combo[b]:
            cases.append({a: combo[a], b: combo[b]})
            cases.append({a: combo[a], b: combo[b], "limit": 1})
    if all(combo.values()):
        cases.append(dict(combo))
        cases.append({k: f" {v.upper()} " for k, v in combo.items()} | {"limit": 25})
    if pkg_h and ag_r:
        cases.append({"package": pkg_h, "agent": ag_r})
    cases += [{"cve": NOTHING}, {"package": NOTHING, "agent": ag_h}]
    out, seen = [], set()
    for c in cases:
        full = {"cve": c.get("cve", ""), "package": c.get("package", ""), "agent": c.get("agent", ""), "limit": c.get("limit", 8)}
        key = tuple(full.values())
        if key not in seen:
            seen.add(key)
            out.append(full)
    return out


def node_rec(n):
    return {"id": n.id, "entity_type": enum_value(n.entity_type), "label": n.label, "severity": n.severity, "risk_score": n.risk_score,
            "attributes": dict(n.attributes), "to_dict": n.to_dict()}


def edge_rec(e):
    return {"source": e.source, "target": e.target, "relationship": enum_value(e.relationship), "direction": e.direction, "traversable": bool(e.traversable)}


def ap(p):
    d = p.to_dict()
    d["edges"] = [enum_value(x) for x in d["edges"]]
    return d


def graph_case(name, g, *, with_graph=True, tenant=""):
    paths = _derived_attack_paths(g)          # persisted paths when present, else the derived ones in ranking order
    focuses = focus_cases(g, paths)
    views, verdicts = [], []
    for f in focuses:
        focus = {k: f[k] for k in ("cve", "package", "agent")}
        views.append({"focus": f, "view": reference_view(g, **focus, limit=f["limit"])})
        if f["limit"] == 8:
            verdicts.append({"focus": focus, "match": "".join("1" if _path_matches_focus(g, p, **focus) else "0" for p in paths)})
    case = {"name": name, "scan_id": g.scan_id, "tenant_id": g.tenant_id, "created_at": g.created_at, "views": views, "verdicts": verdicts,
            "paths": [ap(p) for p in paths], "persisted": bool(g.attack_paths)}
    if with_graph:
        case |= {"nodes": [node_rec(n) for n in g.nodes.values()], "edges": [edge_rec(e) for e in g.edges],
                 "attack_paths": [ap(p) for p in g.attack_paths]}
    else:
        case["tenant"] = tenant
    print(f"fix_first {name}: {len(g.nodes)} nodes, {len(g.edges)} edges, {len(paths)} paths, {len(views)} views, "
          f"matched {[v['view']['summary']['matched_paths'] for v in views]}")
    return case


def snapshot_cases():
    """Views of snapshots in the SQLite file tests/golden/snapshot/graph.sqlite.gz (written by the reference's save_graph)."""
    from agent_bom.db import graph_store as ref_db

    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    tmp.write_bytes(gzip.decompress((OUT / "snapshot" / "graph.sqlite.gz").read_bytes()))
    conn = sqlite3.connect(str(tmp))
    conn.row_factory = sqlite3.Row
    out = []
    for tenant, scan in (("default", "scan-a"), ("default", "scan-b"), ("acme", "scan-a")):
        g = ref_db.load_graph(conn, tenant_id=tenant, scan_id=scan)
        out.append(graph_case(f"snapshot_{tenant}_{scan}", g, with_graph=False, tenant=tenant))
    conn.close()
    return out


def golden():
    probe = kat_probe()
    probe.attack_paths = [     # hand-made persisted paths: missing hops, ghost endpoints, padded vuln ids, pairs without an edge
        AttackPath(source="a", target="d", hops=["a", "d"], edges=["shares_cred"], composite_risk=55.0, summary="bidirectional pair", vuln_ids=[" CVE-X ", "CVE-X"]),
        AttackPath(source="", target="", hops=["s", "b", "c"], edges=[], composite_risk=8.5, summary=""),
        AttackPath(source="s", target="nowhere", hops=["s", "nowhere", "c"], edges=["uses"], composite_risk=3.0, tool_exposure=["t1"], credential_exposure=["K"]),
        AttackPath(source="c", target="d", hops=["c", "d"], edges=["depends_on", "extra"], composite_risk=95.0),
        AttackPath(source="z", target="d", hops=["z", "s", "b", "c", "d"], edges=[], composite_risk=55.0, vuln_ids=["d"], tool_exposure=["exec-tool"]),
    ]
    graphs = [("kat_derived", kat_derived()), ("kat_probe", probe), ("estate_dense", estate(12, dense=(4, 6, 2))), ("mesh", mesh_inventory()),
              ("kat_focus", kat_focus())]
    cases = []
    for name, g in graphs:
        g.scan_id, g.tenant_id, g.created_at = f"{name}-scan", "default", "2026-05-01T00:00:00+00:00"
        cases.append(graph_case(name, g))
    cases += snapshot_cases()
    out = OUT / "fix_first"
    out.mkdir(parents=True, exist_ok=True)
    with gzip.GzipFile(out / "views.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps({"cases": cases}, sort_keys=True).encode())
    print(f"-> {out / 'views.json.gz'} {(out / 'views.json.gz').stat().st_size / 1024:.0f} KiB")


def time_reference(agents: int = 150, reps: int = 5):
    """Wall time of the reference route body (load_graph is the stub) on a generator estate: unfocused and focused."""
    g = estate(agents)
    paths = _derived_attack_paths(g)
    cve = Counter(p.vuln_ids[0] for p in paths).most_common(1)[0][0]
    rec = {"estate_agents": agents, "nodes": len(g.nodes), "edges": len(g.edges), "paths": len(paths), "cases": {}}
    for label, focus in (("unfocused_top8", {"cve": "", "package": "", "agent": ""}), ("heavy_cve", {"cve": cve, "package": "", "agent": ""})):
        reference_view(g, **focus, limit=8)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            reference_view(g, **focus, limit=8)
            ts.append(time.perf_counter() - t0)
        rec["cases"][label] = {"median_s": sorted(ts)[len(ts) // 2], "reps": reps}
    import platform

    rec["host"] = {"machine": platform.machine(), "python": platform.python_version(), "processor": platform.processor()}
    dst = Path(__file__).resolve().parents[1] / "profiles" / "fix_first_reference_route.json"
    dst.write_text(json.dumps(rec, indent=1) + "\n")
    print(json.dumps(rec))


if __name__ == "__main__":
    assert REF.exists()
    if "--time" in sys.argv:
        time_reference()
    else:
        golden()
