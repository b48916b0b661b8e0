#!/usr/bin/env python3
"""Generate tests/golden/clusters/*.json.gz with the UNMODIFIED reference's semantic clusters and its clusters route.

Per graph the fixture holds the node and edge records (when the tests cannot rebuild the graph themselves), per node the
reference's ``_cluster_keys_for_node``, ``_node_risk_100`` and ``_node_severity``, ``build_semantic_clusters`` for
``min_members`` 1, 2 and 3 with their ``semantic_cluster_stats``, and the bodies of ``get_graph_clusters``
(api/routes/graph.py:1485-1528), awaited with a stub request and a store that returns the graph, for several
``(kinds, min_members, limit)``.

    python oracle/make_clusters_golden.py            # writes the fixtures
    python oracle/make_clusters_golden.py --time     # instead times build_semantic_clusters on generator estates (profiles/)

Graphs: the 150-agent and dense 40-agent estates of oracle/make_golden.py, a light-builder graph (this package's builder on
``agent_bom_b200.estate``'s 40-agent report, records wrapped with empty dimensions; the tests rebuild it), and ``kat_clusters``.
"""

from __future__ import annotations

import asyncio
import gzip
import json
import sys
import time
from pathlib import Path
from types import SimpleNamespace

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import OUT, REF, estate  # noqa: E402

import agent_bom.api.routes.graph as route  # noqa: E402
from agent_bom.graph import EntityType, RelationshipType, UnifiedEdge, UnifiedGraph, UnifiedNode  # noqa: E402
from agent_bom.graph.node import NodeDimensions  # noqa: E402
from agent_bom.graph.semantic_clusters import (  # noqa: E402
    _cluster_keys_for_node,
    _node_risk_100,
    _node_severity,
    build_semantic_clusters,
    semantic_cluster_stats,
)

from agent_bom_b200.graph.schema import enum_value  # noqa: E402

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
from clusters_golden import decode  # noqa: E402

LIGHT_AGENTS = 40
E, R = EntityType, RelationshipType


def kat_clusters() -> UnifiedGraph:
    """Key-rule and roll-up edge cases (see the module docstring of tests/test_clusters.py)."""
    g = UnifiedGraph(scan_id="kat-clusters", tenant_id="default", created_at="2026-05-01T00:00:00+00:00")
    D = NodeDimensions

    def n(nid, et, label=None, *, sev="", risk=0.0, attrs=None, ds=None, dims=None):
        g.add_node(UnifiedNode(id=nid, entity_type=et, label=nid if label is None else label, severity=sev, risk_score=risk,
                               attributes=attrs or {}, data_sources=ds or [], dimensions=dims or D()))

    # packages: name@version, scoped, empty label, name attributes, ecosystem from dims / attrs / unknown, pkg: prefix
    n("pkg:a1", E.PACKAGE, "lodash@4.17.0", ds=["sbom"], attrs={"ecosystem": "npm"})
    n("pkg:a2", E.PACKAGE, "lodash@4.18.0", ds=["sbom", "scan"], dims=D(ecosystem="npm"))
    n("pkg:scoped", E.PACKAGE, "@scope/pkg@1.0", ds=["sbom"], dims=D(ecosystem="npm"))
    n("pkg:scoped2", E.PACKAGE, "@scope/pkg@1.0", ds=["sbom"], attrs={"package_ecosystem": "npm"})
    n("pkg:empty", E.PACKAGE, "", ds=[""], attrs={"ecosystem": "  "})
    n("pkg:named", E.PACKAGE, "ignored", attrs={"name": " requests ", "package_ecosystem": "pypi", "source": "attr-src"})
    n("pkg:named2", E.PACKAGE, "x", attrs={"package_name": "requests", "ecosystem": "pypi", "provider": "attr-src"})
    n("pkg:pref", E.PACKAGE, "pkg:left-pad", attrs={"package": "", "environment": "prod"}, risk=8.99995)
    n("pkg:pref2", E.PACKAGE, "left-pad@1", attrs={"env": "prod"}, risk=89.9996)
    # vulnerabilities: CVE in id / label / attribute only, lower case, CWE only, neither
    n("CVE-2024-0001", E.VULNERABILITY, "x", sev="CRITICAL", ds=["scan"])
    n("vuln:label", E.VULNERABILITY, "see CVE-2024-7777 advisory", sev="info", risk=10.0, ds=["scan"])
    n("vuln:attr", E.VULNERABILITY, "advisory", attrs={"ref": "cve-2023-1111-x", "n": 5}, risk=10.5, ds=["scan"])
    n("vuln:lower", E.VULNERABILITY, "cve-2023-0002-", sev="High", risk=150, ds=["scan"])
    n("vuln:cwe", E.VULNERABILITY, "CWE-79 xss", risk=-3.0, sev="medium", ds=["scan"])
    n("vuln:none", E.VULNERABILITY, "", risk=-1.0, ds=["scan"])
    n("vuln:round", E.VULNERABILITY, "plain", risk=6.99995, ds=["scan"])
    n("vuln:round2", E.VULNERABILITY, "plain2", risk=3.99996, ds=["scan"])
    n("vuln:thresh", E.VULNERABILITY, "plain3", risk=0.1, ds=["scan"])
    n("vuln:thresh2", E.VULNERABILITY, "plain4", risk=0.0999, ds=["scan"])
    n("vuln:unknown-sev", E.VULNERABILITY, "plain5", sev="unknown", ds=["scan"])
    # agents / servers: dims, environment, source, attribute fleets, defaults
    n("agent:1", E.AGENT, "a1", dims=D(agent_type="claude", environment="prod"), ds=["mcp"])
    n("agent:2", E.AGENT, "a2", attrs={"fleet": "ops"})
    n("agent:3", E.AGENT, "a3")
    n("agent:4", E.AGENT, "a4", attrs={"workspace": "ws1"}, ds=[])
    n("agent:5", E.AGENT, "a5", attrs={"account": "123", "agent_type": "bot", "kind": "k"})
    n("server:1", E.SERVER, "s1", dims=D(surface="stdio"), ds=["mcp"])
    n("server:2", E.SERVER, "s2", attrs={"server_type": "http"})
    n("server:3", E.SERVER, "s3", attrs={"kind": "remote", "source": "inventory"})
    n("server:4", E.SERVER, "s4")
    # credentials: provider attributes and label tokens
    n("cred:1", E.CREDENTIAL, "AWS_SECRET", ds=["env"])
    n("cred:2", E.CREDENTIAL, "openai_api_key", ds=["env"])
    n("cred:3", E.CREDENTIAL, "token", attrs={"cloud_provider": "gcp"}, ds=["env"])
    n("cred:4", E.CREDENTIAL, "", attrs={"service": "vault"})
    n("cred:github-pat", E.CREDENTIAL, "", ds=["env"])
    n("cred:5", E.CREDENTIAL, "x", attrs={"provider": "  "}, sev="low")
    # tools: label words and explicit capability attributes
    n("tool:1", E.TOOL, "run_shell", ds=["mcp"])
    n("tool:2", E.TOOL, "read_file", ds=["mcp"])
    n("tool:3", E.TOOL, "http_fetch", ds=["mcp"])
    n("tool:4", E.TOOL, "noop", ds=["mcp"])
    n("tool:5", E.TOOL, "x", attrs={"capability": "admin"}, ds=["mcp"])
    n("tool:6", E.TOOL, "", attrs={"category": "admin", "tool_type": "z"})
    # a label tie between two keys: env "a" with source "" and env "a" with source "a" both read "a"
    n("model:1", E.MODEL, "m1", dims=D(environment="a"))
    n("model:2", E.MODEL, "m2", dims=D(environment="a"), ds=["a"])
    n("model:3", E.MODEL, "m3", attrs={"environment": "a"})
    n("model:4", E.MODEL, "m4", ds=["a"])
    n("dataset:1", E.DATASET, "d1", sev="none", risk=100.0)
    edges = [
        ("agent:1", "server:1", R.USES), ("agent:2", "server:1", R.USES), ("agent:3", "server:2", R.USES), ("agent:4", "server:3", R.USES),
        ("server:1", "pkg:a1", R.DEPENDS_ON), ("server:1", "pkg:a2", R.DEPENDS_ON), ("server:2", "pkg:scoped", R.DEPENDS_ON),
        ("server:2", "pkg:named", R.DEPENDS_ON), ("server:3", "pkg:named2", R.DEPENDS_ON), ("server:4", "pkg:pref", R.DEPENDS_ON),
        ("pkg:a1", "CVE-2024-0001", R.VULNERABLE_TO), ("pkg:a2", "vuln:label", R.VULNERABLE_TO), ("pkg:scoped", "vuln:attr", R.VULNERABLE_TO),
        ("pkg:pref", "vuln:lower", R.VULNERABLE_TO), ("pkg:pref2", "vuln:cwe", R.VULNERABLE_TO), ("pkg:empty", "vuln:none", R.VULNERABLE_TO),
        ("server:1", "cred:1", R.EXPOSES_CRED), ("server:1", "cred:2", R.EXPOSES_CRED), ("server:2", "cred:3", R.EXPOSES_CRED),
        ("server:1", "tool:1", R.PROVIDES_TOOL), ("server:1", "tool:2", R.PROVIDES_TOOL), ("server:2", "tool:3", R.PROVIDES_TOOL),
        ("server:3", "tool:5", R.PROVIDES_TOOL), ("server:4", "tool:6", R.PROVIDES_TOOL),
        ("pkg:a1", "pkg:a2", R.DEPENDS_ON),                                  # intra-cluster edge
        ("agent:1", "agent:2", R.SHARES_SERVER, "bidirectional"), ("cred:1", "cred:2", R.SHARES_CRED, "bidirectional"),
        ("agent:5", "agent:5", R.TRUSTS),                                    # self loop
        ("ghost:x", "pkg:a1", R.DEPENDS_ON), ("server:1", "ghost:y", R.HOSTS), ("ghost:x", "ghost:y", R.USES),
        ("model:1", "model:2", "custom_link"), ("model:2", "dataset:1", "custom_link"), ("model:3", "ghost:z", "another_link"),
        ("model:4", "model:1", R.SERVES_MODEL, "directed", False),
    ]
    for e in edges:
        g.add_edge(UnifiedEdge(source=e[0], target=e[1], relationship=e[2], direction=e[3] if len(e) > 3 else "directed",
                               traversable=e[4] if len(e) > 4 else True))
    return g


def light_graph():
    """This package's light builder on the estate generator's report.  Its records carry no dimensions and this package's enum members,
    so they are wrapped with empty dimensions and plain string values (the reference's ``str()`` of a foreign enum is its name)."""
    from agent_bom_b200 import estate as est_mod
    from agent_bom_b200.graph import build_unified_graph_from_report

    g = build_unified_graph_from_report(est_mod.generate(LIGHT_AGENTS, 2145, est_mod.BENCH_KNOBS).report_json())
    nodes = {nid: SimpleNamespace(id=n.id, entity_type=enum_value(n.entity_type), label=n.label, severity=n.severity, risk_score=n.risk_score,
                                  attributes=n.attributes, data_sources=n.data_sources, dimensions=NodeDimensions())
             for nid, n in g.nodes.items()}
    edges = [SimpleNamespace(source=e.source, target=e.target, relationship=enum_value(e.relationship)) for e in g.edges]
    return SimpleNamespace(nodes=nodes, edges=edges, scan_id="light-scan", tenant_id="default", created_at="2026-05-01T00:00:00+00:00")


class Store:
    def __init__(self, graph):
        self.graph = graph

    def latest_snapshot_id(self, *, tenant_id=""):
        return self.graph.scan_id or "latest"

    def load_graph(self, *, scan_id="", tenant_id="", **_kw):
        return self.graph


def reference_view(graph, **params):
    route._get_graph_store = lambda: Store(graph)
    request = SimpleNamespace(state=SimpleNamespace(tenant_id=graph.tenant_id or "default"))
    return asyncio.run(route.get_graph_clusters(request, scan_id=graph.scan_id or None, **params))


def node_rec(n):
    dims = getattr(n, "dimensions", None)
    return {"id": n.id, "entity_type": enum_value(n.entity_type), "label": n.label, "severity": n.severity, "risk_score": n.risk_score,
            "attributes": dict(n.attributes), "data_sources": list(n.data_sources), "dimensions": None if dims is None else dims.to_dict()}


def edge_rec(e):
    return {"source": e.source, "target": e.target, "relationship": enum_value(e.relationship), "direction": e.direction, "traversable": bool(e.traversable)}


def encode(case: dict, node_ids: list[str]) -> dict:
    """The fixture's compact form, which ``tests/clusters_golden.decode`` expands back to ``case`` exactly (checked on write):
    node ids once, member ids and edge endpoints as indices into them, the distinct cluster keys once, each cluster dict once
    (the ``min_members=1`` list, without its ``expansion``, which the reference derives from ``member_ids`` and ``id``), and every
    other cluster list and route body as positions in that list."""
    index = {nid: i for i, nid in enumerate(node_ids)}
    ghosts: dict[str, int] = {}

    def endpoint(nid):
        i = index.get(nid)
        return i if i is not None else len(node_ids) + ghosts.setdefault(nid, len(ghosts))

    def pack_cluster(d):
        assert d["expansion"] == {"mode": "members", "member_ids": d["member_ids"], "collapse_id": d["id"], "reversible": True}
        return {k: ([index[m] for m in v] if k == "member_ids" else v) for k, v in d.items() if k != "expansion"}

    base = case["clusters"]["1"]["clusters"]
    pos: dict[str, int] = {}
    for i, c in enumerate(base):
        pos.setdefault(json.dumps(c, sort_keys=True), i)

    def positions(clusters):
        return [pos[json.dumps(c, sort_keys=True)] for c in clusters]

    key_table: dict[tuple, int] = {}
    out = {k: case[k] for k in ("name", "scan_id", "tenant_id", "created_at", "risk", "severity")}
    out["node_ids"] = node_ids
    out["keys"] = [[key_table.setdefault(tuple(k), len(key_table)) for k in ks] for ks in case["keys"]]
    out["key_table"] = [list(k) for k in key_table]
    out["cluster_list"] = [pack_cluster(c) for c in base]
    out["clusters"] = {m: {"index": positions(v["clusters"]), "stats": v["stats"]} for m, v in case["clusters"].items()}
    out["views"] = [{"params": v["params"], "body": {**{k: x for k, x in v["body"].items() if k != "clusters"}, "clusters": positions(v["body"]["clusters"])}}
                    for v in case["views"]]
    if "nodes" in case:
        out["nodes"] = [{k: x for k, x in n.items() if k != "id"} for n in case["nodes"]]
        assert [n["id"] for n in case["nodes"]] == node_ids
        out["edges"] = [[endpoint(e["source"]), endpoint(e["target"]), e["relationship"], e["direction"] == "bidirectional", e["traversable"]]
                        for e in case["edges"]]
        assert all(e["direction"] in ("directed", "bidirectional") for e in case["edges"])
        out["ghost_ids"] = list(ghosts)
    return out


VIEW_CASES = [
    {}, {"min_members": 1}, {"min_members": 3, "limit": 5}, {"limit": 1}, {"kinds": "package_family"},
    {"kinds": " cve_family , agent_fleet ,", "min_members": 1}, {"kinds": "source_environment,server_fleet", "limit": 2},
    {"kinds": "tool_capability,credential_family", "min_members": 1, "limit": 1000}, {"min_members": 100}, {"kinds": " , "},
]


def graph_case(name, g, *, with_graph=True):
    nodes = list(g.nodes.values())
    case = {"name": name, "scan_id": g.scan_id, "tenant_id": g.tenant_id, "created_at": g.created_at,
            "keys": [[list(k) for k in _cluster_keys_for_node(n)] for n in nodes],
            "risk": [_node_risk_100(n) for n in nodes], "severity": [_node_severity(n) for n in nodes], "clusters": {}, "views": []}
    for m in (1, 2, 3):
        clusters = build_semantic_clusters(g.nodes.values(), g.edges, min_members=m)
        case["clusters"][str(m)] = {"clusters": [c.to_dict() for c in clusters], "stats": semantic_cluster_stats(clusters)}
    for params in VIEW_CASES:
        full = {"kinds": params.get("kinds"), "min_members": params.get("min_members", 2), "limit": params.get("limit", 250)}
        case["views"].append({"params": full, "body": reference_view(g, **full)})
    if with_graph:
        case["nodes"] = [node_rec(n) for n in nodes]
        case["edges"] = [edge_rec(e) for e in g.edges]
    print(f"clusters {name}: {len(nodes)} nodes, {len(g.edges)} edges, {len(case['clusters']['2']['clusters'])} clusters (min 2)")
    return case


def golden():
    out = OUT / "clusters"
    out.mkdir(parents=True, exist_ok=True)
    graphs = [("kat_clusters", kat_clusters(), True), ("light_40", light_graph(), False), ("estate_dense_40", estate(40, dense=(6, 8, 3)), True),
              ("estate_150", estate(150), True)]
    for name, g, with_graph in graphs:
        if not g.scan_id or name.startswith("estate"):
            g.scan_id, g.tenant_id, g.created_at = f"{name}-scan", "default", "2026-05-01T00:00:00+00:00"
        case = graph_case(name, g, with_graph=with_graph)
        packed = encode(case, [n.id for n in g.nodes.values()])
        assert decode(json.loads(json.dumps(packed))) == json.loads(json.dumps(case)), name
        path = out / f"{name}.json.gz"
        with gzip.GzipFile(path, "wb", mtime=0) as fh:
            fh.write(json.dumps(packed, sort_keys=True, separators=(",", ":")).encode())
        print(f"-> {path} {path.stat().st_size / 1024:.0f} KiB")


def time_reference(agent_counts=(40, 150, 600)):
    """One-core wall time of the unmodified builder and build_semantic_clusters on estate-generator estates (BENCH_KNOBS, seed 2145)."""
    import platform

    from agent_bom.graph import build_unified_graph_from_report as ref_build

    from agent_bom_b200 import estate as est_mod

    rec = {"host": {"machine": platform.machine(), "python": platform.python_version(), "processor": platform.processor()}, "estates": []}
    for agents in agent_counts:
        report = est_mod.generate(agents, 2145, est_mod.BENCH_KNOBS).report_json()
        g = ref_build(report)
        t0 = time.perf_counter()
        clusters = build_semantic_clusters(g.nodes.values(), g.edges, min_members=2)
        dt = time.perf_counter() - t0
        rec["estates"].append({"agents": agents, "nodes": len(g.nodes), "edges": len(g.edges), "clusters": len(clusters), "build_semantic_clusters_s": round(dt, 3)})
        print(json.dumps(rec["estates"][-1]))
    dst = Path(__file__).resolve().parents[1] / "profiles" / "clusters_reference.json"
    dst.write_text(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    assert REF.exists()
    if "--time" in sys.argv:
        time_reference()
    else:
        golden()
