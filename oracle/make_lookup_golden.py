#!/usr/bin/env python3
"""Generate tests/golden/lookup/ with the UNMODIFIED reference SQLite store's record lookups.

Graphs are saved with the reference's ``save_graph`` into one SQLite file, and the reference ``SQLiteGraphStore`` answers
``nodes_by_ids``, ``edges_for_node_ids``, ``node_context`` and unfiltered ``snapshot_stats`` on it.  For every ``node_context`` the
reference in-memory engine's ``impact_of`` on the saved graph is recorded too (``impact_engine``): the SQLite store's walk stops at
5 000 nodes / 25 000 edges, the engine's does not, so the fixture decides per node which one a cap-free walk must equal.

- ``est40`` (tenant ``lookup``): the dense 40-agent estate of oracle/make_golden.py.  Its heaviest agent's drilldown set (the agent
  plus its ``bfs_paths`` reachable set), its highest-degree nodes, a median-degree node and a few agents.
- ``kat-a`` / ``kat-b`` (blank tenant, stored as ``default``): a hand-made graph with bidirectional edges, a self loop, several
  relationships on one node pair, stored edges to ids that are not nodes, non-BMP ids, an isolated node, severity strings outside
  the table and a relationship outside the enum (statistics only: the reference's row reader rejects it), and a second scan of it.
- missing ids, a missing scan, an empty id set, the latest scan (blank scan id) and a blank tenant.

The fixture is the database (secondary indexes dropped after the answers were taken) and the answers, records as ``to_dict()``.

    python oracle/make_lookup_golden.py
"""

from __future__ import annotations

import gzip
import json
import sqlite3
import tempfile
from pathlib import Path
import sys

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_delta_golden import report  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402

from agent_bom.api.graph_store import SQLiteGraphStore  # noqa: E402
from agent_bom.db import graph_store as ref_db  # noqa: E402
from agent_bom.graph import EntityType, RelationshipType, UnifiedEdge, UnifiedGraph, UnifiedNode, build_unified_graph_from_report  # noqa: E402
from agent_bom.graph.container import AttackPath, InteractionRisk  # noqa: E402

R = RelationshipType


def kat(second: bool = False) -> UnifiedGraph:
    A, S, P, V, T = EntityType.AGENT, EntityType.SERVER, EntityType.PACKAGE, EntityType.VULNERABILITY, EntityType.TOOL
    g = UnifiedGraph()
    for n in (
        UnifiedNode(id="agent:a", entity_type=A, label="a", severity="high", risk_score=6.0),
        UnifiedNode(id="agent:\U0001F600", entity_type=A, label="smile"),
        UnifiedNode(id="agent:ﬁ", entity_type=A, label="ligature", severity="URGENT"),     # severity outside the table
        UnifiedNode(id="server:s1", entity_type=S, label="s1", severity="medium"),
        UnifiedNode(id="server:s2", entity_type=S, label="s2", attributes={"k": [1, 2]}),
        UnifiedNode(id="server:\U00010400", entity_type=S, label="deseret"),
        UnifiedNode(id="pkg:p1", entity_type=P, label="p1@1.0", severity="low"),
        UnifiedNode(id="vuln:CVE-1", entity_type=V, label="CVE-1", severity="critical", risk_score=9.1),
        UnifiedNode(id="tool:t", entity_type=T, label="t", severity="Weird"),
        UnifiedNode(id="tool:lonely", entity_type=T, label="isolated"),
        UnifiedNode(id="tool:t2", entity_type=T, label="t2"),
    ):
        g.add_node(n)
    for e in (
        UnifiedEdge("agent:a", "server:s1", R.USES), UnifiedEdge("agent:\U0001F600", "server:s1", R.USES),
        UnifiedEdge("agent:ﬁ", "server:s2", R.USES, traversable=False),
        UnifiedEdge("server:s1", "server:s2", R.SHARES_SERVER, direction="bidirectional"),
        UnifiedEdge("server:s2", "server:\U00010400", R.SHARES_SERVER, direction="bidirectional", weight=0.5),
        UnifiedEdge("server:s1", "server:s1", R.SHARES_SERVER),                                   # self loop
        UnifiedEdge("server:s2", "server:s2", R.SHARES_SERVER, direction="bidirectional"),        # bidirectional self loop
        UnifiedEdge("server:s1", "pkg:p1", R.DEPENDS_ON, evidence={"version": "1.0"}),
        UnifiedEdge("pkg:p1", "vuln:CVE-1", R.VULNERABLE_TO), UnifiedEdge("server:s1", "tool:t", R.PROVIDES_TOOL),
        UnifiedEdge("agent:a", "tool:t", R.USES), UnifiedEdge("agent:a", "tool:t", R.INVOKED),        # several relationships on one pair
        UnifiedEdge("agent:a", "tool:t", R.ACCESSED, confidence=0.7, provenance={"src": "runtime"}),
        UnifiedEdge("agent:a", "runtime:ghost", R.INVOKED), UnifiedEdge("runtime:ghost2", "tool:t", R.ACCESSED),   # endpoints that are not nodes
        UnifiedEdge("runtime:\U0001F47B", "server:s2", R.ACCESSED),
        UnifiedEdge("server:\U00010400", "agent:\U0001F600", R.SHARES_SERVER, direction="bidirectional"),
        UnifiedEdge("tool:t2", "tool:t2", "custom_rel"),                                         # relationship outside the enum
    ):
        g.add_edge(e)
    g.attack_paths = [AttackPath("agent:a", "vuln:CVE-1", ["agent:a", "server:s1", "pkg:p1", "vuln:CVE-1"], [], 8.5, "a reaches CVE-1", [], [], ["CVE-1"])]
    g.interaction_risks = [InteractionRisk("shared_server", ["a", "\U0001F600"], 6.5, "two agents share s1", "ASI07")]
    if second:
        g.add_node(UnifiedNode(id="agent:b", entity_type=A, label="b", severity="info"))
        g.add_edge(UnifiedEdge("agent:b", "server:s2", R.USES))
        g.attack_paths, g.interaction_risks = [], []
    return g


def plain(value):
    if hasattr(value, "to_dict"):
        return value.to_dict()
    if isinstance(value, dict):
        return {k: plain(v) for k, v in value.items()}
    if isinstance(value, (list, tuple)):
        return [plain(v) for v in value]
    return value


def main():
    out_dir = OUT / "lookup"
    out_dir.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    conn = sqlite3.connect(str(tmp))
    conn.row_factory = sqlite3.Row
    ref_db._init_db(conn)
    graphs = {}

    def save(g, scan, tenant, created):
        g.scan_id, g.tenant_id, g.created_at = scan, tenant, created
        ref_db.save_graph(conn, g)
        graphs[(ref_db.normalize_graph_tenant_id(tenant), scan)] = g

    save(build_unified_graph_from_report(report(40, dense=(4, 8, 2))), "est40", "lookup", "2026-01-01T00:00:00+00:00")
    save(kat(), "kat-a", "", "2026-02-01T00:00:00+00:00")
    save(kat(second=True), "kat-b", "", "2026-02-02T00:00:00+00:00")
    # fixture size: one timestamp for every row (save_graph stamps each with the wall clock)
    for table in ("graph_nodes", "graph_edges"):
        conn.execute(f"UPDATE {table} SET first_seen = '2026-01-01T00:00:00+00:00', last_seen = '2026-01-01T00:00:00+00:00'")
    conn.execute("UPDATE graph_edges SET valid_from = '2026-01-01T00:00:00+00:00' WHERE valid_from != ''")
    conn.commit()
    conn.close()

    store = SQLiteGraphStore(tmp)
    est = graphs[("lookup", "est40")]
    degree: dict[str, int] = {}
    for e in est.edges:
        degree[e.source] = degree.get(e.source, 0) + 1
        if e.target != e.source:
            degree[e.target] = degree.get(e.target, 0) + 1
    agents = sorted(n for n, v in est.nodes.items() if getattr(v.entity_type, "value", v.entity_type) == "agent")
    reach = {a: store.bfs_paths(tenant_id="lookup", scan_id="est40", source=a)[1] for a in agents}
    heavy = max(agents, key=lambda a: (len(reach[a]), a))
    drill = {heavy} | reach[heavy]
    by_degree = sorted(degree, key=lambda n: (-degree[n], n))
    median = sorted(degree, key=lambda n: (degree[n], n))[len(degree) // 2]
    print(f"est40: {len(est.nodes)} nodes, {len(est.edges)} edges; heaviest agent {heavy} reaches {len(reach[heavy])}; top degree {degree[by_degree[0]]}")

    cases = []

    def case(method, tenant, scan, **kw):
        fn = getattr(store, method)
        body = plain(fn(tenant_id=tenant, scan_id=scan, **kw))
        c = {"method": method, "tenant": tenant, "scan": scan, **{k: sorted(v) if isinstance(v, set) else v for k, v in kw.items()}, "expected": body}
        if method == "node_context" and body is not None:
            resolved = scan or store.latest_snapshot_id(tenant_id=tenant)
            c["impact_engine"] = plain(graphs[(ref_db.normalize_graph_tenant_id(tenant), resolved)].impact_of(kw["node_id"]))
        cases.append(c)

    case("nodes_by_ids", "lookup", "est40", node_ids=drill)
    case("edges_for_node_ids", "lookup", "est40", node_ids=drill)
    case("edges_for_node_ids", "lookup", "est40", node_ids=set(by_degree[:3]))
    case("nodes_by_ids", "lookup", "est40", node_ids=set(by_degree[:3]) | {"missing:1"})
    for nid in by_degree[:3] + [median, heavy, agents[0]]:
        case("node_context", "lookup", "est40", node_id=nid)
    case("snapshot_stats", "lookup", "est40")
    case("snapshot_stats", "lookup", "")
    kat_ids = ["agent:a", "agent:\U0001F600", "agent:ﬁ", "server:s1", "server:s2", "server:\U00010400", "pkg:p1", "vuln:CVE-1", "tool:t", "tool:lonely"]
    for tenant, scan in (("", "kat-a"), ("default", "kat-b"), (" ", "")):
        case("nodes_by_ids", tenant, scan, node_ids=set(kat_ids) | {"runtime:ghost", "nope"})
        case("edges_for_node_ids", tenant, scan, node_ids={"server:s2", "tool:t"})
        case("edges_for_node_ids", tenant, scan, node_ids={"runtime:ghost", "runtime:\U0001F47B", "agent:ﬁ"})
        case("edges_for_node_ids", tenant, scan, node_ids=set(kat_ids))
        for nid in kat_ids + ["runtime:ghost"]:
            case("node_context", tenant, scan, node_id=nid)
        case("snapshot_stats", tenant, scan)
    for tenant, scan in (("", "missing"), ("nobody", ""), ("lookup", "kat-a")):
        case("nodes_by_ids", tenant, scan, node_ids={"agent:a"})
        case("edges_for_node_ids", tenant, scan, node_ids={"agent:a"})
        case("node_context", tenant, scan, node_id="agent:a")
        case("snapshot_stats", tenant, scan)
    case("nodes_by_ids", "", "kat-a", node_ids=set())
    case("edges_for_node_ids", "", "kat-a", node_ids=set())

    conn = sqlite3.connect(str(tmp))
    for (name,) in conn.execute("SELECT name FROM sqlite_master WHERE type = 'index' AND name LIKE 'idx_%'").fetchall():
        conn.execute(f"DROP INDEX {name}")
    conn.commit()
    conn.execute("VACUUM")
    conn.close()
    with gzip.GzipFile(out_dir / "graph.sqlite.gz", "wb", mtime=0) as fh:
        fh.write(tmp.read_bytes())
    with gzip.GzipFile(out_dir / "expected.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps(cases, separators=(",", ":"), sort_keys=True).encode())
    for c in cases:
        e = c["expected"]
        size = len(e) if isinstance(e, list) else (len(e["edges_out"]) + len(e["edges_in"]) if isinstance(e, dict) and "edges_out" in e else "-")
        print(f"{c['method']:<20} {c['tenant']!r:<10} {c['scan']!r:<8} {size}")
    print(f"-> {out_dir} {sum(f.stat().st_size for f in out_dir.iterdir()) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
