#!/usr/bin/env python3
"""Generate tests/golden/delta/ with the UNMODIFIED reference's snapshot diff.

Every pair of graphs is built with the reference builder (or by hand) and saved as scans of one SQLite database through the
reference's ``save_graph``; the fixture records the reference's ``diff_snapshots`` for each (tenant, old scan, new scan).

- ``est40``: the dense 40-agent estate of oracle/make_golden.py, and a second report of it with a seeded perturbation: agents dropped, servers added and removed, package versions changed (new package ids, labels and edge
  evidence), CVEs added and vulnerability severities changed (risk scores follow).
- ``kat``: a hand-made pair with ghost endpoints, an entity type and a relationship outside the enum, non-ASCII and astral-plane
  ids whose UTF-16 order differs from code-point order, NaN and -0.0 risks, bidirectional edges and a direction flip, a
  traversable flip and a weight change, confidence / activity / evidence / provenance changes, evidence text that differs only in
  key order (not a change), and ``severity_id`` set by hand; plus a disjoint scan and the same scan diffed with itself.
- the blank tenant (normalised to ``default``), a blank scan id and a missing scan id.
- ``alerts.json.gz``: the reference's ``compute_delta_alerts`` on the graphs its store loads back, in both directions and from no
  previous snapshot; the hand-made pair adds attack paths, interaction risks, new high / critical / medium / upper-case findings and
  values the event references redact.

The 150-agent estate is not included: its pair of snapshots alone is 2 MB compressed, against about 0.7 MB for everything here.

    python oracle/make_delta_golden.py            # writes the fixtures
    python oracle/make_delta_golden.py --time     # instead times the reference's diff_snapshots on generator estates (profiles/)
"""

from __future__ import annotations

import copy
import gzip
import json
import random
import sqlite3
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import OUT, densify, load_generator  # noqa: E402

from agent_bom.db import graph_store as ref_db  # noqa: E402
from agent_bom.graph import EntityType, RelationshipType, UnifiedEdge, UnifiedGraph, UnifiedNode, build_unified_graph_from_report  # noqa: E402
from agent_bom.graph.container import AttackPath, InteractionRisk  # noqa: E402
from agent_bom.graph.webhooks import compute_delta_alerts  # noqa: E402

R = RelationshipType


def report(agents: int, dense=None):
    rep, _ = load_generator().generate_estate(agents=agents, seed=2145, vulnerable_package_rate=0.08)
    return densify(rep, *dense) if dense else rep


def perturb(rep, seed: int):
    rng = random.Random(seed)
    rep = copy.deepcopy(rep)
    agents = rep["agents"]
    for _ in range(max(1, len(agents) // 20)):
        agents.pop(rng.randrange(len(agents)))
    for ai, agent in enumerate(agents):
        servers = agent["mcp_servers"]
        if rng.random() < 0.1 and len(servers) > 1:
            servers.pop(rng.randrange(len(servers)))
        if rng.random() < 0.1:
            extra = copy.deepcopy(servers[0])
            extra["name"] = f"{extra['name']}-added"
            servers.append(extra)
        for server in servers:
            for pi, pkg in enumerate(server["packages"]):
                u = rng.random()
                if u < 0.04:
                    pkg["version"] = pkg["version"] + ".1"
                elif u < 0.07:
                    pkg.setdefault("vulnerabilities", []).append({"id": f"CVE-2031-{ai:04d}{pi:03d}", "severity": rng.choice(("critical", "high", "low"))})
                for v in pkg.get("vulnerabilities", []):
                    if rng.random() < 0.1:
                        v["severity"] = rng.choice(("critical", "high", "medium", "low"))
    return rep


def kat_pair():
    """Old and new graphs of the hand-made case."""
    A, S, P, V, T = EntityType.AGENT, EntityType.SERVER, EntityType.PACKAGE, EntityType.VULNERABILITY, EntityType.TOOL

    def node(nid, et, label, **kw):
        return UnifiedNode(id=nid, entity_type=et, label=label, **kw)

    def base():
        g = UnifiedGraph()
        for n in (
            node("agent:a", A, "a"), node("agent:b", A, "b"), node("agent:é", A, "é"), node("agent:\U0001F600", A, "smile"),
            node("agent:ﬁ", A, "ligature"),                                     # U+FB01 > U+1F600 in UTF-16 order, < in code points
            node("server:s1", S, "s1"), node("server:s2", S, "s2"),
            node("pkg:p1", P, "p1@1.0"), node("pkg:p2", P, "p2@1.0", risk_score=float("nan")),
            node("pkg:neg", P, "neg", risk_score=-0.0), node("vuln:CVE-1", V, "CVE-1", severity="high", risk_score=7.5),
            node("custom:x", "custom_kind", "x"), node("tool:t", T, "t"),
        ):
            g.add_node(n)
        for e in (
            UnifiedEdge("agent:a", "server:s1", R.USES), UnifiedEdge("agent:b", "server:s1", R.USES),
            UnifiedEdge("agent:é", "server:s2", R.USES), UnifiedEdge("agent:\U0001F600", "server:s2", R.USES),
            UnifiedEdge("agent:ﬁ", "server:s2", R.USES),
            UnifiedEdge("server:s1", "pkg:p1", R.DEPENDS_ON, evidence={"version": "1.0", "a": 1, "b": 2}),
            UnifiedEdge("server:s1", "pkg:p2", R.DEPENDS_ON, evidence={"version": "1.0"}),
            UnifiedEdge("server:s2", "pkg:neg", R.DEPENDS_ON), UnifiedEdge("pkg:p1", "vuln:CVE-1", R.VULNERABLE_TO),
            UnifiedEdge("server:s1", "server:s2", R.SHARES_SERVER, direction="bidirectional"),
            UnifiedEdge("server:s2", "tool:t", R.PROVIDES_TOOL, weight=0.5), UnifiedEdge("agent:a", "tool:t", "custom_rel"),
            UnifiedEdge("agent:b", "custom:x", R.USES, traversable=False),
            UnifiedEdge("agent:a", "runtime:ghost", R.INVOKED), UnifiedEdge("runtime:ghost2", "tool:t", R.ACCESSED),
            UnifiedEdge("agent:b", "server:s2", R.USES, confidence=0.9),
            UnifiedEdge("agent:é", "server:s1", R.USES), UnifiedEdge("agent:\U0001F600", "server:s1", R.USES),
        ):
            g.add_edge(e)
        return g

    old = base()
    new = base()
    new.nodes["pkg:p1"].label = "p1@1.1"
    new.nodes["pkg:p2"].risk_score = 0.0                     # NaN is stored as NULL: reads back 0.0 on both sides
    new.nodes["pkg:neg"].risk_score = 0.0                    # -0.0 == 0.0
    new.nodes["vuln:CVE-1"].severity = "critical"
    new.nodes["custom:x"].entity_type = "other_kind"         # both outside the enum
    new.nodes["agent:ﬁ"].severity_id = 3                # severity_id alone
    del new.nodes["agent:b"]
    new.add_node(node("agent:c", A, "c"))
    new.add_node(node("runtime:ghost", T, "ghost"))          # a ghost endpoint that becomes a node
    new.edges = [e for e in new.edges if e.source != "agent:b" and e.target != "agent:b"]
    by = {(e.source, e.target, getattr(e.relationship, "value", e.relationship)): e for e in new.edges}
    by[("server:s1", "pkg:p1", "depends_on")].evidence = {"b": 2, "a": 1, "version": "1.0"}     # key order only: not a change
    by[("server:s1", "pkg:p2", "depends_on")].evidence = {"version": "1.1"}
    by[("server:s1", "server:s2", "shares_server")].direction = "directed"
    by[("server:s2", "tool:t", "provides_tool")].weight = 0.75
    by[("agent:é", "server:s2", "uses")].traversable = False
    by[("agent:\U0001F600", "server:s2", "uses")].confidence = 0.5
    by[("agent:ﬁ", "server:s2", "uses")].activity_id = 2
    by[("server:s2", "pkg:neg", "depends_on")].provenance = {"source": "sbom"}
    by[("agent:é", "server:s1", "uses")].evidence = {"seen": ["x"]}
    new.add_edge(UnifiedEdge("agent:c", "server:s1", R.USES))
    new.add_edge(UnifiedEdge("agent:c", "runtime:ghost3", R.DELEGATED_TO))
    new.add_edge(UnifiedEdge("server:s2", "server:s1", R.SHARES_SERVER, direction="bidirectional"))
    new.add_edge(UnifiedEdge("agent:a", "tool:t", "another_rel"))
    old.attack_paths = [AttackPath("agent:a", "tool:t", ["agent:a", "server:s1", "tool:t"], [], 8.0, "a reaches t", ["c1"], [], ["CVE-1"])]
    new.attack_paths = old.attack_paths + [AttackPath("agent:c", "vuln:CVE-1", ["agent:c", "server:s1", "pkg:p1", "vuln:CVE-1"], [], 9.5, "", [], [], ["CVE-1"]),
                                           AttackPath("agent:é", "pkg:neg", ["agent:é", "server:s2", "pkg:neg"], [], 5.0, "low", [], [], [])]
    old.interaction_risks = [InteractionRisk("shared_server", ["a", "é"], 7.5, "two agents share s1", "ASI07")]
    new.interaction_risks = [InteractionRisk("shared_server", ["a", "é"], 7.5, "two agents share s1", "ASI07"),
                             InteractionRisk("credential_overlap", ["a", "c"], 9.0, "agents share a credential", None),
                             InteractionRisk("tool_overlap", ["c", "é"], 3.0, "minor", None)]
    new.add_node(node("vuln:CVE-2", V, "CVE-2", severity="critical", risk_score=9.8, attributes={"cvss_score": 9.8, "is_kev": True, "path": "/etc/x"}))
    new.add_node(node("vuln:CVE-3", V, "CVE-3", severity="medium"))
    new.add_node(node("misconf:m1", EntityType.MISCONFIGURATION, "open bucket https://u:p@example.com/b?q=1", severity="high"))
    new.add_node(node("misconf:m2", EntityType.MISCONFIGURATION, "m2", severity="HIGH"))
    disjoint = UnifiedGraph()
    disjoint.add_node(node("zzz:1", A, "1"))
    disjoint.add_node(node("zzz:2", S, "2"))
    disjoint.add_edge(UnifiedEdge("zzz:1", "zzz:2", R.USES))
    disjoint.add_edge(UnifiedEdge("zzz:1", "zzz:ghost", "custom_rel"))
    return old, new, disjoint


def main():
    out_dir = OUT / "delta"
    out_dir.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    conn = sqlite3.connect(str(tmp))
    conn.row_factory = sqlite3.Row
    ref_db._init_db(conn)

    def save(g, scan, tenant, created):
        g.scan_id, g.tenant_id, g.created_at = scan, tenant, created
        ref_db.save_graph(conn, g)

    r40 = report(40, dense=(4, 8, 2))
    save(build_unified_graph_from_report(r40), "est40-a", "delta", "2026-01-01T00:00:00+00:00")
    save(build_unified_graph_from_report(perturb(r40, 40)), "est40-b", "delta", "2026-01-02T00:00:00+00:00")
    old, new, disjoint = kat_pair()
    save(old, "kat-a", "", "2026-02-01T00:00:00+00:00")            # blank tenant: stored under "default"
    save(new, "kat-b", "", "2026-02-02T00:00:00+00:00")
    save(disjoint, "kat-z", "", "2026-02-03T00:00:00+00:00")
    # fixture size: one timestamp for every row (save_graph stamps each with the wall clock) and no secondary indexes; the diff
    # below is computed on the database as it is stored
    for table in ("graph_nodes", "graph_edges"):
        conn.execute(f"UPDATE {table} SET first_seen = '2026-01-01T00:00:00+00:00', last_seen = '2026-01-01T00:00:00+00:00'")
    conn.execute("UPDATE graph_edges SET valid_from = '2026-01-01T00:00:00+00:00' WHERE valid_from != ''")
    conn.execute("UPDATE graph_edges SET valid_to = '2026-01-02T00:00:00+00:00' WHERE valid_to IS NOT NULL")
    for (name,) in conn.execute("SELECT name FROM sqlite_master WHERE type = 'index' AND name LIKE 'idx_%'").fetchall():
        conn.execute(f"DROP INDEX {name}")
    conn.commit()
    conn.execute("VACUUM")

    cases = []
    pairs = [("delta", "est40-a", "est40-b"), ("delta", "est40-b", "est40-a"),
             ("delta", "est40-a", "missing"), ("delta", "", "est40-a"), ("", "kat-a", "kat-b"), ("default", "kat-b", "kat-a"), (" ", "kat-a", "kat-a"),
             ("", "kat-a", "kat-z"), ("", "kat-z", ""), ("", "", ""), ("delta", "kat-a", "kat-b")]
    for tenant, a, b in pairs:
        body = ref_db.diff_snapshots(conn, a, b, tenant_id=tenant)
        cases.append({"tenant": tenant, "old": a, "new": b, "diff": body})
        print(f"{tenant!r} {a!r} -> {b!r}: " + ", ".join(f"{k} {len(v)}" for k, v in body.items()))
    # compute_delta_alerts on the graphs the reference store loads back, both ways and from no previous snapshot.  The reference
    # loader rejects the hand-made graphs' entity type outside the enum, so those are the saved graphs themselves (their stored
    # rows read back the same for every field an alert reads: agent lists are given sorted, as the store writes them)
    in_memory = {"kat-a": old, "kat-b": new, "kat-z": disjoint}

    def load(tenant, scan):
        return in_memory[scan] if scan in in_memory else ref_db.load_graph(conn, tenant_id=tenant, scan_id=scan)

    alerts = []
    for tenant, a, b in (("delta", "est40-a", "est40-b"), ("delta", "est40-b", "est40-a"), ("delta", None, "est40-a"), ("", "kat-a", "kat-b"),
                         ("", "kat-b", "kat-a"), ("", None, "kat-b"), ("", "kat-a", "kat-z")):
        old_g = load(tenant, a) if a else None
        new_g = load(tenant, b)
        body = compute_delta_alerts(old_g, new_g)
        alerts.append({"tenant": tenant, "old": a, "new": b, "alerts": body})
        print(f"alerts {tenant!r} {a!r} -> {b!r}: " + ", ".join(x["type"] for x in body))
    conn.close()
    with gzip.GzipFile(out_dir / "alerts.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps(alerts, separators=(",", ":"), sort_keys=True).encode())
    with gzip.GzipFile(out_dir / "graph.sqlite.gz", "wb", mtime=0) as fh:
        fh.write(tmp.read_bytes())
    with gzip.GzipFile(out_dir / "expected.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps(cases, separators=(",", ":"), sort_keys=True).encode())
    print(f"-> {out_dir} {sum(f.stat().st_size for f in out_dir.iterdir()) / 1024:.0f} KiB")


def time_reference():
    """Reference ``diff_snapshots`` on the 150- and 600-agent estates against their perturbed copies, one process (one core)."""
    import os
    import platform
    import time

    rec = {"what": "reference diff_snapshots(old, new) on SQLite, median of 3 after one warm call", "host": platform.processor() or platform.machine(),
           "cpus_used": 1, "sizes": {}}
    for agents in (150, 600):
        tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
        conn = sqlite3.connect(str(tmp))
        conn.row_factory = sqlite3.Row
        ref_db._init_db(conn)
        rep = report(agents)
        for scan, r in (("a", rep), ("b", perturb(rep, agents))):
            g = build_unified_graph_from_report(r)
            g.scan_id, g.tenant_id = scan, "t"
            ref_db.save_graph(conn, g)
        conn.commit()
        ref_db.diff_snapshots(conn, "a", "b", tenant_id="t")
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            body = ref_db.diff_snapshots(conn, "a", "b", tenant_id="t")
            ts.append(time.perf_counter() - t0)
        n = conn.execute("SELECT COUNT(*) FROM graph_nodes WHERE scan_id = 'a'").fetchone()[0]
        m = conn.execute("SELECT COUNT(*) FROM graph_edges WHERE scan_id = 'a'").fetchone()[0]
        rec["sizes"][str(agents)] = {"nodes_old": n, "edges_old": m, "diff_snapshots_s": round(sorted(ts)[1], 3), "answer": {k: len(v) for k, v in body.items()}}
        conn.close()
        print(agents, rec["sizes"][str(agents)], flush=True)
    rec["compute_delta_alerts"] = "not measured"
    out = Path(__file__).resolve().parents[1] / "profiles" / "delta_reference.json"
    out.write_text(json.dumps(rec, indent=1) + "\n")
    print(f"-> {out} (os.cpu_count() = {os.cpu_count()})")


if __name__ == "__main__":
    if "--time" in sys.argv:
        time_reference()
    else:
        main()
