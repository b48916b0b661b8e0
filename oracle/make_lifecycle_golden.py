#!/usr/bin/env python3
"""Generate tests/golden/lifecycle/ with the UNMODIFIED reference's edge lifecycle reads.

One SQLite database is written through the reference's own ``save_graph``, so ``valid_from`` carries over from the previous
snapshot and ``valid_to`` is closed on the edges a save drops.  It holds:

- the blank tenant (stored as ``default``): five snapshots with explicit, distinct ``created_at`` in which edges disappear and come
  back, one snapshot re-saved under the same scan id, ghost endpoints, a relationship outside the enum, non-ASCII and astral-plane
  ids whose UTF-16 order differs from code-point order (U+FB01 against U+1F600), an explicit ``valid_to`` on an edge;
- rows edited after the saves: ``valid_from = ''`` (read as ``first_seen``), ``valid_to`` set to ``''`` and left NULL, and an edge
  row of a scan with no ``graph_snapshots`` row (the reference's JOIN drops it);
- tenant ``t2`` with four snapshots whose ``created_at`` ties are broken by scan id, and tenant ``empty`` with edge rows but no
  snapshot.

``expected.json.gz`` records ``active_edges_at`` for each tenant at: before everything, exactly each ``created_at``, exactly each
``valid_to``, between snapshots, after everything, ``''`` and strings that are not timestamps (``'2026'``, ``'z'``, non-ASCII); and
``changed_edges_between_scans`` for pairs of these snapshots and for the pairs of tests/golden/delta/graph.sqlite.gz (read only).
Timestamps are kept as stored.  The fixture is about 290 KiB, most of it the 40-agent delta pairs' row lists.

    python oracle/make_lifecycle_golden.py            # writes the fixtures
    python oracle/make_lifecycle_golden.py --time     # instead times the reference on generator estates (profiles/)
"""

from __future__ import annotations

import copy
import gzip
import json
import sqlite3
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import OUT  # noqa: E402

from agent_bom.db import graph_store as ref_db  # noqa: E402
from agent_bom.graph import EntityType, RelationshipType, UnifiedEdge, UnifiedGraph, UnifiedNode  # noqa: E402

R = RelationshipType
A, S, P, V, T = EntityType.AGENT, EntityType.SERVER, EntityType.PACKAGE, EntityType.VULNERABILITY, EntityType.TOOL

IDS = ["agent:a", "agent:b", "agent:é", "agent:\U0001F600", "agent:ﬁ", "server:s1", "server:s2", "pkg:p1", "pkg:p2", "vuln:CVE-1", "tool:t"]
KINDS = {"agent": A, "server": S, "pkg": P, "vuln": V, "tool": T}


def graph(edges, nodes=IDS) -> UnifiedGraph:
    g = UnifiedGraph()
    for nid in nodes:
        g.add_node(UnifiedNode(id=nid, entity_type=KINDS[nid.split(":")[0]], label=nid.split(":")[1]))
    for e in edges:
        g.add_edge(copy.deepcopy(e))
    return g


E = {
    "a-s1": UnifiedEdge("agent:a", "server:s1", R.USES),
    "b-s1": UnifiedEdge("agent:b", "server:s1", R.USES),
    "é-s2": UnifiedEdge("agent:é", "server:s2", R.USES),
    "smile-s2": UnifiedEdge("agent:\U0001F600", "server:s2", R.USES),
    "fi-s2": UnifiedEdge("agent:ﬁ", "server:s2", R.USES),
    "s1-p1": UnifiedEdge("server:s1", "pkg:p1", R.DEPENDS_ON, evidence={"version": "1.0"}),
    "s1-p2": UnifiedEdge("server:s1", "pkg:p2", R.DEPENDS_ON),
    "p1-cve": UnifiedEdge("pkg:p1", "vuln:CVE-1", R.VULNERABLE_TO),
    "s1-s2": UnifiedEdge("server:s1", "server:s2", R.SHARES_SERVER, direction="bidirectional"),
    "s2-t": UnifiedEdge("server:s2", "tool:t", R.PROVIDES_TOOL, weight=0.5),
    "a-t-custom": UnifiedEdge("agent:a", "tool:t", "custom_rel"),
    "a-ghost": UnifiedEdge("agent:a", "runtime:ghost", R.INVOKED),
    "ghost-t": UnifiedEdge("runtime:ghost2", "tool:t", R.ACCESSED),
    "b-s2-until": UnifiedEdge("agent:b", "server:s2", R.USES, valid_to="2026-03-02T12:00:00+00:00"),
}


def history(conn):
    def save(g, scan, tenant, created):
        g.scan_id, g.tenant_id, g.created_at = scan, tenant, created
        for n in g.nodes.values():                 # the builder stamps the wall clock: seen at the snapshot's time instead
            n.first_seen = n.last_seen = created
        for e in g.edges:
            e.first_seen = e.last_seen = created
            e.valid_from = ""
        ref_db.save_graph(conn, g)

    base = ["a-s1", "b-s1", "é-s2", "smile-s2", "fi-s2", "s1-p1", "s1-p2", "p1-cve", "s1-s2", "s2-t", "a-t-custom", "a-ghost", "ghost-t"]
    snaps = [
        ("s1", "2026-03-01T00:00:00+00:00", base + ["b-s2-until"]),
        ("s2", "2026-03-02T00:00:00+00:00", [k for k in base if k not in ("b-s1", "s1-p2", "a-ghost")]),          # three edges disappear
        ("s3", "2026-03-03T00:00:00+00:00", [k for k in base if k not in ("s1-p2",)]),                            # two of them come back
        ("s4", "2026-03-04T00:00:00+00:00", [k for k in base if k not in ("fi-s2", "a-t-custom")] + ["s1-p2"]),
    ]
    for scan, created, keys in snaps:
        edges = [copy.deepcopy(E[k]) for k in keys]
        if scan == "s3":
            for e in edges:
                if e.source == "server:s2" and e.target == "tool:t":
                    e.weight = 0.75
        save(graph(edges), scan, "", created)
    # s3 re-saved under the same scan id with a later created_at and one more edge
    edges = [copy.deepcopy(E[k]) for k in base if k != "s1-p2"] + [UnifiedEdge("agent:ﬁ", "tool:t", R.INVOKED)]
    for e in edges:
        if e.source == "server:s2" and e.target == "tool:t":
            e.weight = 0.75
        elif e.source == "agent:a" and e.target == "server:s1":
            e.confidence, e.evidence = 0.5, {"seen": ["x"]}
    save(graph(edges), "s3", "", "2026-03-03T06:00:00+00:00")
    save(graph([copy.deepcopy(E[k]) for k in base[:8]]), "s5", "", "2026-03-05T00:00:00+00:00")
    # tenant t2: a created_at tie broken by scan id
    for scan, created, keys in (("b", "2026-03-01T00:00:00+00:00", base[:6]), ("a", "2026-03-01T00:00:00+00:00", base[2:9]),
                                ("c", "2026-03-02T00:00:00+00:00", base[:4]), ("d", "2026-03-06T00:00:00+00:00", base)):
        save(graph([copy.deepcopy(E[k]) for k in keys]), scan, "t2", created)
    # rows edited after the saves
    conn.execute("UPDATE graph_edges SET valid_from = '' WHERE tenant_id = 'default' AND scan_id = 's1' AND source_id = 'agent:a'")
    conn.execute("UPDATE graph_edges SET valid_from = '', first_seen = '2026-02-15T00:00:00+00:00' WHERE tenant_id = 'default' AND scan_id = 's5' "
                 "AND source_id = 'pkg:p1'")
    conn.execute("UPDATE graph_edges SET valid_to = '' WHERE tenant_id = 'default' AND scan_id = 's2' AND source_id = 'agent:é'")
    conn.execute("UPDATE graph_edges SET valid_to = '2026-03-04T12:00:00+00:00' WHERE tenant_id = 't2' AND scan_id = 'd' AND source_id = 'server:s1'")
    for tenant, scan in (("default", "orphan"), ("empty", "e1")):
        conn.execute("INSERT INTO graph_edges (source_id, target_id, relationship, first_seen, last_seen, valid_from, scan_id, tenant_id) "
                     "VALUES ('agent:zz', 'server:s1', 'uses', '2026-01-01T00:00:00+00:00', '2026-01-01T00:00:00+00:00', '', ?, ?)", (scan, tenant))
    conn.commit()


def at_values(conn, tenant: str) -> list[str]:
    created = [r[0] for r in conn.execute("SELECT created_at FROM graph_snapshots WHERE tenant_id = ? ORDER BY created_at", (tenant,))]
    ends = [r[0] for r in conn.execute("SELECT DISTINCT valid_to FROM graph_edges WHERE tenant_id = ? AND valid_to != '' ORDER BY 1", (tenant,))]
    between = [a[:11] + "12:00:00+00:00" for a in created]
    return sorted(set(["2025-01-01T00:00:00+00:00", "2027-01-01T00:00:00+00:00", "", "2026", "z", "2026-03-0é", "\U0001F600"] + created + ends + between))


def main():
    out_dir = OUT / "lifecycle"
    out_dir.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    conn = sqlite3.connect(str(tmp))
    conn.row_factory = sqlite3.Row
    ref_db._init_db(conn)
    history(conn)
    conn.execute("VACUUM")
    active = []
    for tenant in ("", "default", " ", "t2", "empty", "nobody"):
        for at in at_values(conn, ref_db.normalize_graph_tenant_id(tenant)):
            body = ref_db.active_edges_at(conn, at, tenant_id=tenant)
            active.append({"tenant": tenant, "at": at, "edges": body})
    changes = []
    pairs = [("", "s1", "s2"), ("", "s2", "s3"), ("", "s3", "s4"), ("", "s4", "s1"), ("default", "s3", "s5"), ("", "s2", "s2"), ("t2", "a", "d"),
             ("", "s1", ""), ("", "", "s4"), ("", "s1", "missing"), ("", "orphan", "s1"), ("empty", "e1", "e1"), ("nobody", "s1", "s2")]
    for tenant, a, b in pairs:
        changes.append({"db": "lifecycle", "tenant": tenant, "old": a, "new": b, "body": ref_db.changed_edges_between_scans(conn, a, b, tenant_id=tenant)})
    conn.close()
    delta_db = Path(tempfile.mkdtemp()) / "delta.sqlite"
    delta_db.write_bytes(gzip.decompress((OUT / "delta" / "graph.sqlite.gz").read_bytes()))
    dconn = sqlite3.connect(f"file:{delta_db}?mode=ro", uri=True)
    dconn.row_factory = sqlite3.Row
    for tenant, a, b in (("delta", "est40-a", "est40-b"), ("delta", "est40-b", "est40-a"), ("", "kat-a", "kat-b"), ("default", "kat-b", "kat-a"),
                         ("", "kat-a", "kat-z"), ("", "kat-z", ""), ("delta", "est40-a", "missing")):
        changes.append({"db": "delta", "tenant": tenant, "old": a, "new": b, "body": ref_db.changed_edges_between_scans(dconn, a, b, tenant_id=tenant)})
    dconn.close()
    for c in changes:
        print(f"{c['db']} {c['tenant']!r} {c['old']!r} -> {c['new']!r}: {c['body']['summary']}")
    print(f"{len(active)} active_edges_at cases, {sum(len(a['edges']) for a in active)} edges")
    with gzip.GzipFile(out_dir / "graph.sqlite.gz", "wb", mtime=0) as fh:
        fh.write(tmp.read_bytes())
    with gzip.GzipFile(out_dir / "expected.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps({"active": active, "changes": changes}, separators=(",", ":"), sort_keys=True).encode())
    print(f"-> {out_dir} {sum(f.stat().st_size for f in out_dir.iterdir()) / 1024:.0f} KiB")


def time_reference(bound_s: float = 600.0):
    """The reference's two reads on the 150- and 600-agent estates saved as S = 2 and S = 8 perturbed snapshots, one process (one
    core).  A size whose first call exceeds ``bound_s`` is recorded as not finished within the bound."""
    import os
    import platform
    import time

    from agent_bom.graph import build_unified_graph_from_report
    from oracle.make_delta_golden import perturb, report

    rec = {"what": "reference active_edges_at (at = after the last snapshot) and changed_edges_between_scans (first -> last) on SQLite, "
                   "median of 3 after one warm call", "host": platform.processor() or platform.machine(), "cpus_used": 1,
           "bound_s": bound_s, "sizes": {}}
    for agents in (150, 600):
        rep = report(agents)
        for snaps in (2, 8):
            tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
            conn = sqlite3.connect(str(tmp))
            conn.row_factory = sqlite3.Row
            ref_db._init_db(conn)
            r = rep
            for s in range(snaps):
                g = build_unified_graph_from_report(r)
                g.scan_id, g.tenant_id, g.created_at = f"s{s}", "t", f"2026-04-{s + 1:02d}T00:00:00+00:00"
                ref_db.save_graph(conn, g)
                r = perturb(r, 1000 * agents + s)
            conn.commit()
            rows = conn.execute("SELECT COUNT(*) FROM graph_edges WHERE tenant_id = 't'").fetchone()[0]
            entry = {"snapshots": snaps, "edge_rows": rows}
            for name, call in (("active_edges_at_s", lambda: ref_db.active_edges_at(conn, "2027", tenant_id="t")),
                               ("changed_edges_between_scans_s", lambda: ref_db.changed_edges_between_scans(conn, "s0", f"s{snaps - 1}", tenant_id="t"))):
                t0 = time.perf_counter()
                call()
                first = time.perf_counter() - t0
                if first > bound_s:
                    entry[name] = f"not finished within {bound_s:.0f} s"
                    continue
                ts = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    call()
                    ts.append(time.perf_counter() - t0)
                entry[name] = round(sorted(ts)[1], 3)
            conn.close()
            rec["sizes"][f"{agents}x{snaps}"] = entry
            print(agents, snaps, entry, flush=True)
    out = Path(__file__).resolve().parents[1] / "profiles" / "lifecycle_reference.json"
    out.write_text(json.dumps(rec, indent=1) + "\n")
    print(f"-> {out} (os.cpu_count() = {os.cpu_count()})")


if __name__ == "__main__":
    if "--time" in sys.argv:
        time_reference()
    else:
        main()
