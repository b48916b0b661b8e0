#!/usr/bin/env python3
"""Generate tests/golden/ocsf/events.json.gz with the UNMODIFIED reference's ``UnifiedGraph.to_ocsf_events``.

Runs only where the reference tree is importable (the tests read the fixture alone).  Per graph the fixture holds the node
records (a finding's whole ``to_dict()``, of other nodes what the export reads) and the edge stream, so the graph can be
replayed; graphs of the builder-identity reports are replayed from those reports instead.  The reference's events are run with
enrichment on and off under two product versions and stored factored (see ``reference_events``), without their ``time``
field.  The reference builds ``blast_by_type`` by iterating a set of strings, so
its key order changes from one process to the next: the fixture is written with sorted keys (and gzip mtime 0), which makes
re-running this script reproduce it byte for byte.

    python oracle/make_ocsf_golden.py            # writes the fixture
    python oracle/make_ocsf_golden.py --time     # instead times the reference export (profiles/ocsf_reference.json)

Kept apart from oracle/make_golden.py and oracle/make_fix_first_golden.py so the fixtures they write are untouched; graph
builders are shared with them.
"""

from __future__ import annotations

import gzip
import json
import sqlite3
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_golden import AG, CRED, MIS, OUT, PKG, REF, SRV, TOOL, VULN, R, estate, kat_derived, kat_probe, mesh_inventory  # noqa: E402
from oracle.make_fix_first_golden import kat_focus  # noqa: E402

from agent_bom.graph import FINDING_ENTITY_TYPES, EntityType, UnifiedEdge, UnifiedGraph, UnifiedNode  # noqa: E402
from agent_bom.graph.builder import build_unified_graph_from_report  # noqa: E402

from agent_bom_b200.graph.schema import enum_value  # noqa: E402

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
from ocsf_golden import expand  # noqa: E402

VERSIONS = ("0.0.0", "3.1.4-rc1")


def kat_ocsf():
    """Edge cases of the export: every listed and unlisted source kind, duplicate and bidirectional sources, a long reverse row,
    a deep reverse chain, stored classification values, odd severities, attribute value kinds, tags and empty labels."""
    E = EntityType
    g = UnifiedGraph(scan_id="golden")

    def node(nid, et, label=None, **kw):
        g.add_node(UnifiedNode(id=nid, entity_type=et, label=nid if label is None else label, **kw))

    def edge(s, t, rel, direction="directed"):
        g.add_edge(UnifiedEdge(source=s, target=t, relationship=rel, direction=direction))

    node("vuln:hub", VULN, "CVE-2032-0001", severity="critical", attributes={"cvss": 9.8, "kev": True, "epss": 1, "refs": ["a", "b"], "nested": {"x": 1},
                                                                             "note": None, "vendor": "acme"},
         compliance_tags=["OWASP-LLM05", "NIST-CSF-ID.RA"])
    node("agent:a", AG, "agent-a")
    node("server:s", SRV, "")
    node("pkg:p", PKG, "left-pad")
    node("cred:k", CRED, "API_KEY")
    node("tool:t", TOOL, "run_shell")
    node("user:u", E.USER, "dana")
    for s, rel in (("agent:a", R.USES), ("server:s", R.VULNERABLE_TO), ("pkg:p", R.AFFECTS), ("pkg:p", R.VULNERABLE_TO), ("cred:k", R.EXPOSES_CRED),
                   ("tool:t", R.EXPLOITABLE_VIA), ("user:u", R.ASSUMES), ("ghost:gone", R.VULNERABLE_TO)):
        edge(s, "vuln:hub", rel)
    edge("vuln:hub", "agent:a", R.LATERAL_PATH, "bidirectional")            # the reversed twin lists agent:a again
    edge("vuln:hub", "server:s", R.REMEDIATES)                              # out-edge only: not a source
    # more than 64 in-neighbours of mixed kinds
    node("vuln:wide", VULN, "CVE-2032-0002", severity="HIGH")
    for i in range(75):
        kind = (PKG, SRV, AG, CRED, TOOL)[i % 5]
        node(f"wide:{i:03d}", kind, f"w{i:03d}" if i % 7 else "")
        edge(f"wide:{i:03d}", "vuln:wide", R.VULNERABLE_TO if i % 3 else R.AFFECTS)
    edge("wide:004", "vuln:wide", R.EXPLOITABLE_VIA)
    edge("ghost:wide", "vuln:wide", R.VULNERABLE_TO)
    # a reverse chain deeper than 4
    node("vuln:deep", VULN, "CVE-2032-0003", severity="bogus")
    prev = "vuln:deep"
    for d in range(7):
        nid = f"chain:{d}"
        node(nid, (PKG, SRV, AG)[d % 3], f"c{d}")
        edge(nid, prev, R.DEPENDS_ON if d else R.VULNERABLE_TO)
        prev = nid
    # no in-edges; a misconfiguration; stored classification values; empty severity and label
    node("vuln:alone", VULN, "", severity="")
    node("mis:open", MIS, "Open-Port", severity="medium", attributes={"port": 22, "ratio": 0.5, "open": False})
    edge("server:s", "mis:open", R.VULNERABLE_TO)
    edge("cred:k", "mis:open", R.EXPOSES_CRED)
    node("vuln:stored", VULN, "Stored-Class", severity="low", class_uid=2003, category_uid=7, type_uid=123456, severity_id=5, compliance_tags=["CIS-1.1"])
    edge("pkg:p", "vuln:stored", R.VULNERABLE_TO)
    node("mis:stored", MIS, "Stored-2001", severity="HIGH", class_uid=2001)
    edge("agent:a", "mis:stored", R.USES, "bidirectional")
    return g


def node_rec(n):
    """A finding's ``to_dict()`` without its creation timestamps (wall-clock values the export never reads); of any other node only
    what the export reads from it: id, entity type and label."""
    if n.entity_type in FINDING_ENTITY_TYPES:
        d = n.to_dict()
        d.pop("first_seen")
        d.pop("last_seen")
        return d
    return {"id": n.id, "entity_type": enum_value(n.entity_type), "label": n.label}


def edge_rec(e):
    return {"source": e.source, "target": e.target, "relationship": enum_value(e.relationship), "direction": e.direction, "traversable": bool(e.traversable)}


def strip_time(events):
    out = []
    for ev in events:
        ev = dict(ev)
        assert isinstance(ev.pop("time"), int)
        out.append(ev)
    return json.loads(json.dumps(out))


def reference_events(g):
    """The reference's events with enrichment on and off under every product version, stored factored: the un-enriched events of
    the first version and each event's ``graph_context``.  Every run is checked to be exactly what ``ocsf_golden.expand`` rebuilds
    from that pair (an enriched event is the plain one plus its context; versions differ only in ``metadata.product.version``)."""
    runs = {(v, enrich): strip_time(g.to_ocsf_events(v, enrich_neighbors=enrich)) for v in VERSIONS for enrich in (True, False)}
    stored = {"plain": runs[(VERSIONS[0], False)], "graph_context": [ev["graph_context"] for ev in runs[(VERSIONS[0], True)]]}
    for (v, enrich), evs in runs.items():
        assert expand(stored, v, enrich) == evs, (v, enrich)
    return stored


def graph_case(name, g, *, with_graph=True, **extra):
    case = {"name": name, "scan_id": g.scan_id, "tenant_id": g.tenant_id, "created_at": g.created_at, "events": reference_events(g), **extra}
    if with_graph:
        case |= {"nodes": [node_rec(n) for n in g.nodes.values()], "edges": [edge_rec(e) for e in g.edges]}
    print(f"ocsf {name}: {len(g.nodes)} nodes, {len(g.edges)} edges, {len(case['events']['plain'])} findings")
    return case


def snapshot_cases():
    """Snapshots in the SQLite file tests/golden/snapshot/graph.sqlite.gz (written by the reference's save_graph), loaded by the
    reference's load_graph."""
    from agent_bom.db import graph_store as ref_db

    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    tmp.write_bytes(gzip.decompress((OUT / "snapshot" / "graph.sqlite.gz").read_bytes()))
    conn = sqlite3.connect(str(tmp))
    conn.row_factory = sqlite3.Row
    out = []
    for tenant, scan in (("default", "scan-a"), ("default", "scan-b"), ("acme", "scan-a")):
        g = ref_db.load_graph(conn, tenant_id=tenant, scan_id=scan)
        out.append(graph_case(f"snapshot_{tenant}_{scan}", g, with_graph=False, tenant=tenant, snapshot_scan=scan))
    conn.close()
    return out


def builder_cases():
    """The reference builder's graphs of the builder-identity reports (tests/golden/identity/builder_identity.json.gz), so the
    light builder's record and columnar graphs of the same reports can be checked against them."""
    docs = json.loads(gzip.decompress((OUT / "identity" / "builder_identity.json.gz").read_bytes()))
    out = []
    for doc in docs:
        g = build_unified_graph_from_report(json.loads(json.dumps(doc["report"])))
        g.scan_id, g.tenant_id, g.created_at = f"builder-{doc['label']}-scan", "default", "2026-05-01T00:00:00+00:00"
        out.append(graph_case(f"builder_{doc['label']}", g, with_graph=False, builder=doc["label"]))   # replayed from the report
    return out


def golden():
    graphs = [("mesh", mesh_inventory()), ("estate_150", estate(150)), ("estate_dense_40", estate(40, dense=(4, 6, 2))), ("kat_probe", kat_probe()),
              ("kat_derived", kat_derived()), ("kat_focus", kat_focus()), ("kat_ocsf", kat_ocsf())]
    cases = []
    for name, g in graphs:
        g.scan_id, g.tenant_id, g.created_at = f"{name}-scan", "default", "2026-05-01T00:00:00+00:00"
        cases.append(graph_case(name, g))
    cases += snapshot_cases()
    cases += builder_cases()
    out = OUT / "ocsf"
    out.mkdir(parents=True, exist_ok=True)
    with gzip.GzipFile(out / "events.json.gz", "wb", mtime=0) as fh:
        fh.write(json.dumps({"versions": list(VERSIONS), "cases": cases}, sort_keys=True).encode())
    print(f"-> {out / 'events.json.gz'} {(out / 'events.json.gz').stat().st_size / 1024:.0f} KiB")


def time_reference(reps: int = 5):
    """Wall time of the reference's to_ocsf_events() (enriched) on generator estates and on the bench-knob estate."""
    import platform

    from agent_bom_b200 import estate as est_mod

    rec = {"cases": [], "host": {"machine": platform.machine(), "python": platform.python_version(), "processor": platform.processor(), "threads": 1}}
    bench = est_mod.generate(300, 2145, est_mod.BENCH_KNOBS, exact_rank=True)
    for label, g, r in (("generator_150", estate(150), reps), ("generator_1000", estate(1000), 3),
                        ("bench_knobs_300", build_unified_graph_from_report(bench.report_json()), 3)):
        g.to_ocsf_events()
        ts = []
        for _ in range(r):
            t0 = time.perf_counter()
            ev = g.to_ocsf_events()
            ts.append(time.perf_counter() - t0)
        med = sorted(ts)[len(ts) // 2]
        rec["cases"].append({"estate": label, "nodes": len(g.nodes), "edges": len(g.edges), "findings": len(ev), "median_s": med, "reps": r,
                             "events_per_s": len(ev) / med})
        print(rec["cases"][-1])
    dst = Path(__file__).resolve().parents[1] / "profiles" / "ocsf_reference.json"
    dst.write_text(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    assert REF.exists()
    if "--time" in sys.argv:
        time_reference()
    else:
        golden()
