#!/usr/bin/env python3
"""Generate tests/golden/compliance/ with the UNMODIFIED reference SQLite store's compliance posture.

Graphs are saved with the reference ``SQLiteGraphStore.save_graph`` into one SQLite file, and the same store answers
``compliance_summary`` on it.

- ``est40`` (tenant ``compliance``): the dense 40-agent estate of oracle/make_golden.py, built by the reference builder, with every
  blast radius given a seeded pick of each tag list ``_collect_compliance_tags`` reads, plus CIS and ``skill_audit:`` findings.
- ``kat`` (blank tenant, stored as ``default``): a hand-made graph with repeated tags in a row, tags without ``-``, a leading ``-``
  and an empty tag, lower-case and non-ASCII tags (``ß``, ``ﬁ``, ``İ``), empty and NULL severity, entity types outside the enum, a
  framework tagging 130 nodes, and ``[]``, NULL, ``{}`` and ``"x"`` stored as ``compliance_tags``.
- ``kat2`` (blank tenant, the latest scan there): a second scan with other tags.
- ``bad-json`` / ``bad-tag`` (tenant ``errors``): malformed JSON, and tags that are not strings, whose errors are recorded.

Calls cover framework filters (``""``, ``owasp``, ``OWASP``, ``ss``, prefixes without ``-``, an absent prefix) and latest,
blank-tenant and missing scans.  Answers are recorded in the store's key order (the tests compare JSON text); an exception as
``{"error": "<type>: <message>"}``.

    python oracle/make_compliance_golden.py
"""

from __future__ import annotations

import gzip
import json
import random
import sqlite3
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_delta_golden import report  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402

from agent_bom.api.graph_store import SQLiteGraphStore  # noqa: E402
from agent_bom.graph import EntityType, UnifiedGraph, UnifiedNode, build_unified_graph_from_report  # noqa: E402

# reference-shaped tag vocabulary per blast-radius key (graph/builder.py _collect_compliance_tags)
VOCAB = {
    "owasp_tags": ["LLM01", "LLM02", "LLM05", "LLM06", "LLM08"],
    "atlas_tags": ["AML.T0010", "AML.T0051", "AML.T0054"],
    "attack_tags": ["T1059", "T1195.002", "T1552"],
    "nist_ai_rmf_tags": ["GOVERN-1.1", "MAP-3.4", "MEASURE-2.7", "MANAGE-4.1"],
    "owasp_mcp_tags": ["MCP01", "MCP04", "MCP07"],
    "owasp_agentic_tags": ["ASI01", "ASI03", "ASI06"],
    "eu_ai_act_tags": ["ART-9", "ART-15"],
    "nist_csf_tags": ["ID.RA-01", "PR.DS-01", "DE.CM-08"],
    "iso_27001_tags": ["A.5.23", "A.8.8", "A.8.28"],
    "soc2_tags": ["CC6.1", "CC7.1", "CC8.1"],
    "cis_tags": ["CIS-2.1", "CIS-7.4", "CIS-16.1"],
}


def est40() -> UnifiedGraph:
    rep = report(40, dense=(4, 8, 2))
    rng = random.Random(20261017)
    for br in rep["blast_radius"]:
        for key, words in VOCAB.items():
            if rng.random() < 0.6:
                br[key] = rng.sample(words, rng.randint(1, len(words)))
    g = build_unified_graph_from_report(rep)
    for i in range(12):            # CIS benchmark and skill-audit findings
        tags = [f"CIS-{1 + i % 5}.{i % 3}"] if i % 2 else [f"skill_audit:{('credential_exposure', 'shell_access', 'prompt_injection')[i % 3]}", "OWASP-LLM01"]
        g.add_node(UnifiedNode(id=f"misconfig:finding-{i:02d}", entity_type=EntityType.MISCONFIGURATION, label=f"finding {i}",
                               severity=("critical", "high", "medium", "low")[i % 4], risk_score=float(i), compliance_tags=tags))
    return g


def kat(second: bool = False) -> UnifiedGraph:
    V, P, S, A = EntityType.VULNERABILITY, EntityType.PACKAGE, EntityType.SERVER, EntityType.AGENT
    g = UnifiedGraph()
    rows = [
        ("vuln:a", V, "high", ["OWASP-LLM01", "OWASP-LLM01", "soc2"]),                 # a repeated tag
        ("vuln:b", V, "critical", ["owasp-llm02", "OWASP-LLM01", "AML.T0051"]),
        ("vuln:c", V, "", ["T1059", "skill_audit:shell", "", "-lead"]),                # no '-', empty, leading '-'
        ("vuln:d", V, "low", ["ß", "ss-1", "straße-x", "SS"]),                          # ß -> SS
        ("vuln:e", V, "medium", ["ﬁ-1", "fi", "İ-x", "ı-y", "i"]),                      # ﬁ -> FI, İ stays, ı -> I
        ("vuln:f", P, "high", ["owasp-llm05", "CIS-1.1"]),                              # severity NULL below
        ("vuln:g", S, "medium", ["CIS-1.1", "cis-2"]),                                  # entity type outside the enum below
        ("vuln:h", A, "high", ["x"]),                                                   # compliance_tags '[]' below
        ("vuln:i", A, "high", ["x"]),                                                   # NULL below
        ("vuln:j", A, "high", ["x"]),                                                   # '{}' below
        ("vuln:k", A, "high", ["x"]),                                                   # '"x"' below
        ("agent:z", A, "low", ["OWASP-LLM01", "owasp"]),
        ("agent:é", A, "low", ["OWASP-LLM09"]),
    ]
    if second:
        rows = [("vuln:a", V, "high", ["OWASP-LLM03"]), ("vuln:q", V, "low", ["SOC2-CC6", "soc2"]), ("pkg:r", P, "", ["ATLAS-1", "OWASP-LLM03"])]
    for nid, t, sev, tags in rows:
        g.add_node(UnifiedNode(id=nid, entity_type=t, label=nid, severity=sev, risk_score=1.0, compliance_tags=tags))
    if not second:
        for i in range(130):                                                           # a framework tagging more than 100 nodes
            g.add_node(UnifiedNode(id=f"pkg:bulk-{i:03d}", entity_type=P, label=f"bulk {i}", severity=("high", "low", "")[i % 3], risk_score=0.0,
                                   compliance_tags=[f"BULK-{i % 7}", "bulk-0"] if i % 5 else ["BULK-0"]))
    return g


def main():
    out_dir = OUT / "compliance"
    out_dir.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    store = SQLiteGraphStore(tmp)

    def save(g, scan, tenant, created):
        g.scan_id, g.tenant_id, g.created_at = scan, tenant, created
        store.save_graph(g)

    save(est40(), "est40", "compliance", "2026-01-01T00:00:00+00:00")
    save(kat(), "kat", "", "2026-02-01T00:00:00+00:00")
    save(kat(second=True), "kat2", "", "2026-02-02T00:00:00+00:00")
    bad = UnifiedGraph()
    for nid in ("vuln:1", "vuln:2", "vuln:3"):
        bad.add_node(UnifiedNode(id=nid, entity_type=EntityType.VULNERABILITY, label=nid, severity="high", compliance_tags=["OWASP-LLM01"]))
    save(bad, "bad-json", "errors", "2026-03-01T00:00:00+00:00")
    save(bad, "bad-tag", "errors", "2026-03-02T00:00:00+00:00")
    save(bad, "bad-list", "errors", "2026-03-03T00:00:00+00:00")
    conn = sqlite3.connect(str(tmp))
    for nid, raw in (("vuln:h", "[]"), ("vuln:i", None), ("vuln:j", "{}"), ("vuln:k", '"x"')):
        conn.execute("UPDATE graph_nodes SET compliance_tags = ? WHERE id = ? AND scan_id = 'kat'", (raw, nid))
    conn.execute("UPDATE graph_nodes SET severity = NULL WHERE id = 'vuln:f' AND scan_id = 'kat'")
    conn.execute("UPDATE graph_nodes SET entity_type = 'custom_kind' WHERE id IN ('vuln:g', 'pkg:bulk-007') AND scan_id = 'kat'")
    conn.execute("UPDATE graph_nodes SET compliance_tags = '[\"A-1\", ' WHERE id = 'vuln:2' AND scan_id = 'bad-json'")
    conn.execute("UPDATE graph_nodes SET compliance_tags = '[\"A-1\", 5]' WHERE id = 'vuln:2' AND scan_id = 'bad-tag'")
    conn.execute("UPDATE graph_nodes SET compliance_tags = '[\"A-1\", [\"B-2\"]]' WHERE id = 'vuln:3' AND scan_id = 'bad-list'")
    # fixture size: one timestamp for every row (save_graph stamps each with the wall clock)
    for table in ("graph_nodes", "graph_edges"):
        conn.execute(f"UPDATE {table} SET first_seen = '2026-01-01T00:00:00+00:00', last_seen = '2026-01-01T00:00:00+00:00'")
    conn.execute("UPDATE graph_edges SET valid_from = '2026-01-01T00:00:00+00:00' WHERE valid_from != ''")
    conn.commit()
    conn.close()

    cases = []

    def case(**kw):
        try:
            body = store.compliance_summary(**kw)
        except Exception as exc:
            body = {"error": f"{type(exc).__name__}: {exc}"}
        cases.append({"kwargs": kw, "expected": body})

    filters = ("", "owasp", "OWASP", "ss", "SS", "llm05", "cc6.1", "aml.t0051", "cis", "bulk", "i", "fi", "İ", "skill_audit:shell", "absent", "-")
    for scan, tenant in (("est40", "compliance"), ("kat", ""), ("kat2", "")):
        for flt in filters:
            case(tenant_id=tenant, scan_id=scan, framework=flt)
    for tenant, scan in (("", ""), (" ", "kat"), ("default", "kat"), ("", "missing"), ("nobody", ""), ("compliance", ""), ("compliance", "kat")):
        case(tenant_id=tenant, scan_id=scan)
        case(tenant_id=tenant, scan_id=scan, framework="owasp")
    for scan in ("bad-json", "bad-tag", "bad-list"):
        case(tenant_id="errors", scan_id=scan)
        case(tenant_id="errors", scan_id=scan, framework="absent")

    conn = sqlite3.connect(str(tmp))
    for (name,) in conn.execute("SELECT name FROM sqlite_master WHERE type = 'index' AND name LIKE 'idx_%'").fetchall():
        conn.execute(f"DROP INDEX {name}")
    conn.commit()
    conn.execute("VACUUM")
    conn.close()
    with gzip.GzipFile(out_dir / "graph.sqlite.gz", "wb", mtime=0) as fh:
        fh.write(tmp.read_bytes())
    with gzip.GzipFile(out_dir / "expected.json.gz", "wb", mtime=0) as fh:       # key order kept: it is part of the answer
        fh.write(json.dumps(cases, separators=(",", ":")).encode())
    for c in cases:
        e = c["expected"]
        print(f"{json.dumps(c['kwargs'], ensure_ascii=False):<70} {e.get('error') or (e['framework_count'], e['total_tagged_findings'])}")
    print(f"-> {out_dir} {sum(f.stat().st_size for f in out_dir.iterdir()) / 1024:.0f} KiB, {len(cases)} cases")


if __name__ == "__main__":
    main()
