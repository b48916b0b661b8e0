#!/usr/bin/env python3
"""Generate tests/golden/search/ with the UNMODIFIED reference SQLite store's node search and node pages.

Graphs are saved with the reference ``SQLiteGraphStore.save_graph`` (which writes the ``graph_node_search`` FTS5 index) into one
SQLite file, and the same store answers ``search_nodes`` and ``page_nodes`` on it.

- ``est40`` (tenant ``search``): the dense 40-agent estate of oracle/make_golden.py.
- ``kat`` (blank tenant, stored as ``default``): a hand-made graph with non-ASCII ids, labels and attribute values (diacritics,
  ``ß``, ``İ``, combining marks, CJK, emoji), NULL and NaN risk, NULL ``severity_id``, ties on every sort key, and compliance-tag and
  data-source strings that hit each LIKE clause of the filters and the missing ``'% p'`` clause.
- ``kat-noindex`` (blank tenant, the latest scan there): the same graph saved by ``db/graph_store.save_graph`` alone, so it has
  no index rows: every search finds nothing while ``page_nodes`` pages it.

Calls: FTS phrases, multi-token AND, last-token prefix, phrases that tokenise to nothing, LIKE-path queries, every filter alone
and combined, offset pages, cursor walks to the last page, invalid cursors, a blank tenant, a missing scan and the latest scan;
``page_nodes`` by offset and by cursor.  Answers are recorded as ``to_dict()``; an exception as ``{"error": "<type>: <message>"}``.

    python oracle/make_search_golden.py
"""

from __future__ import annotations

import gzip
import json
import sqlite3
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle.make_delta_golden import report  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402

from agent_bom.api.graph_store import SQLiteGraphStore  # noqa: E402
from agent_bom.db import graph_store as ref_db  # noqa: E402
from agent_bom.graph import EntityType, UnifiedGraph, UnifiedNode, build_unified_graph_from_report  # noqa: E402

NAN = float("nan")


def kat() -> UnifiedGraph:
    A, S, P, V, T = EntityType.AGENT, EntityType.SERVER, EntityType.PACKAGE, EntityType.VULNERABILITY, EntityType.TOOL
    g = UnifiedGraph()
    rows = [
        # id, type, label, severity, risk, compliance tags, data sources, attributes
        ("agent:claude-desktop", A, "Claude Desktop", "high", 7.5, ["OWASP-LLM01", "soc2"], ["mcp-config"], {"note": "Café naïve"}),
        ("agent:cursor", A, "Cursor", "high", 7.5, ["x", "owasp"], ["mcp-config", "runtime"], {}),            # no '% p' clause
        ("agent:cursor-2", A, "Cursor", "high", 7.5, ["owasp", "llm"], ["OSV"], {}),                          # ties on every key but id
        ("agent:cursor-0", A, "Cursor", "high", 7.5, ["cis", "owasp", "soc2"], ["a", "osv", "b"], {}),
        ("agent:zero", A, "Ŝkip", "high", 0.0, [], [], {}),
        ("agent:negzero", A, "Ŝkip", "high", -0.0, [], [], {}),                                              # -0.0 = 0.0
        ("agent:nullsev", A, "Null severity", "high", 8.0, ["owasp_x"], ["osvx"], {}),                       # severity_id NULL below
        ("server:straße", S, "Straße", "medium", 5.0, ["owasp"], ["runtime"], {"city": "Straße"}),
        ("server:İstanbul", S, "İstanbul", "medium", 5.0, ["cis", "owasp-llm05"], ["osv", "nvd"], {"city": "İSTANBUL"}),
        ("server:ｆｕｌｌ", S, "ＦＵＬＬ width", "medium", 5.0, [], ["nvd", "osv"], {}),
        ("pkg:éclair", P, "éclair", "low", NAN, [], [], {"desc": "pâte à choux"}),               # NaN is stored as NULL
        ("pkg:loné", P, "́ lone mark", "low", None, [], [], {"k": "́̂ x́"}),
        ("pkg:nullrisk", P, "Null risk", "low", None, [], [], {}),
        ("vuln:CVE-2024-0001", V, "CVE-2024-0001", "critical", 9.8, ["OWASP-LLM05", "cis"], ["osv", "nvd"], {"summary": "日本語 テキスト"}),
        ("vuln:CVE-2024-0002", V, "CVE-2024-0002", "critical", 9.8, [], ["nvd osv"], {"summary": "agent:claude-desktop::x"}),
        ("vuln:CVE-2023-9999", V, "CVE-2023-9999", "critical", 9.8, [], [], {"summary": "ǅ Ǆ ǆ dz"}),
        ("tool:😀-emoji", T, "😀 emoji tool", "info", 1.0, [], [], {"e": "🚀 rocket_launch", "nested": {"a.b": "c:d"}}),
        ("tool:日本", T, "日本", "", 0.0, [], [], {}),
        ("tool:ελληνικά", T, "ΣΊΣΥΦΟΣ", "low", 2.0, [], [], {"w": "ΌΣΟΣ"}),
    ]
    for nid, t, label, sev, risk, tags, src, attrs in rows:
        g.add_node(UnifiedNode(id=nid, entity_type=t, label=label, severity=sev, risk_score=risk, compliance_tags=tags, data_sources=src,
                               attributes=attrs))
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
    out_dir = OUT / "search"
    out_dir.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp()) / "graph.sqlite"
    store = SQLiteGraphStore(tmp)

    def save(g, scan, tenant, created, index=True):
        g.scan_id, g.tenant_id, g.created_at = scan, tenant, created
        if index:
            store.save_graph(g)
        else:
            conn = sqlite3.connect(str(tmp))
            conn.row_factory = sqlite3.Row
            ref_db._init_db(conn)
            ref_db.save_graph(conn, g)
            conn.commit()
            conn.close()

    save(build_unified_graph_from_report(report(40, dense=(4, 8, 2))), "est40", "search", "2026-01-01T00:00:00+00:00")
    save(kat(), "kat", "", "2026-02-01T00:00:00+00:00")
    save(kat(), "kat-noindex", "", "2026-02-02T00:00:00+00:00", index=False)
    conn = sqlite3.connect(str(tmp))
    conn.execute("UPDATE graph_nodes SET severity_id = NULL WHERE id IN ('agent:nullsev', 'pkg:nullrisk')")
    # fixture size: one timestamp for every row (save_graph stamps each with the wall clock)
    for table in ("graph_nodes", "graph_edges"):
        conn.execute(f"UPDATE {table} SET first_seen = '2026-01-01T00:00:00+00:00', last_seen = '2026-01-01T00:00:00+00:00'")
    conn.execute("UPDATE graph_edges SET valid_from = '2026-01-01T00:00:00+00:00' WHERE valid_from != ''")
    conn.commit()
    conn.close()

    cases = []

    def run(method, **kw):
        try:
            return plain(getattr(store, method)(**kw))
        except Exception as exc:          # the route turns ValueError into 400
            return {"error": f"{type(exc).__name__}: {exc}"}

    def case(method, **kw):
        body = run(method, **kw)
        cases.append({"method": method, "kwargs": {k: sorted(v) if isinstance(v, set) else v for k, v in kw.items()}, "expected": body})
        return body

    def walk(method, limit, **kw):
        """Cursor pages to the last one."""
        cursor = None
        for _ in range(200):
            body = case(method, limit=limit, cursor=cursor, **kw)
            cursor = body[-1] if isinstance(body, list) else None
            if not cursor:
                return

    est = {"tenant_id": "search", "scan_id": "est40"}
    for q in ("agent", "cve", "server", "ag", "mcp server", "critical", "high agent", "agent-0001", "pkg:", "cve-2024", "nomatch", "-", "::", "é",
              "", "é.", "x ..", "a_b", "CVE"):
        case("search_nodes", query=q, **est)
    case("search_nodes", query="agent", entity_types={"agent"}, **est)
    case("search_nodes", query="cve", min_severity_rank=4, **est)
    case("search_nodes", query="agent", offset=5, limit=7, **est)
    case("search_nodes", query="server", offset=1000, limit=7, **est)
    walk("search_nodes", 17, query="agent", **est)
    walk("search_nodes", 25, query="-", **est)
    case("search_nodes", query="agent", tenant_id="search", scan_id="")
    case("page_nodes", entity_types={"agent"}, limit=10, **est)
    case("page_nodes", entity_types={"agent"}, offset=10, limit=10, **est)
    walk("page_nodes", 9, entity_types={"agent"}, **est)
    case("page_nodes", min_severity_rank=3, limit=50, **est)

    kat_ = {"tenant_id": "", "scan_id": "kat"}
    for q in ("claude-desktop", "agent:claude-desk", "cafe", "naive", "CAFÉ", "strasse", "straße", "stra", "istanbul", "eclair", "clair", "lone",
              "日本", "日本語", "rocket", "rocket_launch", "emoji", "cve-2024", "2024 0001", "cve 2024-0002", "cve-2024-000", "a.b", "c:d",
              "é", "::", "-", "é.", "x .", "null", "cursor", "σισυφοσ", "σίσυφος", "dz", "ǆ", "full", "ｆｕｌｌ", "'", '"quoted"', "%", "_", "\\",
              "owasp", "OWASP-LLM0", "llm", "x owasp"):
        case("search_nodes", query=q, **kat_)
    for flt in ({"entity_types": {"agent"}}, {"entity_types": {"agent", "server"}}, {"entity_types": {"nothing"}}, {"min_severity_rank": 3},
                {"min_severity_rank": 5}, {"min_severity_rank": -1}, {"compliance_prefixes": {"OWASP"}}, {"compliance_prefixes": {"owasp_x"}},
                {"compliance_prefixes": {"soc2", "CIS"}}, {"compliance_prefixes": {"x"}}, {"data_sources": {"osv"}}, {"data_sources": {"OSV", "runtime"}},
                {"data_sources": {"mcp-config"}}, {"entity_types": {"agent"}, "compliance_prefixes": {"owasp"}, "data_sources": {"osv"}},
                {"entity_types": {"server", "vulnerability"}, "min_severity_rank": 3, "data_sources": {"nvd"}}):
        case("search_nodes", query="", **flt, **kat_)
        case("search_nodes", query="agent", **flt, **kat_)
    walk("search_nodes", 2, query="", **kat_)
    walk("search_nodes", 3, query="-", **kat_)
    case("search_nodes", query="", offset=3, limit=4, **kat_)
    case("search_nodes", query="", offset=-2, limit=4, **kat_)
    case("search_nodes", query="", limit=0, **kat_)
    case("search_nodes", query="", limit=-3, **kat_)
    for bad in ("!!!", "eyJ4IjoxfQ", "WzEsMl0", "not-base64-json"):
        case("search_nodes", query="agent", cursor=bad, **kat_)
        case("page_nodes", cursor=bad, **kat_)
    for tenant, scan in (("", ""), (" ", "kat"), ("default", "kat"), ("", "missing"), ("nobody", ""), ("search", "kat"), ("", "kat-noindex")):
        case("search_nodes", query="agent", tenant_id=tenant, scan_id=scan)
        case("search_nodes", query="-", tenant_id=tenant, scan_id=scan)
        case("page_nodes", limit=5, tenant_id=tenant, scan_id=scan)
    case("search_nodes", query="agent", cursor="!!!", tenant_id="", scan_id="missing")
    case("search_nodes", query="agent", cursor="!!!", tenant_id="nobody", scan_id="")
    case("page_nodes", cursor="!!!", tenant_id="", scan_id="missing")
    walk("page_nodes", 4, **kat_)
    walk("page_nodes", 4, tenant_id="", scan_id="kat-noindex")
    case("page_nodes", entity_types={"agent"}, offset=2, limit=3, **kat_)
    walk("page_nodes", 2, entity_types={"agent"}, min_severity_rank=1, **kat_)
    case("page_nodes", offset=-1, limit=-1, **kat_)

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
        size = e["error"] if isinstance(e, dict) else (len(e[0]), e[1]) if c["method"] == "search_nodes" else (len(e[2]), e[3])
        print(f"{c['method']:<13} {json.dumps(c['kwargs'], ensure_ascii=False)[:90]:<90} {size}")
    print(f"-> {out_dir} {sum(f.stat().st_size for f in out_dir.iterdir()) / 1024:.0f} KiB, {len(cases)} cases")


if __name__ == "__main__":
    main()
