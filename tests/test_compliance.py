"""Compliance posture on the host: ``B200GraphStore.compliance_summary`` with the numpy oracle standing in for the device, against the
unmodified SQLite store on every golden case (oracle/make_compliance_golden.py), compared as JSON text so key order counts; the host
interning against a restatement of the reference's per-pair loop on seeded random rows; an audit of the SQL a warm call sends; and
delegation without a SQLite inner store.
"""

from __future__ import annotations

import gzip
import json
import random
import sqlite3
from collections import defaultdict
from pathlib import Path
from types import SimpleNamespace

import pytest
from oracle.compliance_oracle import ComplianceOracle

from agent_bom_b200.graph import lookup
from agent_bom_b200.graph.compliance import ComplianceInputs, ComplianceSummary, summarize
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.store import B200GraphStore, B200UnsupportedOperationError

GOLD = Path(__file__).parent / "golden" / "compliance"
CASES = json.loads(gzip.decompress((GOLD / "expected.json.gz").read_bytes()))
IDS = [f"{i}-{c['kwargs'].get('tenant_id')}-{c['kwargs'].get('scan_id')}-{c['kwargs'].get('framework', '')}" for i, c in enumerate(CASES)]


@pytest.fixture(scope="module")
def db_path(tmp_path_factory) -> Path:
    path = tmp_path_factory.mktemp("compliance") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.fixture
def oracle_device(monkeypatch):
    """Every graph's compliance table built by the oracle."""

    def device_graph(self):
        if self._dg is None:
            self._dg = ComplianceOracle()
        return self._dg

    monkeypatch.setattr(UnifiedGraph, "device_graph", property(device_graph))


def store(db_path) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


def call(s: B200GraphStore, kwargs) -> str:
    try:
        body = s.compliance_summary(**kwargs)
    except Exception as exc:
        body = {"error": f"{type(exc).__name__}: {exc}"}
    return json.dumps(body)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_compliance_matches_reference(db_path, oracle_device, case):
    s = store(db_path)
    want = json.dumps(case["expected"])
    assert call(s, case["kwargs"]) == want
    assert call(s, case["kwargs"]) == want             # warm: from the cached summary (or, after an error, built again)


def test_goldens_cover_the_edge_cases():
    def body(**kw):
        return next(c["expected"] for c in CASES if c["kwargs"] == kw)

    kat = body(tenant_id="", scan_id="kat", framework="")["frameworks"]
    assert {"", "SS", "FI", "İ", "I", "T1059", "AML.T0051", "SKILL_AUDIT:SHELL", "BULK"} <= set(kat)
    assert kat["SS"]["tags"] == ["SS", "ss-1", "ß"] and kat["SS"]["total_findings"] == 3                 # ß -> SS; straße-x -> STRASSE
    assert kat["OWASP"]["total_findings"] == 8 and kat["OWASP"]["node_count"] == 5                         # a repeated tag counts twice
    assert kat["BULK"]["node_count"] == 130 and len(kat["BULK"]["node_ids"]) == 100
    assert "unknown" in kat["CIS"]["by_severity"] and "custom_kind" in kat["CIS"]["by_entity_type"]
    assert not {"vuln:h", "vuln:i", "vuln:j", "vuln:k"} & {n for f in kat.values() for n in f["node_ids"]}  # [], NULL, {}, "x"
    assert body(tenant_id="errors", scan_id="bad-json") == {"error": "OperationalError: malformed JSON"}
    assert body(tenant_id="errors", scan_id="bad-tag", framework="absent")["error"].startswith("TypeError")
    assert body(tenant_id="errors", scan_id="bad-list")["error"].startswith("AttributeError")
    assert body(tenant_id="", scan_id="missing") == {"scan_id": "missing", "framework_count": 0, "total_tagged_findings": 0, "frameworks": {}}


def test_a_build_that_raises_caches_nothing(db_path, oracle_device):
    s = store(db_path)
    for _ in range(2):
        with pytest.raises(sqlite3.OperationalError, match="malformed JSON"):
            s.compliance_summary(tenant_id="errors", scan_id="bad-json")
    assert s._graph("errors", "bad-json")._compliance is None


def test_sql_audit_warm_calls_send_only_latest_scan_resolution(db_path, oracle_device, monkeypatch):
    statements: list[str] = []
    real_connect = lookup.sqlite3.connect

    def traced(*a, **k):
        conn = real_connect(*a, **k)
        conn.set_trace_callback(statements.append)
        return conn

    monkeypatch.setattr(sqlite3, "connect", traced)
    s = store(db_path)

    def requests():
        s.compliance_summary(tenant_id="compliance", scan_id="est40")
        s.compliance_summary(tenant_id="compliance", scan_id="est40", framework="owasp")
        s.compliance_summary(tenant_id="", scan_id="", framework="ss")
        s.compliance_summary(tenant_id="", scan_id="kat", framework="bulk")

    requests()
    assert any("json_array_length" in q for q in statements)
    statements.clear()
    requests()
    assert statements
    for q in statements:
        assert "graph_snapshots" in q, q
    statements.clear()
    s.compliance_summary(tenant_id="", scan_id="kat")
    assert statements == []


def test_without_sqlite_inner_store_delegates(tmp_path):
    calls = []
    inner = SimpleNamespace(compliance_summary=lambda **kw: calls.append(kw) or {"scan_id": "x"})
    s = B200GraphStore(inner)
    assert s.compliance_summary(tenant_id="t", scan_id="x", framework="owasp") == {"scan_id": "x"}
    assert calls == [{"tenant_id": "t", "scan_id": "x", "framework": "owasp"}]
    inner._db_path = str(tmp_path / "absent.sqlite")                # a SQLite path that does not exist is not SQLite-backed
    s.compliance_summary()
    assert calls[-1] == {"tenant_id": "", "scan_id": "", "framework": ""}
    with pytest.raises(B200UnsupportedOperationError):
        B200GraphStore().compliance_summary(scan_id="x")


# ── the host interning against the reference's per-pair loop ──
def loop_summary(rows, scan_id: str, framework: str) -> dict:
    """The reference's roll-up (api/graph_store.py:987-1031) restated over ``rows`` = (id, entity_type, severity, tags text) in id order."""
    flt = framework.upper()
    stats: dict = {}
    for node_id, entity_type, severity, raw in rows:
        for tag in json.loads(raw):
            name = tag.split("-")[0].upper() if "-" in tag else tag.upper()
            if flt and flt != name:
                continue
            st = stats.setdefault(name, {"n": 0, "sev": defaultdict(int), "type": defaultdict(int), "tags": set(), "ids": {}})
            st["n"] += 1
            st["sev"][severity or "unknown"] += 1
            st["type"][entity_type] += 1
            st["tags"].add(tag)
            st["ids"].setdefault(node_id, None)
    frameworks = {name: {"total_findings": st["n"], "by_severity": dict(st["sev"]), "by_entity_type": dict(st["type"]), "tags": sorted(st["tags"]),
                         "node_count": len(st["ids"]), "node_ids": list(st["ids"])[:100]} for name, st in sorted(stats.items())}
    return {"scan_id": scan_id, "framework_count": len(frameworks), "total_tagged_findings": sum(f["total_findings"] for f in frameworks.values()),
            "frameworks": frameworks}


_WORDS = ["owasp-llm01", "OWASP-LLM01", "LLM05", "cc6.1", "CIS-1.1", "cis-2", "T1059", "AML.T0051", "skill_audit:x", "", "-", "-x", "a-b-c", "ß", "ss-2",
          "straße-x", "ﬁ-1", "fi", "İ-1", "ı", "i", "ǅ-1", "Σ-σ", "日本-1", "😀", "MCP01", "x-"]


def random_rows(rng: random.Random, n: int) -> list[tuple]:
    vocab = _WORDS + [f"F{k}-{k % 3}" for k in range(60)]
    texts = [json.dumps(rng.sample(vocab, rng.randint(1, 4)) + ([rng.choice(vocab)] if rng.random() < 0.2 else [])) for _ in range(max(1, n // 4))]
    ids = sorted({f"{rng.choice('anpsv')}:{rng.randrange(10 * n)}{rng.choice(['', 'é', '日'])}" for _ in range(n)})
    return [(i, rng.choice(["agent", "package", "vulnerability", None, "custom"]), rng.choice(["high", "low", "", None, "critical", "HIGH"]),
             rng.choice(texts)) for i in ids]


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_host_interning_equals_the_reference_loop(seed):
    rng = random.Random(seed)
    rows = random_rows(rng, rng.choice([7, 150, 1200]))
    inputs = ComplianceInputs(rows)
    table = ComplianceOracle().compliance_table(inputs.row_text, inputs.row_sev, inputs.row_type, inputs.text_off, inputs.text_tags, inputs.tag_fw,
                                                len(inputs.frameworks), len(inputs.severities), len(inputs.types))
    summary = ComplianceSummary.__new__(ComplianceSummary)
    summary.frameworks = summarize(inputs, table)
    summary.total = sum(v["total_findings"] for v in summary.frameworks.values())
    for flt in ["", "owasp", "ss", "f1", "", "nope", "İ", "i", "日本"]:
        assert json.dumps(summary.select("scan", flt)) == json.dumps(loop_summary(rows, "scan", flt)), flt
