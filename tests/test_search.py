"""Node search and node pages on the host: ``B200GraphStore.search_nodes`` / ``page_nodes``, with the numpy oracle standing in for the
device, against the unmodified SQLite store on every golden case (oracle/make_search_golden.py); the token-text rule against real
FTS5 ``MATCH`` on random documents; an audit of the SQL a warm call sends; and delegation without a SQLite inner store.
"""

from __future__ import annotations

import gzip
import json
import random
import re
import sqlite3
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
from oracle.search_oracle import SearchOracle, token_text

from agent_bom_b200.graph import lookup
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.graph.search import MODE_FTS, compliance_match, fold_table, query_plan, source_match
from agent_bom_b200.store import B200GraphStore

GOLD = Path(__file__).parent / "golden" / "search"
CASES = json.loads(gzip.decompress((GOLD / "expected.json.gz").read_bytes()))
IDS = [f"{i}-{c['method']}" for i, c in enumerate(CASES)]


@pytest.fixture(scope="module")
def db_path(tmp_path_factory) -> Path:
    path = tmp_path_factory.mktemp("search") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.fixture
def oracle_device(monkeypatch):
    """Every graph's search calls answered by the oracle."""

    def device_graph(self):
        if self._dg is None:
            self._dg = SearchOracle()
        return self._dg

    monkeypatch.setattr(UnifiedGraph, "device_graph", property(device_graph))


def store(db_path) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


def plain(value):
    if hasattr(value, "to_dict"):
        return value.to_dict()
    if isinstance(value, dict):
        return {k: plain(v) for k, v in value.items()}
    if isinstance(value, (list, tuple)):
        return [plain(v) for v in value]
    return value


def call(s: B200GraphStore, c):
    kwargs = {k: (set(v) if k in ("entity_types", "compliance_prefixes", "data_sources") else v) for k, v in c["kwargs"].items()}
    try:
        body = plain(getattr(s, c["method"])(**kwargs))
    except Exception as exc:
        body = {"error": f"{type(exc).__name__}: {exc}"}
    return json.loads(json.dumps(body))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_search_matches_reference(db_path, oracle_device, case):
    assert call(store(db_path), case) == case["expected"]


def test_goldens_cover_the_edge_cases():
    def body(method, **kw):
        return next(c["expected"] for c in CASES if c["method"] == method and all(c["kwargs"].get(k) == v for k, v in kw.items()))

    assert body("search_nodes", query="CAFÉ", scan_id="kat")[1] == 1                   # LIKE: attributes are stored as JSON escapes
    assert body("search_nodes", query="istanbul", scan_id="kat")[1] == 1               # İ lowered to i + U+0307, the mark folded away
    assert body("search_nodes", query="eclair", scan_id="kat")[1] == 1                 # a combining acute folded away inside a token
    assert body("search_nodes", query="é.", scan_id="kat")[1] == 0                     # an FTS phrase that tokenises to nothing
    assert body("search_nodes", query="x .", scan_id="kat")[1] == 0
    assert body("search_nodes", query="cve-2024-000", scan_id="kat")[1] == 2           # consecutive tokens, the last a prefix
    ids = [n["id"] for n in body("search_nodes", query="", compliance_prefixes=["OWASP"], scan_id="kat")[0]]
    assert "agent:cursor" not in ids and "server:straße" in ids                          # no '% p' clause; '=' clause
    assert body("search_nodes", query="agent", scan_id="kat-noindex")[1] == 0          # no index rows
    assert body("page_nodes", limit=5, scan_id="kat-noindex")[3] == 19
    assert body("page_nodes", cursor="!!!", scan_id="kat") == {"error": "ValueError: Invalid graph cursor"}


# ── the token-text rule against real FTS5 ──
_SCHEMA = ("CREATE VIRTUAL TABLE gns USING fts5(tenant_id UNINDEXED, scan_id UNINDEXED, node_id UNINDEXED, entity_type, severity, "
           "compliance_tags, data_sources, search_text)")
_ALPHABET = ("abcdefghijklmnopqrstuvwxyz0123456789 _.:-/\"'{}[],@#" + "éèêëÉàâäçñøœßİıŁłŠšŽžΣσςΆάЖжЯя" + "̧́̈̊"
             + "日本語中文한국어ｆｕｌｌＡＢ" + "😀🚀\U00010400" + "ǅǄǆﬁﬂ" + "  ​　" + "٣٤۵߀")


def _doc(rng: random.Random) -> tuple[str, list[str]]:
    words = ["".join(rng.choice(_ALPHABET) for _ in range(rng.randint(1, 9))) for _ in range(rng.randint(1, 12))]
    cols = [rng.choice(["agent", "server", "package"]), rng.choice(["high", "", "low"]), " ".join(words[:2]).lower(), " ".join(words[2:3]).lower()]
    text = " ".join(p for p in [cols[0], *words, cols[1], cols[2], cols[3]] if p).lower()
    return text, cols


def _query(rng: random.Random, docs: list[str]) -> str:
    if rng.random() < 0.7:          # pieces of a document: ids, words and splits of them
        doc = rng.choice(docs)
        a = rng.randrange(len(doc))
        return doc[a: a + rng.randint(1, 14)]
    return "".join(rng.choice(_ALPHABET + "AGENTXYZ") for _ in range(rng.randint(1, 8)))


def test_token_text_equals_fts5_match():
    """For random documents over a wide code-point mix, a phrase matches the token text at a token start exactly when FTS5 ``MATCH``
    finds the row, both on ``search_text`` alone and on the whole row with the reference schema."""
    rng = random.Random(20261017)
    conn = sqlite3.connect(":memory:")
    conn.execute(_SCHEMA)
    docs = []
    for i in range(3000):
        text, cols = _doc(rng)
        conn.execute("INSERT INTO gns(rowid, tenant_id, scan_id, node_id, entity_type, severity, compliance_tags, data_sources, search_text) "
                     "VALUES (?, 't', 's', ?, ?, ?, ?, ?, ?)", (i, str(i), *cols, text))
        docs.append(text)
    fold = fold_table(sorted({ord(c) for d in docs for c in d if ord(c) >= 0x80}))      # lowering adds code points (İ -> i + U+0307)
    toks = [" " + token_text(d, fold) for d in docs]
    checked = 0
    for _ in range(600):
        q = _query(rng, docs)
        mode, phrases = query_plan(q)
        if mode != MODE_FTS:
            continue
        expr = " AND ".join(f'"{t}"*' for t in (t.strip() for t in re.findall(r"[A-Za-z0-9_.:-]+", q)) if t)
        whole = {r for (r,) in conn.execute("SELECT rowid FROM gns WHERE gns MATCH ?", (expr,))}
        text_only = {r for (r,) in conn.execute("SELECT rowid FROM gns WHERE search_text MATCH ?", (expr,))}
        mine = set() if phrases is None else {i for i, t in enumerate(toks) if all((" " + p.decode()) in t for p in phrases)}
        assert whole == text_only == mine, q
        checked += bool(whole)
    assert checked > 100


def test_filter_clauses():
    assert compliance_match("owasp", "OWASP") and compliance_match("owasp-llm01 soc2", "owasp") and compliance_match("owasp llm", "owasp")
    assert compliance_match("cis owasp-llm05", "owasp") and compliance_match("cis owasp soc2", "owasp")
    assert not compliance_match("x owasp", "owasp")                 # the reference has no '% p' clause
    assert not compliance_match("owasp_x", "owasp_x")               # '=' compares the escaped prefix
    assert source_match("osv", "OSV") and source_match("osv nvd", "osv") and source_match("nvd osv", "osv") and source_match("a osv b", "osv")
    assert not source_match("osvx", "osv")


def test_sql_audit_warm_calls_are_keyed(db_path, oracle_device, monkeypatch):
    """A warm call sends SQLite only the latest-snapshot lookup and keyed record reads."""
    statements: list[str] = []
    real_connect = lookup.sqlite3.connect

    def traced(*a, **k):
        conn = real_connect(*a, **k)
        conn.set_trace_callback(statements.append)
        return conn

    monkeypatch.setattr(sqlite3, "connect", traced)
    s = store(db_path)

    def requests():
        s.search_nodes(tenant_id="search", scan_id="est40", query="agent", limit=5)
        s.search_nodes(tenant_id="", scan_id="", query="-", entity_types={"agent"})
        s.search_nodes(tenant_id="", scan_id="kat", query="cve", compliance_prefixes={"owasp"}, data_sources={"osv"})
        _, _, _, _, nxt = s.page_nodes(tenant_id="search", scan_id="est40", entity_types={"agent"}, limit=3)
        s.page_nodes(tenant_id="search", scan_id="", entity_types={"agent"}, limit=3, cursor=nxt)

    requests()
    assert any("graph_node_search" in q for q in statements)
    statements.clear()
    requests()
    assert statements
    for q in statements:
        assert "graph_snapshots" in q or "AND id IN (" in q, q


def test_without_sqlite_inner_store_delegates(tmp_path):
    calls = []
    inner = SimpleNamespace(search_nodes=lambda **kw: calls.append(("search_nodes", kw)) or ([], 0, None),
                            page_nodes=lambda **kw: calls.append(("page_nodes", kw)) or ("x", "", [], 0, None))
    s = B200GraphStore(inner)
    assert s.search_nodes(tenant_id="t", scan_id="x", query="q", cursor="c") == ([], 0, None)
    assert s.page_nodes(tenant_id="t", scan_id="x", limit=3) == ("x", "", [], 0, None)
    assert calls[0] == ("search_nodes", {"tenant_id": "t", "scan_id": "x", "query": "q", "entity_types": None, "min_severity_rank": 0,
                                         "compliance_prefixes": None, "data_sources": None, "cursor": "c", "offset": 0, "limit": 50})
    assert calls[1] == ("page_nodes", {"tenant_id": "t", "scan_id": "x", "entity_types": None, "min_severity_rank": 0, "cursor": None,
                                       "offset": 0, "limit": 3})
    inner._db_path = str(tmp_path / "absent.sqlite")                # a SQLite path that does not exist is not SQLite-backed
    assert s.search_nodes(query="q") == ([], 0, None)


def test_oracle_order_nulls_last_and_negative_zero():
    o = SearchOracle()
    o.search_text(np.zeros(5, np.int64), b"")
    o.build_search_table(np.full(0x110000, -1, np.int32), [3, -(1 << 31), 3, 3], [1.0, 9.0, float("nan"), -0.0], [0, 0, 0, 0], [0] * 4, [0] * 4,
                         [0] * 4, 1, 1, 1)
    page, total, _ = o.search(0, [])
    assert page.tolist() == [0, 3, 2, 1] and total == 4
