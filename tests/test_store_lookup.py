"""Snapshot lookups on the host: ``B200GraphStore.nodes_by_ids`` / ``edges_for_node_ids`` / ``node_context`` / ``snapshot_stats``, with
the numpy oracle standing in for the device, against the unmodified SQLite store on every golden case (oracle/make_lookup_golden.py);
delegation without a SQLite inner store and for filtered statistics; and an audit of the SQL a warm call sends.
"""

from __future__ import annotations

import gzip
import json
import sqlite3
from pathlib import Path
from types import SimpleNamespace

import pytest
from oracle.lookup_oracle import LookupOracle, impact_of

from agent_bom_b200.graph import lookup
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.store import B200GraphStore, B200UnsupportedOperationError

GOLD = Path(__file__).parent / "golden" / "lookup"
CASES = json.loads(gzip.decompress((GOLD / "expected.json.gz").read_bytes()))


def case_id(c) -> str:
    arg = c.get("node_id") or (f"{len(c['node_ids'])}ids" if "node_ids" in c else "")
    return f"{c['method']}:{c['tenant'].strip() or '-'}:{c['scan'] or 'latest'}:{arg}"


IDS = [f"{i}-{case_id(c)}" for i, c in enumerate(CASES)]


@pytest.fixture(scope="module")
def db_path(tmp_path_factory) -> Path:
    path = tmp_path_factory.mktemp("lookup") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.fixture
def oracle_device(monkeypatch):
    """Every graph's lookup calls and its ``impact_of`` walk answered by the oracle."""

    def device_graph(self):
        if self._dg is None:
            self._dg = LookupOracle(self.csr)
        return self._dg

    monkeypatch.setattr(UnifiedGraph, "device_graph", property(device_graph))
    monkeypatch.setattr(UnifiedGraph, "impact_of", lambda self, node_id, max_depth=4: impact_of(self, node_id, max_depth))


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
    kwargs = {k: (set(v) if k == "node_ids" else v) for k, v in c.items() if k in ("node_ids", "node_id")}
    return json.loads(json.dumps(plain(getattr(s, c["method"])(tenant_id=c["tenant"], scan_id=c["scan"], **kwargs))))


def expected(c):
    """The SQLite store's answer; ``node_context.impact`` is the reference engine's walk, which the store's walk caps can truncate."""
    body = c["expected"]
    if c["method"] == "node_context" and body is not None:
        body = dict(body, impact=c["impact_engine"])
    return body


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_lookup_matches_reference(db_path, oracle_device, case):
    assert call(store(db_path), case) == expected(case)


def test_goldens_cover_the_edge_cases():
    by = {(c["method"], c["tenant"], c["scan"], c.get("node_id")): c["expected"] for c in CASES}
    s2 = by[("node_context", "", "kat-a", "server:s2")]
    assert ["server:s2", "server:s2"] in [[e["source"], e["target"]] for e in s2["edges_out"]]        # the bidirectional self loop
    tool = by[("node_context", "", "kat-a", "tool:t")]
    assert sum(e["source"] == "agent:a" for e in tool["edges_in"]) == 3                                 # three relationships, one pair
    assert any(e["source"] == "runtime:ghost2" for e in tool["edges_in"])                               # a row whose source is not a node
    assert by[("node_context", "", "kat-a", "tool:lonely")]["edges_out"] == []
    # no golden walk meets the SQLite store's caps: its impact is the reference engine's, dangling rows included
    assert all(c["expected"]["impact"] == c["impact_engine"] for c in CASES if c["method"] == "node_context" and c["expected"])
    assert "runtime:ghost2" in by[("node_context", "", "kat-a", "tool:t")]["impact"]["affected_nodes"]
    stats = by[("snapshot_stats", "", "kat-a", None)]
    assert stats["relationship_types"]["custom_rel"] == 1 and "URGENT" in stats["severity_counts"]


def test_more_ids_than_sqlite_variables(db_path, oracle_device):
    """The reference binds two parameters per id; this store answers any number of ids."""
    ids = {f"missing:{i}" for i in range(40_000)} | {"server:s1"}
    got = store(db_path).edges_for_node_ids(tenant_id="", scan_id="kat-a", node_ids=ids)
    want = next(c for c in CASES if c["method"] == "edges_for_node_ids" and c["scan"] == "kat-a" and len(c["node_ids"]) == 10)["expected"]
    assert [e.to_dict() for e in got] == [e for e in want if "server:s1" in (e["source"], e["target"])]


def test_sql_audit_warm_calls_are_keyed(db_path, oracle_device, monkeypatch):
    """A warm call sends SQLite only keyed hydration statements, and no ``graph_edges`` read without a key predicate."""
    statements: list[str] = []
    real_connect = lookup.sqlite3.connect

    def traced(*a, **k):
        conn = real_connect(*a, **k)
        conn.set_trace_callback(statements.append)
        return conn

    monkeypatch.setattr(sqlite3, "connect", traced)
    s = store(db_path)

    def requests():
        s.nodes_by_ids(tenant_id="lookup", scan_id="est40", node_ids={"agent:agent-00007", "nope"})
        s.edges_for_node_ids(tenant_id="lookup", scan_id="est40", node_ids={"agent:agent-00007"})
        s.node_context(tenant_id="", scan_id="kat-a", node_id="tool:t")
        s.edges_for_node_ids(tenant_id="", scan_id="kat-a", node_ids={"runtime:ghost", "server:s2"})
        s.snapshot_stats(tenant_id="", scan_id="kat-a")

    requests()
    assert any("row_number()" in q for q in statements)          # the cold call's one query per scan for the rows the loader leaves out
    statements.clear()
    requests()
    assert statements
    for q in statements:
        assert "graph_snapshots" in q or " IN (" in q, q
        if "graph_edges" in q:
            assert "(source_id, target_id, relationship) IN (VALUES" in q, q
        if "graph_nodes" in q:
            assert "AND id IN (" in q, q


def test_without_sqlite_inner_store_delegates(tmp_path):
    calls = []

    def rec(name):
        return lambda **kw: calls.append((name, kw)) or name

    inner = SimpleNamespace(**{m: rec(m) for m in ("nodes_by_ids", "edges_for_node_ids", "node_context", "snapshot_stats")})
    s = B200GraphStore(inner)
    assert s.nodes_by_ids(tenant_id="t", scan_id="x", node_ids={"a"}) == "nodes_by_ids"
    assert s.edges_for_node_ids(tenant_id="t", scan_id="x", node_ids={"a"}) == "edges_for_node_ids"
    assert s.node_context(tenant_id="t", scan_id="x", node_id="a") == "node_context"
    assert s.snapshot_stats(tenant_id="t", scan_id="x") == "snapshot_stats"
    assert calls[1] == ("edges_for_node_ids", {"tenant_id": "t", "scan_id": "x", "node_ids": {"a"}})
    # a SQLite path that does not exist is not SQLite-backed
    inner._db_path = str(tmp_path / "absent.sqlite")
    assert s.snapshot_stats(tenant_id="t") == "snapshot_stats"
    for name in ("nodes_by_ids", "edges_for_node_ids"):
        with pytest.raises(B200UnsupportedOperationError):
            getattr(B200GraphStore(), name)(node_ids={"a"})
    with pytest.raises(B200UnsupportedOperationError):
        B200GraphStore().node_context(node_id="a")
    with pytest.raises(B200UnsupportedOperationError):
        B200GraphStore().snapshot_stats()


def test_filtered_stats_go_to_the_inner_store(db_path):
    calls = []
    inner = SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None,
                            snapshot_stats=lambda **kw: calls.append(kw) or {"filtered": True})
    s = B200GraphStore(inner)
    assert s.snapshot_stats(tenant_id="", scan_id="kat-a", entity_types={"agent"}) == {"filtered": True}
    assert s.snapshot_stats(tenant_id="", scan_id="kat-a", min_severity_rank=3) == {"filtered": True}
    assert calls == [{"tenant_id": "", "scan_id": "kat-a", "entity_types": {"agent"}, "min_severity_rank": 0},
                     {"tenant_id": "", "scan_id": "kat-a", "entity_types": None, "min_severity_rank": 3}]


def test_oracle_context_order_and_incident_set():
    """The oracle's rules on a hand-made CSR: a self loop and an edge inside the set count once; the context sorts by rank."""
    g = UnifiedGraph()
    from agent_bom_b200.graph.model import UnifiedEdge, UnifiedNode

    for nid in ("b", "a", "c"):
        g.add_node(UnifiedNode(id=nid, entity_type="agent", label=nid))
    for s_, t_, r in (("b", "a", "uses"), ("a", "a", "uses"), ("c", "b", "uses"), ("b", "a", "invoked"), ("a", "c", "uses")):
        g.add_edge(UnifiedEdge(s_, t_, r, direction="bidirectional" if s_ == "c" else "directed"))
    o = LookupOracle(g.csr)
    idx = g.csr.idx
    assert o.incident_edges([idx("a"), idx("b")]).tolist() == [0, 1, 2, 3, 4]
    assert o.incident_edges([idx("c")]).tolist() == [2, 4]
    erel, names = lookup.relationship_slots(g)
    o.build_lookup_table(3, [0, 0, 0], erel)
    keys = [(g.csr.node_ids[g.csr.src[e]], g.csr.node_ids[g.csr.dst[e]], names[erel[e]]) for e in o.context_edges(idx("a")).tolist()]
    assert keys == sorted(keys) and len(keys) == 4
