"""Edge lifecycle reads on the host: the Python oracle against the reference's goldens (oracle/make_lifecycle_golden.py); the whole
``active_edges_at`` and ``changed_edges_between_scans`` store pipelines with the oracle standing in for the device; the dictionary
rank and bisect against SQLite's own ``<=`` and ``>``; the snapshot fingerprint under saves, re-saves and deletion; delegation and
refusal without a SQLite inner store.
"""

from __future__ import annotations

import gzip
import json
import random
import shutil
import sqlite3
from pathlib import Path
from types import SimpleNamespace

import pytest
from oracle import lifecycle_oracle
from oracle.lifecycle_oracle import HistoryOracle, SharedDeltaOracle

from agent_bom_b200.graph import lifecycle
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.store import B200GraphStore, B200UnsupportedOperationError

GOLD = Path(__file__).parent / "golden"
EXPECTED = json.loads(gzip.decompress((GOLD / "lifecycle" / "expected.json.gz").read_bytes()))
ACTIVE, CHANGES = EXPECTED["active"], EXPECTED["changes"]
ACTIVE_IDS = [f"{c['tenant'].strip() or '-'}@{c['at'] or 'blank'}" for c in ACTIVE]
CHANGE_IDS = [f"{c['db']}:{c['tenant'].strip() or '-'}:{c['old'] or 'blank'}>{c['new'] or 'blank'}" for c in CHANGES]


def plain(body):
    return json.loads(json.dumps(body))


@pytest.fixture(scope="module")
def dbs(tmp_path_factory) -> dict[str, Path]:
    root = tmp_path_factory.mktemp("lifecycle")
    out = {}
    for name, src in (("lifecycle", GOLD / "lifecycle" / "graph.sqlite.gz"), ("delta", GOLD / "delta" / "graph.sqlite.gz")):
        out[name] = root / f"{name}.sqlite"
        out[name].write_bytes(gzip.decompress(src.read_bytes()))
    return out


@pytest.fixture
def oracle_device(monkeypatch):
    """Every device call answered by the oracles: the tenant history and the diff with its shared pairs."""

    def device_graph(self):
        if self._dg is None:
            self._dg = SharedDeltaOracle(self.csr)
        return self._dg

    monkeypatch.setattr(UnifiedGraph, "device_graph", property(device_graph))
    monkeypatch.setattr(lifecycle, "make_history", lambda codes, n_ids, n_rels, device, id_limit: HistoryOracle(
        codes["src"], codes["tgt"], codes["rel"], codes["created"], codes["valid_from"], codes["valid_to"], n_ids, n_rels, id_limit=id_limit))


def store(db_path) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


def ro(db_path) -> sqlite3.Connection:
    return sqlite3.connect(f"file:{db_path}?mode=ro", uri=True)


@pytest.mark.parametrize("case", ACTIVE, ids=ACTIVE_IDS)
def test_oracle_active_matches_reference(dbs, case):
    conn = ro(dbs["lifecycle"])
    try:
        assert plain(lifecycle_oracle.active_edges_at(conn, case["at"], case["tenant"])) == case["edges"]
    finally:
        conn.close()


@pytest.mark.parametrize("case", CHANGES, ids=CHANGE_IDS)
def test_oracle_changes_match_reference(dbs, case):
    conn = ro(dbs[case["db"]])
    try:
        assert plain(lifecycle_oracle.changed_edges_between_scans(conn, case["old"], case["new"], case["tenant"])) == case["body"]
    finally:
        conn.close()


def test_store_active_matches_reference(dbs, oracle_device):
    s = store(dbs["lifecycle"])
    for case in ACTIVE:
        assert plain(s.active_edges_at(case["at"], tenant_id=case["tenant"])) == case["edges"], (case["tenant"], case["at"])
    assert len(s._histories) <= s._histories.max_histories


@pytest.mark.parametrize("case", CHANGES, ids=CHANGE_IDS)
def test_store_changes_match_reference(dbs, oracle_device, case):
    body = store(dbs[case["db"]]).changed_edges_between_scans(case["old"], case["new"], tenant_id=case["tenant"])
    assert plain(body) == case["body"]


def test_goldens_cover_the_cases():
    """The fixture holds what the generator claims: versions that close and reopen, every kind of `at`, and an answer per tenant."""
    by = {(c["tenant"], c["at"]): c["edges"] for c in ACTIVE}
    assert {"", "2026", "z", "\U0001F600"} <= {at for _, at in by}
    assert by[("", "2025-01-01T00:00:00+00:00")] == [] and by[("nobody", "2027-01-01T00:00:00+00:00")] == []
    assert by[("empty", "2027-01-01T00:00:00+00:00")] == []            # rows without a snapshot row are not joined
    every = [e for edges in by.values() for e in edges]
    assert any(e["valid_to"] == "" for e in every) and any(e["valid_to"] is None for e in every) and any(e["valid_to"] for e in every)
    def keys(at):
        return {(e["source_id"], e["target_id"]) for e in by[("", at)]}

    assert ("agent:b", "server:s1") in keys("2026-03-01T12:00:00+00:00")           # closed by s2 ...
    assert ("agent:b", "server:s1") not in keys("2026-03-02T12:00:00+00:00")
    assert ("agent:b", "server:s1") in keys("2026-03-03T12:00:00+00:00")           # ... and back in s3
    assert any(c["body"]["summary"]["changed"] for c in CHANGES if c["db"] == "lifecycle")


def test_rank_predicate_equals_sqlite():
    """rank(s) < bisect_right(dict, at) is SQLite's s <= at, and rank(s) >= it is s > at, for any strings, '' included."""
    rng = random.Random(5)
    alphabet = ["", "0", "1", "2", "9", "-", ":", "T", "Z", "a", "z", "é", "ﬁ", "\U0001F600", "ÿ", "Ā", "\x7f", " "]

    def word():
        return "".join(rng.choice(alphabet) for _ in range(rng.randrange(0, 5)))

    conn = sqlite3.connect(":memory:")
    try:
        for _ in range(40):
            stamps = sorted({word() for _ in range(rng.randrange(1, 30))})
            rank = {s: i for i, s in enumerate(stamps)}
            for at in [word() for _ in range(20)] + stamps:
                r = lifecycle.timestamp_rank(stamps, at)
                for s in stamps:
                    le, gt = conn.execute("SELECT ? <= ?, ? > ?", (s, at, s, at)).fetchone()
                    assert (rank[s] < r) == bool(le) and (rank[s] >= r) == bool(gt), (s, at)
    finally:
        conn.close()


def _save(conn, tenant: str, scan: str, created: str, keys, previous: str | None) -> None:
    """A save in the order the SQLite store writes one: edge rows, the close-out of the previous scan's dropped edges, then the
    snapshot row (INSERT OR REPLACE)."""
    conn.executemany("INSERT OR REPLACE INTO graph_edges (source_id, target_id, relationship, first_seen, last_seen, valid_from, scan_id, tenant_id) "
                     "VALUES (?, ?, ?, ?, ?, ?, ?, ?)", [(s, t, r, created, created, created, scan, tenant) for s, t, r in keys])
    if previous:
        have = {tuple(k) for k in keys}
        for s, t, r in conn.execute("SELECT source_id, target_id, relationship FROM graph_edges WHERE tenant_id = ? AND scan_id = ?",
                                    (tenant, previous)).fetchall():
            if (s, t, r) not in have:
                conn.execute("UPDATE graph_edges SET valid_to = COALESCE(valid_to, ?) WHERE tenant_id = ? AND scan_id = ? AND source_id = ? AND "
                             "target_id = ? AND relationship = ?", (created, tenant, previous, s, t, r))
    conn.execute("INSERT OR REPLACE INTO graph_snapshots VALUES (?, ?, ?, ?, ?, ?)", (scan, tenant, created, 0, len(keys), "{}"))
    conn.commit()


def test_fingerprint_changes_on_save_resave_and_delete(dbs, tmp_path):
    path = tmp_path / "graph.sqlite"
    shutil.copy(dbs["lifecycle"], path)
    conn = sqlite3.connect(str(path))
    try:
        seen = [lifecycle.fingerprint(conn, "t2")]
        _save(conn, "t2", "e", "2026-03-07T00:00:00+00:00", [("agent:a", "server:s1", "uses")], "d")
        seen.append(lifecycle.fingerprint(conn, "t2"))
        _save(conn, "t2", "e", "2026-03-07T00:00:00+00:00", [("agent:a", "server:s1", "uses")], "d")     # same scan id, same created_at
        seen.append(lifecycle.fingerprint(conn, "t2"))
        for table in ("graph_edges", "graph_snapshots"):
            conn.execute(f"DELETE FROM {table} WHERE tenant_id = 't2'")
        conn.commit()
        seen.append(lifecycle.fingerprint(conn, "t2"))
        assert len(set(seen)) == 4 and seen[-1] == ()
        assert lifecycle.fingerprint(conn, "default") == lifecycle.fingerprint(ro(dbs["lifecycle"]), "default")
    finally:
        conn.close()


def test_store_sees_a_new_save(dbs, oracle_device, tmp_path):
    path = tmp_path / "graph.sqlite"
    shutil.copy(dbs["lifecycle"], path)
    s = store(path)
    at = "2027-01-01T00:00:00+00:00"
    first = s.active_edges_at(at, tenant_id="t2")
    writer = sqlite3.connect(str(path))
    try:
        _save(writer, "t2", "e", "2026-03-07T00:00:00+00:00", [("agent:a", "server:s1", "uses"), ("agent:new", "tool:t", "uses")], "d")
    finally:
        writer.close()
    second = s.active_edges_at(at, tenant_id="t2")
    assert second != first
    assert plain(second) == plain(lifecycle_oracle.active_edges_at(ro(path), at, "t2"))


def test_not_a_string(dbs, oracle_device):
    s = store(dbs["lifecycle"])
    assert s.active_edges_at(None) == [] and s.active_edges_at(20260301) == []
    with pytest.raises(TypeError):
        s.active_edges_at(b"2026")


def test_delegates_without_sqlite_and_refuses_without_inner():
    calls = []
    inner = SimpleNamespace(active_edges_at=lambda at, tenant_id="": calls.append(("active", at, tenant_id)) or ["a"],
                            changed_edges_between_scans=lambda a, b, tenant_id="": calls.append(("changes", a, b, tenant_id)) or {"x": 1})
    s = B200GraphStore(inner)
    assert s.active_edges_at("2026", tenant_id="t") == ["a"]
    assert s.changed_edges_between_scans("a", "b", tenant_id="t") == {"x": 1}
    assert calls == [("active", "2026", "t"), ("changes", "a", "b", "t")]
    bare = B200GraphStore()
    with pytest.raises(B200UnsupportedOperationError):
        bare.active_edges_at("2026")
    with pytest.raises(B200UnsupportedOperationError):
        bare.changed_edges_between_scans("a", "b")
