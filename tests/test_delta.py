"""Snapshot diff on the host: the whole ``B200GraphStore.diff_snapshots`` pipeline, with the Python oracle standing in for the
device, against the reference's ``diff_snapshots`` on every golden pair (oracle/make_delta_golden.py); the SQL candidate queries
and the JSON check; the blank-scan and tenant rules; delegation without a SQLite inner store; and refusal without a device.
"""

from __future__ import annotations

import gzip
import json
from pathlib import Path
from types import SimpleNamespace

import pytest
from oracle.delta_oracle import DeltaOracle

from agent_bom_b200 import _lib
from agent_bom_b200.graph import delta
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.store import B200GraphStore, B200UnsupportedOperationError

GOLD = Path(__file__).parent / "golden" / "delta"
CASES = json.loads(gzip.decompress((GOLD / "expected.json.gz").read_bytes()))
IDS = [f"{c['tenant'].strip() or '-'}:{c['old'] or 'blank'}>{c['new'] or 'blank'}" for c in CASES]


@pytest.fixture(scope="module")
def db_path(tmp_path_factory) -> Path:
    path = tmp_path_factory.mktemp("delta") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.fixture
def oracle_device(monkeypatch):
    """Every graph's device calls answered by the oracle."""

    def device_graph(self):
        if self._dg is None:
            self._dg = DeltaOracle(self.csr)
        return self._dg

    monkeypatch.setattr(UnifiedGraph, "device_graph", property(device_graph))


def store(db_path) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


def plain(body):
    return json.loads(json.dumps(body))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_diff_matches_reference(db_path, oracle_device, case):
    body = store(db_path).diff_snapshots(case["old"], case["new"], tenant_id=case["tenant"])
    assert plain(body) == case["diff"]


def test_kat_covers_each_change(db_path):
    """The hand-made pair exercises what it claims: every kind of node and edge change, and a key-order-only evidence edit."""
    kat = next(c for c in CASES if (c["tenant"], c["old"], c["new"]) == ("", "kat-a", "kat-b"))["diff"]
    assert set(kat["nodes_changed"]) == {"pkg:p1", "vuln:CVE-1", "custom:x", "agent:ﬁ"}
    changed = {(e["before"]["source_id"], e["before"]["target_id"]): e for e in kat["edges_changed"]}
    assert ("server:s1", "pkg:p1") not in changed
    assert {("server:s1", "server:s2"), ("server:s2", "tool:t"), ("agent:é", "server:s2"), ("agent:\U0001F600", "server:s2"), ("agent:ﬁ", "server:s2"),
            ("server:s2", "pkg:neg"), ("agent:é", "server:s1"), ("server:s1", "pkg:p2")} <= set(changed)
    assert ["agent:c", "runtime:ghost3", "delegated_to"] in kat["edges_added"]
    assert ["runtime:ghost2", "tool:t", "accessed"] not in kat["edges_removed"]


def test_sql_candidates_and_json_check(db_path):
    import sqlite3

    conn = sqlite3.connect(str(db_path))
    try:
        cand = delta.rich_edge_candidates(conn, "default", "kat-a", "kat-b")
        assert ("server:s1", "pkg:p1", "depends_on") in cand          # the stored text differs ...
        assert ("server:s1", "server:s2", "shares_server") in cand    # direction string
        assert ("server:s2", "tool:t", "provides_tool") in cand       # weight
        nodes = delta.rich_node_candidates(conn, "default", "kat-a", "kat-b")
        assert nodes == ["agent:ﬁ"]
        assert delta.unloaded_edge_keys(conn, "default", "kat-a") == {("agent:a", "runtime:ghost", "invoked"), ("runtime:ghost2", "tool:t", "accessed")}
    finally:
        conn.close()
    conn = sqlite3.connect(str(db_path))
    conn.row_factory = sqlite3.Row
    try:
        before = delta._edge_rows(conn, "default", "kat-a", [("server:s1", "pkg:p1", "depends_on")])
        after = delta._edge_rows(conn, "default", "kat-b", [("server:s1", "pkg:p1", "depends_on")])
    finally:
        conn.close()
    k = ("server:s1", "pkg:p1", "depends_on")
    assert delta.edge_fingerprint(before[k]) == delta.edge_fingerprint(after[k])   # ... but decodes equal: not a change


def test_blank_scan_is_empty_not_latest(db_path, oracle_device):
    s = store(db_path)
    s.latest_snapshot_id = lambda **_: "est40-b"          # a latest snapshot exists; a blank id must still be empty
    body = s.diff_snapshots("", "kat-z", tenant_id="")
    assert [n["id"] for n in body["nodes_added"]] == ["zzz:1", "zzz:2"] and not body["nodes_removed"]


def test_tenant_is_normalised(db_path, oracle_device):
    s = store(db_path)
    a = s.diff_snapshots("kat-a", "kat-b", tenant_id="  ")
    b = s.diff_snapshots("kat-a", "kat-b", tenant_id="default")
    assert plain(a) == plain(b) and a["nodes_changed"]
    assert not any(s.diff_snapshots("kat-a", "kat-b", tenant_id="delta").values())


def test_without_sqlite_inner_store_delegates():
    calls = []
    inner = SimpleNamespace(diff_snapshots=lambda a, b, *, tenant_id="": calls.append((a, b, tenant_id)) or {"inner": True})
    assert B200GraphStore(inner).diff_snapshots("x", "y", tenant_id="t") == {"inner": True}
    assert calls == [("x", "y", "t")]
    with pytest.raises(B200UnsupportedOperationError):
        B200GraphStore().diff_snapshots("x", "y")


def test_snapshot_diff_needs_a_database():
    with pytest.raises(ValueError, match="db_path"):
        delta.snapshot_diff(UnifiedGraph(), UnifiedGraph())


def test_refuses_without_device(db_path):
    if _lib.load().abb_device_count() > 0:
        pytest.skip("a device is present")
    with pytest.raises(_lib.EngineUnavailable):
        store(db_path).diff_snapshots("kat-a", "kat-b")


# ── compute_delta_alerts ──
ALERT_CASES = json.loads(gzip.decompress((GOLD / "alerts.json.gz").read_bytes()))
ALERT_IDS = [f"{c['old'] or 'none'}>{c['new']}" for c in ALERT_CASES]
UNORDERED = ("new_vulnerability", "new_misconfiguration")


def normalise_alerts(alerts):
    """The reference emits new findings and the removed-agent list in Python set order: compare those order-free, the rest exactly."""
    alerts = json.loads(json.dumps(alerts))
    out, i = [], 0
    while i < len(alerts):
        kind = alerts[i]["type"]
        if kind in UNORDERED:
            j = i
            while j < len(alerts) and alerts[j]["type"] == kind:
                j += 1
            out.append(sorted(json.dumps(a, sort_keys=True) for a in alerts[i:j]))
            i = j
            continue
        a = alerts[i]
        if kind == "agent_removed":
            a["node_ids"] = sorted(a["node_ids"])
            a["details"]["node_ids"] = sorted(a["details"]["node_ids"])
            a["event_relationships"]["targets"] = sorted(a["event_relationships"]["targets"], key=lambda t: t["id"])
        out.append(a)
        i += 1
    return out


def alert_graphs(db_path, case):
    from agent_bom_b200.graph.snapshot import load_snapshot

    old = load_snapshot(db_path, tenant_id=case["tenant"], scan_id=case["old"]) if case["old"] else None
    return old, load_snapshot(db_path, tenant_id=case["tenant"], scan_id=case["new"])


@pytest.mark.parametrize("case", ALERT_CASES, ids=ALERT_IDS)
def test_delta_alerts_match_reference(db_path, oracle_device, case):
    from agent_bom_b200.graph import compute_delta_alerts

    got = compute_delta_alerts(*alert_graphs(db_path, case))
    assert normalise_alerts(got) == normalise_alerts(case["alerts"])
    for kind in ("new_vulnerability", "new_misconfiguration"):      # id order
        ids = [a["node_ids"][0] for a in got if a["type"] == kind]
        assert ids == sorted(ids)


def test_alert_goldens_cover_each_block():
    kinds = {a["type"] for c in ALERT_CASES for a in c["alerts"]}
    assert kinds == {"new_vulnerability", "new_misconfiguration", "new_attack_path", "new_interaction_risk", "agent_removed"}
    assert any(c["old"] is None for c in ALERT_CASES)


def test_event_refs_redact_like_the_reference():
    from agent_bom_b200.graph.alerts import event_ref, sanitize_payload

    assert sanitize_payload("https://u:p@example.com/b?q=1", key="label") == "https://example.com/b"
    assert sanitize_payload("/etc/passwd", key="path") == "<path:passwd>"
    assert sanitize_payload("x", key="api_key") == "***REDACTED***"
    assert sanitize_payload("ghp_" + "a" * 36) == "***REDACTED***"
    assert event_ref(ref_type="agent", ref_id="", name="n") is None
    assert event_ref(ref_type="agent", ref_id="agent:a", name="a", role="r", attributes={"severity": "", "risk_score": 0.0, "status": "active"}) == {
        "type": "agent", "id": "agent:a", "name": "a", "role": "r", "attributes": {"risk_score": 0.0, "status": "active"}}
