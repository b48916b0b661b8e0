"""CPU: OCSF events of findings without enrichment equal the reference's on every record family (adopted reference records, the
light builder's records and columns, SQLite snapshots), and the oracle's finding context reproduces the reference's
``graph_context`` on every golden graph.  Fixture: tests/golden/ocsf/events.json.gz (oracle/make_ocsf_golden.py)."""

from __future__ import annotations

import time

import pytest

import ocsf_golden as og

GRAPH_CASES = og.graph_cases()
BUILDER_CASES = og.builder_cases()
SNAPSHOT_CASES = og.snapshot_cases()


def _window():
    return int(time.time() * 1000)


def check_plain(graph, case):
    for v in og.versions():
        t0 = _window()
        got = graph.to_ocsf_events(v, enrich_neighbors=False)
        t1 = _window()
        assert og.without_time(got, t0, t1) == og.events(case, v, False)


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_plain_events_adopted(case):
    check_plain(og.adopted(case), case)


def _without_data(evs):
    out = []
    for ev in evs:
        ev = dict(ev)
        ev["resources"] = [{k: v for k, v in r.items() if k != "data"} for r in ev["resources"]]
        out.append(ev)
    return out


@pytest.mark.parametrize("columnar", [False, True], ids=["records", "columnar"])
@pytest.mark.parametrize("case", BUILDER_CASES, ids=[c["name"] for c in BUILDER_CASES])
def test_plain_events_light_builder(case, columnar):
    """Every field equals the reference's except ``resources[0].data``: the light builder does not record the reference builder's
    bookkeeping attributes (``canonical_id``, ``is_kev``), so there ``data`` is checked against the light graph's own attributes."""
    g = og.built(case, columnar)
    for v in og.versions():
        t0 = _window()
        got = og.without_time(g.to_ocsf_events(v, enrich_neighbors=False), t0, _window())
        assert _without_data(got) == _without_data(og.events(case, v, False))
        if columnar:      # read from the columns: no record was synthesised
            assert not g.nodes._cache
        else:
            for ev in got:
                attrs = g.nodes[ev["resources"][0]["uid"]].attributes
                assert ev["resources"][0]["data"] == {k: x for k, x in attrs.items() if isinstance(x, (str, int, float, bool))}


@pytest.mark.parametrize("case", SNAPSHOT_CASES, ids=[c["name"] for c in SNAPSHOT_CASES])
def test_plain_events_snapshot(case, tmp_path):
    check_plain(og.loaded(case, og.snapshot_db(tmp_path)), case)


def test_plain_events_batching_and_pages():
    from agent_bom_b200.graph import iter_ocsf_events

    case = next(c for c in GRAPH_CASES if c["name"] == "estate_dense_40")
    g = og.adopted(case)
    want = og.events(case, "0.0.0", False)
    for bs in (1, 7, 65536):
        assert og.without_time(list(iter_ocsf_events(g, enrich_neighbors=False, batch_size=bs))) == want
    assert og.without_time(list(iter_ocsf_events(g, enrich_neighbors=False, offset=5, limit=9))) == want[5:14]
    assert list(iter_ocsf_events(g, enrich_neighbors=False, offset=len(want))) == []
    with pytest.raises(ValueError):
        list(iter_ocsf_events(g, batch_size=0))


def test_event_rules_on_light_records():
    """Classification derived from kind and severity string; stored non-zero values win; data keeps scalar attributes only."""
    from agent_bom_b200.graph import UnifiedNode, ocsf_event

    n = UnifiedNode(id="v", entity_type="vulnerability", label="", severity="HIGH", attributes={"a": 1, "b": [1], "c": None, "d": {"x": 1}, "e": True})
    ev = ocsf_event(n, "1.0")
    assert (ev["class_uid"], ev["category_uid"], ev["type_uid"], ev["severity_id"], ev["severity"]) == (2001, 2, 200101, 4, "High")
    assert ev["resources"][0]["data"] == {"a": 1, "e": True} and ev["finding_info"]["title"] == "" and "compliance" not in ev
    assert ev["message"] == "vulnerability:" and isinstance(ev["time"], int)
    m = UnifiedNode(id="m", entity_type="misconfiguration", label="M", severity="bogus", compliance_tags=["CIS"])
    ev = ocsf_event(m)
    assert (ev["class_uid"], ev["severity_id"], ev["severity"]) == (2003, 0, "Unknown") and "finding_info" not in ev
    assert ev["compliance"] == {"standards": ["CIS"]}


def _oracle_contexts(graph):
    from agent_bom_b200.graph.ocsf import label_column
    from oracle import ocsf_oracle

    ograph, findings = og.oracle_of(graph)
    ctx = ocsf_oracle.finding_context(ograph, findings)
    labels = label_column(graph)
    return [og.oracle_context(graph, ctx, q, labels) for q in range(len(findings))]


def _assert_contexts(got, case):
    for v in og.versions():
        want = [ev["graph_context"] for ev in og.events(case, v, True)]
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert a == b      # dict equality: blast_by_type's key order is not pinned (the reference iterates a set)


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_oracle_context_matches_reference(case):
    _assert_contexts(_oracle_contexts(og.adopted(case)), case)


@pytest.mark.parametrize("columnar", [False, True], ids=["records", "columnar"])
@pytest.mark.parametrize("case", BUILDER_CASES, ids=[c["name"] for c in BUILDER_CASES])
def test_oracle_context_matches_reference_light_builder(case, columnar):
    g = og.built(case, columnar)
    _assert_contexts(_oracle_contexts(g), case)
    if columnar:      # labels come from the label column
        assert not g.nodes._cache


@pytest.mark.parametrize("case", SNAPSHOT_CASES, ids=[c["name"] for c in SNAPSHOT_CASES])
def test_oracle_context_matches_reference_snapshot(case, tmp_path):
    _assert_contexts(_oracle_contexts(og.loaded(case, og.snapshot_db(tmp_path))), case)


def test_kat_ocsf_covers_the_edge_cases():
    """The edge-case graph really has the shapes the export must get right."""
    case = next(c for c in GRAPH_CASES if c["name"] == "kat_ocsf")
    ctx = {ev["resources"][0]["uid"]: ev["graph_context"] for ev in og.events(case, "0.0.0", True)}
    hub = ctx["vuln:hub"]
    assert hub["affected_agents"] == ["agent-a", "agent-a"] and hub["affected_packages"] == ["left-pad", "left-pad"] and hub["affected_servers"] == [""]
    assert sum(e["target"] == "vuln:wide" for e in case["edges"]) > 64           # a reverse row the device hands to a whole warp
    assert len(sum((ctx["vuln:wide"][k] for k in ("affected_agents", "affected_servers", "affected_packages", "exposed_credentials")), [])) == 60
    assert ctx["vuln:deep"]["blast_radius"] == 4 and ctx["vuln:alone"]["blast_radius"] == 0
    stored = next(ev for ev in og.events(case, "0.0.0", True) if ev["resources"][0]["uid"] == "vuln:stored")
    assert (stored["class_uid"], stored["category_uid"], stored["type_uid"], stored["severity_id"]) == (2003, 7, 123456, 5)
