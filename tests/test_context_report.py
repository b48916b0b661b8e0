"""Context-graph report (agent_bom_b200.context_report), everything that runs without a device, against the unmodified
reference's answers in tests/golden/context/report.json.xz (oracle/make_context_report_golden.py): interaction risks on every
golden graph, report assembly from the golden's own paths, the builder's structure before scoring, and the CPU oracle's
restatement of the path enrichment."""

from __future__ import annotations

import json

import pytest
from context_report_golden import BUILT, DOCS, IDS, assert_body, golden_paths, graph_doc, injected, rebuild

from agent_bom_b200 import context_report as cr


def _risk_dicts(risks):
    return [{"pattern": r.pattern, "agents": r.agents, "risk_score": r.risk_score, "description": r.description, "owasp_agentic_tag": r.owasp_agentic_tag}
            for r in risks]


@pytest.mark.parametrize("doc", DOCS, ids=IDS)
def test_interaction_risks_match_the_reference(doc):
    g = rebuild(doc)
    errors = {r["error"] for r in doc["reports"] if "error" in r}
    if doc["body"] is None:              # every body raised: the risks do too, with the reference's exception
        (error,) = errors
        with pytest.raises(Exception) as info:
            cr.compute_interaction_risks(g)
        assert f"{type(info.value).__name__}: {info.value}" == error
        return
    assert json.dumps(_risk_dicts(cr.compute_interaction_risks(g))) == doc["body"]["interaction_risks"]


@pytest.mark.parametrize("doc", DOCS, ids=IDS)
def test_report_assembly_from_the_golden_paths(doc):
    """to_serializable over the reference's own paths and this package's risks gives the reference's bodies."""
    if doc["body"] is None:
        pytest.skip("every body of this graph raises")
    g = rebuild(doc)
    risks = cr.compute_interaction_risks(g)
    for report in doc["reports"]:
        assert_body(doc, report, cr.to_serializable(g, golden_paths(report), risks))


@pytest.mark.parametrize("doc", DOCS, ids=IDS)
def test_absent_agent_needs_no_device(doc):
    """An agent without a node gets an empty path list; nothing reaches the device."""
    if doc["body"] is None:
        pytest.skip("every body of this graph raises")
    g = rebuild(doc)
    report = next(r for r in doc["reports"] if r["agent"] == "no-such-agent")
    assert_body(doc, report, cr.context_graph_report(g, agent="no-such-agent", max_depth=4))


@pytest.mark.parametrize("doc", BUILT, ids=[d["name"] for d in BUILT])
def test_builder_structure_before_scoring(doc, monkeypatch):
    """The builder's loops alone (scorer stubbed out): the reference's graph without its effective-reach annotations."""
    from agent_bom_b200 import effective_reach

    calls = []
    monkeypatch.setattr(effective_reach, "annotate_graph", lambda graph, device=0: calls.append(graph))
    g = cr.build_context_graph(json.loads(json.dumps(doc["input"]["agents"])), json.loads(json.dumps(doc["input"]["blast"])), **injected(doc))
    assert calls == [g]
    want = json.loads(json.dumps(doc["graph"]))
    for _nid, _kind, _label, meta in want["nodes"]:
        meta.pop("effective_reach", None)
    for entry in want["edges"] + [e for _nid, row in want["adjacency"] for e in row]:
        entry[4].pop("effective_reach_score", None)
    assert json.dumps(graph_doc(g)) == json.dumps(want)


def test_builder_defaults_and_untrusted_text():
    """Without injected rules: no capabilities, graph.builder's credential rule; descriptions are blanked, prefixed and cut."""
    from agent_bom_b200 import effective_reach

    saved = effective_reach.annotate_graph
    effective_reach.annotate_graph = lambda graph, device=0: None
    try:
        g = cr.build_context_graph([{"name": "a", "mcp_servers": [{"name": "s", "env": {"API_TOKEN": "x", "HOME": "/"},
                                                                   "tools": [{"name": "t", "description": "a\nb c" + "x" * 2000, "capabilities": ["execute"]}]}]}], [])
    finally:
        effective_reach.annotate_graph = saved
    assert list(g.nodes) == ["agent:a", "server:a:s", "cred:API_TOKEN", "tool:server:a:s:t"]
    meta = g.nodes["tool:server:a:s:t"].metadata
    assert meta["capabilities"] == [] and meta["description"] == "[UNTRUSTED MCP METADATA] a b c" + "x" * 995
    assert [e.weight for e in g.edges] == [1.0, 2.0, 1.0]


@pytest.mark.parametrize("doc", [d for d in DOCS if d["body"] is not None], ids=[d["name"] for d in DOCS if d["body"] is not None])
def test_oracle_enrichment_matches_the_goldens(doc):
    """oracle/context_report_oracle.describe (label -> servers index) restates what the reference folds into each path."""
    from oracle import context_report_oracle as oracle

    g = rebuild(doc)
    index = oracle.servers_by_label(g)
    n = 0
    for report in doc["reports"]:
        for p in json.loads(report.get("lateral_paths", "[]")):
            creds, tools, vulns, execute, sev = oracle.describe(g, p["hops"], p["edges"], index)
            assert (creds, tools, vulns) == (p["credential_exposure"], p["tool_exposure"], p["vuln_ids"])
            assert round(min(sev + len(creds) * 0.3 + execute * 0.2, 10.0), 1) == p["composite_risk"]
            n += 1
    assert n or all(json.loads(r["stats"])["lateral_path_count"] == 0 for r in doc["reports"])
