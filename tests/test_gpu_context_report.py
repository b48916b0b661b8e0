"""Context-graph report on the device: the builder with the device scorer equals the reference's graph on every golden input
(annotations included), every report body equals the reference's as JSON text, the device path enrichment equals the CPU
oracle on a 4 000-agent fleet with 200-agent shared-server cliques at depths 1-6, a search that exceeds its safety valve
raises instead of returning a partial body, and device memory returns to its level once the graph is gone."""

from __future__ import annotations

import functools
import gc
import json

import pytest
from context_report_golden import BUILT, DOCS, IDS, assert_body, graph_doc, injected, rebuild

from agent_bom_b200 import context_report as cr
from agent_bom_b200 import lateral

pytestmark = pytest.mark.gpu


def _built(doc):
    if doc["input"] is None:
        return rebuild(doc)
    return cr.build_context_graph(json.loads(json.dumps(doc["input"]["agents"])), json.loads(json.dumps(doc["input"]["blast"])), **injected(doc))


@pytest.mark.parametrize("doc", BUILT, ids=[d["name"] for d in BUILT])
def test_builder_equals_the_reference_graph(doc):
    assert json.dumps(graph_doc(_built(doc))) == json.dumps(doc["graph"])


@pytest.mark.parametrize("doc", DOCS, ids=IDS)
def test_report_bodies_equal_the_reference(doc):
    g = _built(doc)
    for report in doc["reports"]:
        if "error" in report:
            with pytest.raises(Exception) as info:
                cr.context_graph_report(g, agent=report["agent"], max_depth=report["max_depth"])
            assert f"{type(info.value).__name__}: {info.value}" == report["error"]
        else:
            assert_body(doc, report, cr.context_graph_report(g, agent=report["agent"], max_depth=report["max_depth"]))


def _fleet_graph(agents, seed, clique):
    from oracle import context_report_oracle as oracle

    agents_data, blast, classify, is_cred = oracle.fleet(agents, seed, clique=clique, cred_share=0.1)
    return cr.build_context_graph(agents_data, blast, classify_tool=classify, is_credential_key=is_cred)


def test_device_enrichment_matches_the_oracle_on_a_large_fleet():
    """Every 97th agent's paths, enriched on the device, against the oracle's restatement of the reference; all agents searched
    and enriched in one call per depth."""
    from oracle import context_report_oracle as oracle

    g = _fleet_graph(4000, 41, 200)
    index = oracle.servers_by_label(g)
    assert max(len(v) for k, v in index.items() if k.startswith("shared-")) >= 200
    sources = [nid for nid, n in g.nodes.items() if n.kind.value == "agent"]
    assert len(sources) == 4000
    checked = 0
    for depth in range(1, 7):
        got = lateral.find_lateral_paths_many(g, sources, depth)
        raw, _ms = lateral.search_many(g, sources, depth)
        assert [len(x) for x in got] == [len(x) for x in raw]
        for q in range(0, len(sources), 97):
            want = []
            for hops, kinds in raw[q]:
                creds, tools, vulns, execute, sev = oracle.describe(g, hops, kinds, index)
                want.append({"hops": hops, "edges": [k.value for k in kinds], "composite_risk": round(min(sev + len(creds) * 0.3 + execute * 0.2, 10.0), 1),
                             "summary": " → ".join(g.nodes[h].label for h in hops if g.nodes.get(h)), "credential_exposure": creds,
                             "tool_exposure": tools, "vuln_ids": vulns})
            want.sort(key=lambda p: p["composite_risk"], reverse=True)
            have = [{"hops": p.hops, "edges": [k.value for k in p.edges], "composite_risk": p.composite_risk, "summary": p.summary,
                     "credential_exposure": p.credential_exposure, "tool_exposure": p.tool_exposure, "vuln_ids": p.vuln_ids} for p in got[q]]
            assert have == want, (sources[q], depth)
            checked += len(want)
    assert checked > 10_000


def test_enrichment_of_no_paths_and_of_paths_without_surfaces():
    """Zero records, and records whose hops add nothing (agents only, no sharing metadata)."""
    from agent_bom_b200.context_graph import ContextGraph, EdgeKind, GraphEdge, GraphNode, NodeKind

    g = ContextGraph()
    for a in "ab":
        g.add_node(GraphNode(id=f"agent:{a}", kind=NodeKind.AGENT, label=a))
    g.add_edge(GraphEdge(source="agent:a", target="agent:b", kind=EdgeKind.SHARES_SERVER))
    arr, _off, rec, W, _ms = lateral._search_records(g, ["agent:a"], 4, 0)
    off, items, execute, sev, flags, _ems = lateral.enrich_records(g, arr, rec[:0], W)
    assert off.tolist() == [0] and len(items) == len(execute) == len(sev) == len(flags) == 0
    off, items, execute, sev, flags, _ems = lateral.enrich_records(g, arr, rec, W)
    assert off.tolist() == [0, 0] and execute.tolist() == [0] and sev.tolist() == [0.0] and flags.tolist() == [0]
    assert [p.composite_risk for p in lateral.find_lateral_paths(g, "agent:a")] == [0.0]


def test_safety_valve_raises_instead_of_a_partial_body(monkeypatch):
    g = _fleet_graph(60, 5, 20)
    monkeypatch.setattr(lateral, "_search_records", functools.partial(lateral._search_records, max_pops=3))
    with pytest.raises(lateral.LateralSearchOverflow):
        cr.context_graph_report(g, max_depth=4)


def test_device_memory_returns_after_the_graph_is_freed():
    import torch

    def cycle():
        g = _fleet_graph(400, 9, 40)
        body = cr.context_graph_report(g, max_depth=4)
        assert body["stats"]["lateral_path_count"] > 0
        del g, body

    cycle()
    gc.collect()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
        gc.collect()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20
