"""The context-graph report golden (tests/golden/context/report.json.xz, oracle/make_context_report_golden.py): loading, graph
rebuilding and body comparison shared by tests/test_context_report.py and tests/test_gpu_context_report.py."""

from __future__ import annotations

import json
import lzma
from pathlib import Path

from agent_bom_b200.context_graph import ContextGraph, EdgeKind, GraphEdge, GraphNode, NodeKind
from agent_bom_b200.lateral import LateralPath

DOCS = json.loads(lzma.decompress((Path(__file__).parent / "golden" / "context" / "report.json.xz").read_bytes()))
IDS = [d["name"] for d in DOCS]
BUILT = [d for d in DOCS if d["input"] is not None]


def _entry(e):
    return [e.source, e.target, e.kind.value, e.weight, e.metadata]


def graph_doc(g) -> dict:
    """The golden's record of a graph: nodes, edges and adjacency rows with weights and metadata, in order."""
    return {"nodes": [[n.id, n.kind.value, n.label, n.metadata] for n in g.nodes.values()],
            "edges": [_entry(e) for e in g.edges],
            "adjacency": [[nid, [_entry(e) for e in lst]] for nid, lst in g.adjacency.items()]}


def rebuild(doc) -> ContextGraph:
    """The recorded graph on this package's container: nodes, ``add_edge`` per edge (mirrored twins share the metadata dict),
    then the hand-wired adjacency entries; checked against the recorded adjacency."""
    g = ContextGraph()
    rec = doc["graph"]
    for nid, kind, label, meta in rec["nodes"]:
        g.add_node(GraphNode(id=nid, kind=NodeKind(kind), label=label, metadata=meta))
    for s, t, k, w, meta in rec["edges"]:
        g.add_edge(GraphEdge(source=s, target=t, kind=EdgeKind(k), weight=w, metadata=meta))
    for owner, s, t, k, w, meta in doc.get("extra_adjacency") or []:
        g.adjacency[owner].append(GraphEdge(source=s, target=t, kind=EdgeKind(k), weight=w, metadata=meta))
    assert json.dumps(graph_doc(g)) == json.dumps(rec)
    return g


def injected(doc) -> dict:
    """The reference's classifier and credential rule for this input, as recorded."""
    caps = doc["input"]["tool_caps"]
    creds = set(doc["input"]["cred_keys"])
    return {"classify_tool": lambda name, desc, declared: caps[json.dumps([name, desc, declared])], "is_credential_key": lambda k: k in creds}


def golden_paths(report) -> list[LateralPath]:
    return [LateralPath(source=p["source"], target=p["target"], hops=p["hops"], edges=[EdgeKind(k) for k in p["edges"]], composite_risk=p["composite_risk"],
                        summary=p["summary"], credential_exposure=p["credential_exposure"], tool_exposure=p["tool_exposure"], vuln_ids=p["vuln_ids"])
            for p in json.loads(report["lateral_paths"])]


def assert_body(doc, report, body) -> None:
    """The body equals the golden as JSON text, key by key and in key order."""
    assert list(body) == report["keys"]
    for key in ("nodes", "edges", "interaction_risks"):
        assert json.dumps(body[key]) == doc["body"][key], key
    assert json.dumps(body["lateral_paths"]) == report["lateral_paths"], (report["agent"], report["max_depth"])
    assert json.dumps(body["stats"]) == report["stats"], (report["agent"], report["max_depth"])
