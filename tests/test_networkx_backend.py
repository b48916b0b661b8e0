"""B200NetworkXBackend (name "b200-networkx"), the drop-in for the reference's NetworkXBackend — host side and the CPU oracle.

``tests/golden/context/networkx_backend.json.gz`` (``oracle/make_networkx_golden.py``): op sequences replayed on the unmodified
reference ``NetworkXBackend`` (networkx 3.6.1) with every protocol method's answer.  The GPU answers are checked in
``test_gpu_networkx_backend.py``; here the DiGraph host semantics and the oracle (``oracle/nx_oracle.c``) are pinned bit for bit.
"""

from __future__ import annotations

import gzip
import json
from pathlib import Path

import numpy as np
import pytest

from oracle import nx_oracle

GOLD = json.loads(gzip.decompress((Path(__file__).parent / "golden" / "context" / "networkx_backend.json.gz").read_bytes()))
CASES = GOLD["cases"]
LABELS = [c["label"] for c in CASES]


def replay(ops, **kwargs):
    from agent_bom_b200.backend import get_backend

    b = get_backend("b200-networkx", **kwargs)
    for op in ops:
        if op[0] == "n":
            b.add_node(op[1], op[2], op[3], **op[4])
        else:
            b.add_edge(op[1], op[2], op[3], op[4], directed=op[5], **op[6])
    return b


@pytest.mark.parametrize("case", CASES, ids=LABELS)
def test_host_methods_match_the_reference(case):
    b = replay(case["ops"])
    assert (b.node_count(), b.edge_count()) == (case["node_count"], case["edge_count"])
    assert list(b._nodes) == case["node_ids"]                  # implicit endpoints take their place in node order
    if "to_dict" in case:
        assert b.to_dict() == case["to_dict"]
        for nid, want in case["neighbors"].items():
            assert b.neighbors(nid) == want
        for s, t, want in case["has_edge"]:
            assert b.has_edge(s, t) is want
    assert b.has_node("missing") is False and b.neighbors("missing") == [] and b.bfs("missing") == []
    for s, t, want in case["shortest"]:
        if s not in b._nodes or t not in b._nodes or s == t:   # answered on the host
            assert b.shortest_path(s, t) == want


@pytest.mark.parametrize("case", CASES, ids=LABELS)
def test_oracle_matches_networkx_bit_for_bit(case):
    g = nx_oracle.replay(case["ops"])
    assert g.ids == case["node_ids"]
    pr, it = nx_oracle.pagerank(g)
    bc, _ = nx_oracle.betweenness(g)
    assert pr.tolist() == case["pagerank"] and (it > 0 or not g.ids)
    assert bc.tolist() == case["betweenness"]
    assert nx_oracle.betweenness(g, threads=1)[0].tolist() == case["betweenness"]      # the batch sum is in source order


def test_path_counts_exceed_2_pow_53():
    """The layered complete-bipartite chain makes sigma pass 2**53, where the order of the path-count sums matters."""
    case = next(c for c in CASES if c["label"] == "bipartite-chain")
    width = sum(1 for v in case["node_ids"] if v.startswith("L00_"))
    layers = len(case["node_ids"]) // width
    assert width ** (layers - 1) > 2 ** 53


def test_digraph_semantics():
    b = replay([])
    b.add_edge("a", "b", "uses", 2.0, directed=True, note="x")
    assert b.node_count() == 2 and b.to_dict()["nodes"] == [{"id": "a"}, {"id": "b"}]        # endpoints without attributes
    b.add_node("b", "server", "B", tier=1)
    b.add_node("a", "agent", "A")
    b.add_node("b", "server", "B2")
    assert b.to_dict()["nodes"] == [{"id": "a", "kind": "agent", "label": "A"}, {"id": "b", "kind": "server", "label": "B2", "tier": 1}]
    b.add_edge("a", "b", "calls", 0.5, directed=True, extra=True)                               # merged, keeps its place
    b.add_edge("a", "c", "uses", directed=True)
    assert b.to_dict()["edges"][0] == {"source": "a", "target": "b", "kind": "calls", "weight": 0.5, "note": "x", "extra": True}
    assert b.neighbors("a") == ["b", "c"] and b.neighbors("b") == [] and b.edge_count() == 1      # number_of_edges() // 2
    b.add_edge("c", "a", "uses", 3.0)
    assert b.edge_count() == 1 and b.neighbors("c") == ["a"] and b.has_edge("a", "c") and b.has_edge("c", "a")


def test_csr_export_keeps_dict_orders_and_weights():
    """Forward rows are the successor dicts, reverse rows the predecessor dicts (first insertion order), weights per forward entry."""
    b = replay([["e", "x", "z", "k", 1.5, True, {}], ["e", "y", "z", "k", 2.5, True, {}], ["e", "z", "x", "k", 0.5, False, {}],
                ["e", "x", "z", "k", 4.0, True, {}], ["n", "w", "agent", "w", {}]])
    c = b.csr
    ids = c.node_ids
    assert ids == ["x", "z", "y", "w"]
    rows = lambda off, nbr: [[ids[j] for j in nbr[off[i]:off[i + 1]]] for i in range(len(ids))]    # noqa: E731
    assert rows(c.fwd_off, c.fwd_nbr) == [["z"], ["x"], ["z"], []]
    assert rows(c.rev_off, c.rev_nbr) == [["z"], ["x", "y"], [], []]
    assert b.weights.tolist() == [4.0, 0.5, 2.5]


def test_empty_graph_answers_on_the_host():
    b = replay([])
    assert b.centrality_scores() == {} and b.bottleneck_nodes() == [] and b.bfs("a") == [] and b.shortest_path("a", "a") is None


def test_protocol_shape_and_backend_names():
    import inspect

    from agent_bom_b200.backend import B200Backend, B200NetworkXBackend, GraphBackend, from_context_graph, get_backend

    sig = inspect.signature(B200NetworkXBackend.add_edge)
    assert list(sig.parameters)[:5] == ["self", "source", "target", "kind", "weight"] and sig.parameters["directed"].kind is inspect.Parameter.KEYWORD_ONLY
    assert isinstance(get_backend("b200-networkx"), GraphBackend)
    assert type(get_backend("b200")) is B200Backend and type(get_backend("auto")) is B200Backend
    with pytest.raises(ValueError):
        get_backend("networkx")
    c = from_context_graph({"nodes": [{"id": "a", "kind": "agent"}], "edges": [{"source": "a", "target": "s", "kind": "uses"}]}, backend="b200-networkx")
    assert type(c) is B200NetworkXBackend and c.node_count() == 2 and c.edge_count() == 1


def test_unified_graph_bridge():
    """from_unified_graph(backend="b200-networkx") issues the reference bridge's calls (mesh inventory, weights aside: the walk
    fixture does not carry them)."""
    from golden_util import graph_from_fixture, load

    from agent_bom_b200.backend import from_unified_graph

    case = next(c for c in CASES if c["label"] == "mesh:from_unified_graph")
    b = from_unified_graph(graph_from_fixture(load("mesh_inventory")), backend="b200-networkx")
    want = replay(case["ops"])
    assert list(b._nodes) == list(want._nodes) and b.to_dict()["nodes"] == want.to_dict()["nodes"]
    strip = lambda d: [{k: v for k, v in e.items() if k != "weight"} for e in d["edges"]]    # noqa: E731
    assert strip(b.to_dict()) == strip(want.to_dict()) and b.edge_count() == want.edge_count()
    assert np.array_equal(b.csr.fwd_nbr, want.csr.fwd_nbr) and np.array_equal(b.csr.rev_nbr, want.csr.rev_nbr)
