"""B200NetworkXBackend on the GPU: every answer of the reference's NetworkXBackend (``tests/golden/context/networkx_backend.json.gz``)
with ``==`` on floats, and the device against the CPU oracle (``oracle/nx_oracle.c``) on estates NetworkX is too slow for."""

from __future__ import annotations

import numpy as np
import pytest

from oracle import nx_oracle
from test_networkx_backend import CASES, LABELS, replay

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=LABELS)
def test_every_answer_matches_networkx(case):
    b = replay(case["ops"])
    ids = case["node_ids"]
    assert b.centrality_scores() == dict(zip(ids, case["pagerank"]))
    for key, top in (("bottleneck_5", 5), ("bottleneck_20", 20), ("bottleneck_n", len(ids))):
        assert [list(x) for x in b.bottleneck_nodes(top)] == case[key], key
    if ids:
        assert b.device_graph.betweenness().tolist() == case["betweenness"]
    for s, d, want in case["bfs"]:
        assert b.bfs(s, d) == want, (s, d)
    for s, t, want in case["shortest"]:
        assert b.shortest_path(s, t) == want, (s, t)


def test_batching_is_invisible():
    """Betweenness batches and path-search slots forced down to a few per launch give the same answers."""
    for label in ("random:4", "bipartite-chain", "mesh:from_unified_graph"):
        case = CASES[LABELS.index(label)]
        b = replay(case["ops"])
        dg = b.device_graph
        for cap in (1, 3, 7):
            dg.set_option("nx_batch", cap)
            assert dg.get_option("nx_batch") == cap
            assert dg.betweenness().tolist() == case["betweenness"]
            for s, t, want in case["shortest"]:
                assert b.shortest_path(s, t) == want
            for s, d, want in case["bfs"]:
                assert b.bfs(s, d) == want


def test_mutation_after_a_query_reexports_the_csr_and_weights():
    case = CASES[LABELS.index("random:1")]
    b = replay(case["ops"])
    assert b.centrality_scores() == dict(zip(case["node_ids"], case["pagerank"]))
    s, t = case["node_ids"][0], case["node_ids"][1]
    b.add_edge(s, t, "uses", 9.0, directed=True)                # a merged weight on an existing edge, or a new edge
    b.add_edge("late", s, "uses", 0.25, directed=True)
    ops = case["ops"] + [["e", s, t, "uses", 9.0, True, {}], ["e", "late", s, "uses", 0.25, True, {}]]
    g = nx_oracle.replay(ops)
    pr, _ = nx_oracle.pagerank(g)
    assert b.centrality_scores() == dict(zip(g.ids, pr.tolist()))
    assert b.device_graph.betweenness().tolist() == nx_oracle.betweenness(g)[0].tolist()
    assert b.shortest_path("late", t)[:2] == ["late", s]


def estate_backend(agents: int, knobs):
    """A generator estate as a DiGraph: bidirectional edges both ways, weights varied by relationship."""
    from agent_bom_b200 import estate

    est = estate.generate(agents, 2145, knobs, exact_rank=False)
    ids = [f"v{i}" for i in range(len(est.node_type))]
    ops = [["n", v, "node", v, {}] for v in ids]
    weights = (1.0, 0.5, 0.25, 1.5, 2.0, 1 / 3)
    for s, d, r, f in zip(est.src.tolist(), est.dst.tolist(), est.rel.tolist(), est.flags.tolist()):
        ops.append(["e", ids[s], ids[d], "rel", weights[r % len(weights)], not (f & 2), {}])
    return replay(ops), nx_oracle.replay(ops)


@pytest.mark.parametrize("agents,bench_knobs", [(1000, False), (2000, True)], ids=["1000-agents", "M1"])
def test_device_matches_the_oracle_on_estates(agents, bench_knobs):
    from agent_bom_b200 import estate

    b, g = estate_backend(agents, estate.BENCH_KNOBS if bench_knobs else estate.Knobs())
    assert list(b._nodes) == g.ids
    dg = b.device_graph
    pr, it = dg.pagerank(b.weights)
    want_pr, want_it = nx_oracle.pagerank(g)
    assert it == want_it and np.array_equal(pr, want_pr)
    assert np.array_equal(dg.betweenness(), nx_oracle.betweenness(g)[0])
    rng = np.random.default_rng(agents)
    src = rng.integers(0, g.n, 2000, dtype=np.int32)
    dst = rng.integers(0, g.n, 2000, dtype=np.int32)
    paths = dg.bidirectional_paths(src, dst)
    for s, t, p in zip(src.tolist(), dst.tolist(), paths):
        if p is not None:                                   # a valid path: starts at s, ends at t, every hop an edge
            assert p[0] == s and p[-1] == t
            assert all(int(v) in b.csr.fwd_nbr[b.csr.fwd_off[int(u)]:b.csr.fwd_off[int(u) + 1]] for u, v in zip(p[:-1], p[1:]))
