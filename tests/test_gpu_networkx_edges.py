"""The NetworkX backend on the GPU at the edges of the estate golden (``tests/golden/context/networkx_edges.json.gz``): non-finite
and degenerate weights, every row length around numpy's pairwise-sum blocks, overflowing path counts, paths that outgrow the
first path arena; exact shortest paths on estates against the restatement of ``nx.shortest_path``; and PageRank on a graph
large enough that every PageRank kernel strides its grid."""

from __future__ import annotations

import numpy as np
import pytest

from oracle import nx_oracle
from test_networkx_backend import replay
from test_networkx_edges import (CASE, PAGERANK_LABELS, arrays_of, assert_bitwise, check_pagerank, estate_ops, estate_pairs, hub_of,
                                 ops_of, scale_graph)

pytestmark = pytest.mark.gpu

ABB_ERR_ARG = -2            # include/abb200.h: what abb_pagerank_host returns when the power iteration does not converge


@pytest.mark.parametrize("label", PAGERANK_LABELS)
def test_pagerank_matches_networkx(label):
    """Scores bit for bit (NaN by position) and iterations; where networkx raises PowerIterationFailedConvergence the device
    call fails with ABB_ERR_ARG."""
    from agent_bom_b200._lib import AbbError

    case = CASE[label]
    b = replay(ops_of(label))
    dg = b.device_graph
    if case["iterations"] == 0:
        with pytest.raises(AbbError) as err:
            dg.pagerank(b.weights)
        assert err.value.code == ABB_ERR_ARG
    else:
        check_pagerank(case, *dg.pagerank(b.weights))
        assert b.centrality_scores() == dict(zip(b.csr.node_ids, dg.pagerank(b.weights)[0].tolist()))


def test_betweenness_keeps_networkx_nans():
    """Path counts overflow to inf on the chain: NaN wherever networkx has NaN, 0.0 on the two sources of layer 0."""
    case = CASE["chain"]
    dg = replay(ops_of("chain")).device_graph
    assert_bitwise(dg.betweenness(), case["betweenness"], "chain")
    dg.set_option("nx_batch", 3)
    assert_bitwise(dg.betweenness(), case["betweenness"], "chain, 3 sources per batch")


@pytest.mark.parametrize("cap", [0, 3])
def test_long_paths_outgrow_the_first_arena(cap):
    """The answers total more than the first path arena (max(8 per pair, 65 536) nodes), so the search reruns with the arena
    it measured; every answer, ``None`` included, equals networkx's."""
    case = CASE["long-path"]
    b = replay(ops_of("long-path"))
    dg = b.device_graph
    dg.set_option("nx_batch", cap)
    src = np.asarray([s for s, _, _ in case["shortest"]], dtype=np.int32)
    dst = np.asarray([t for _, t, _ in case["shortest"]], dtype=np.int32)
    got = dg.bidirectional_paths(src, dst)
    assert [None if p is None else p.tolist() for p in got] == [p for _, _, p in case["shortest"]]
    total = sum(p.shape[0] for p in got if p is not None)
    assert total > max(65_536, 8 * len(got))
    ids = b.csr.node_ids
    for s, d, want in case["bfs"]:
        assert b.bfs(ids[s], d) == [[ids[i] for i in p] for p in want], (s, d)


ESTATES = [(1000, False, False), (1000, False, True), (2000, True, False), (2000, True, True)]


@pytest.mark.parametrize("agents,bench_knobs,both_ways", ESTATES, ids=["1000-agents", "1000-agents-both-ways", "M1", "M1-both-ways"])
def test_estate_paths_equal_networkx(agents, bench_knobs, both_ways):
    """Every pair of ``estate_pairs`` (seeded pairs, the longest answers, pairs without a path, s == t, pairs from and to the
    node of largest degree) gives the restated ``nx.shortest_path`` answer exactly, with the search slots sized from memory,
    capped at 3 and at 1 (one slot reused for every pair).  On the directed estates ``bfs(source, 4)`` and ``bfs(source, 6)``
    for 20 sources, the hub among them, equal the restated ``bfs``."""
    from agent_bom_b200 import estate

    b = replay(estate_ops(agents, estate.BENCH_KNOBS if bench_knobs else estate.Knobs(), both_ways=both_ways))
    c = b.csr
    rows = nx_oracle.Rows.of(c)
    pairs = estate_pairs(rows, agents)
    want = [nx_oracle.shortest_path(rows, s, t) for s, t in pairs]
    assert sum(p is None for p in want) >= 20 or both_ways
    assert sum(p is not None and len(p) > 1 for p in want) > len(pairs) // 3
    src = np.asarray([s for s, _ in pairs], dtype=np.int32)
    dst = np.asarray([t for _, t in pairs], dtype=np.int32)
    dg = b.device_graph
    for cap in (0, 3, 1):
        dg.set_option("nx_batch", cap)
        got = dg.bidirectional_paths(src, dst)
        bad = [i for i, (p, w) in enumerate(zip(got, want)) if (None if p is None else p.tolist()) != w]
        assert not bad, f"nx_batch {cap}: {len(bad)} pairs differ, first {pairs[bad[0]]}"
    if both_ways:
        return
    dg.set_option("nx_batch", 0)
    rng = np.random.default_rng(agents + 1)
    hub = hub_of(rows)
    sources = [hub] + rng.choice(np.flatnonzero(np.diff(c.fwd_off.astype(np.int64)) > 0), 19, replace=False).tolist()
    ids = c.node_ids
    for s in sources:
        for d in (4, 6):
            assert b.bfs(ids[s], d) == [[ids[i] for i in p] for p in nx_oracle.bfs(rows, s, d)], (s, d)


def test_pagerank_grid_stride():
    """700 000 nodes and about 3 M entries, three rows and one column of 70 000 entries: more items than the 16 blocks per SM x
    256 threads of the PageRank launches, so the row-sum, value and step kernels all loop over their grids.  Scores and iterations
    equal the oracle's bit for bit."""
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    n = 700_000
    src, dst, w = scale_graph(n, 3_400_000, 3, 70_000, 700)
    assert src.shape[0] > 2_900_000
    host = csrmod.from_arrays(None, np.zeros(n, dtype=np.uint8), src, dst, np.zeros(src.shape[0], dtype=np.uint8),
                              np.full(src.shape[0], csrmod.EDGE_TRAVERSABLE, dtype=np.uint8))
    dg = DeviceGraph.upload(host, 0)
    try:
        pr, it = dg.pagerank(w[host.fwd_eid >> 1])
    finally:
        dg.close()
    want, want_it = nx_oracle.pagerank(arrays_of(n, src, dst, w))
    assert want_it > 0 and it == want_it
    assert_bitwise(pr, want, "700 K nodes")
