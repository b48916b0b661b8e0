"""The graph shapes of graph_shapes.py against answers known by construction, through the CPU oracle (no GPU).

These keep the shapes honest: a chain really is a chain of that many levels, a hub row really has its 100 000 entries in insertion
order, and the oracle's answers on them — the reference the GPU tests of test_gpu_graph_shapes.py compare with — are the closed forms.
"""

from __future__ import annotations

import numpy as np
import pytest

import graph_shapes as gs
from oracle import oracle as orc
from test_gpu_slice_consumers import reference_bottleneck_counts, subtree_counts

REACH4 = (1 << 1) | (1 << 2) | (1 << 7) | (1 << 3)
VULN_PKG = (1 << 8) | (1 << 9)
UNBOUNDED = 2**31 - 1

_cache: dict = {}


def shape(name):
    if name not in _cache:
        s = getattr(gs, name)()
        _cache[name] = (s, orc.build_csr(len(s.node_type), s.src, s.dst, s.rel, s.flags, s.node_type))
    return _cache[name]


def test_deep_shape():
    s, og = shape("deep")
    assert og.n_nodes >= 70_000 and min(og.n_nodes + 4096, 1 << 16) == 65_536        # G1's queue is 65 536 entries on this graph
    # the renaming really scatters consecutive chain members over bitmap words
    c = s.names[f"chain_{gs.LONG_CHAIN}"]
    assert np.mean((c[1:] >> 5) == (c[:-1] >> 5)) < 0.01
    for k in gs.CHAIN_LENGTHS + (gs.LONG_CHAIN,):
        c = s.names[f"chain_{k}"]
        assert len(c) == k and len(np.unique(c)) == k
        assert (og.node_type[c] != gs.AGENT).all() and (og.node_type[c] != gs.GHOST).all()
    assert (s.flags == 0).any() and (s.flags & gs.BIDIR).any()
    assert len(np.unique(og.node_type)) >= 8


@pytest.mark.parametrize("k", gs.CHAIN_LENGTHS + (gs.LONG_CHAIN,))
def test_chain_depths_and_parents(k):
    """Node i of a chain is at depth i and its BFS parent is node i - 1; the reverse walk from the tail is the chain reversed."""
    s, og = shape("deep")
    c = s.names[f"chain_{k}"]
    head, tail = c[:1], c[-1:]
    w = orc.distances_many(og, head, 0xFFFFFFFF)
    np.testing.assert_array_equal(w.nodes, c[1:])
    np.testing.assert_array_equal(w.aux, np.arange(1, k))
    assert int(w.maxd[0]) == k - 1
    b = orc.bfs_many(og, head, UNBOUNDED, True)
    np.testing.assert_array_equal(b.nodes, c[1:])
    np.testing.assert_array_equal(b.aux, np.arange(-1, k - 2))              # parent = position of node i - 1 in the slice
    imp = orc.impact_many(og, tail, UNBOUNDED)
    np.testing.assert_array_equal(imp.nodes, c[-2::-1])
    np.testing.assert_array_equal(imp.hist[0], np.bincount(og.node_type[c[:-1]], minlength=orc.NHIST)[: orc.NHIST])


@pytest.mark.parametrize("depth", [254, 255, 256, 257, -1])
@pytest.mark.parametrize("k", [257, 300, 4100])
def test_bounded_walks_return_the_chain_prefix(k, depth):
    """reachable / bfs / impact to ``depth`` levels return exactly the first ``depth`` nodes after the source; a negative depth
    returns nothing (the reference's ``depth >= max_depth`` skips the source itself)."""
    s, og = shape("deep")
    c = s.names[f"chain_{k}"]
    want = c[1: 1 + max(depth, 0)]
    for trav in (False, True):
        r = orc.reachable_many(og, c[:1], depth, trav)
        np.testing.assert_array_equal(r.nodes, want)
        np.testing.assert_array_equal(r.aux, np.arange(1, len(want) + 1))
        np.testing.assert_array_equal(orc.bfs_many(og, c[:1], depth, trav).nodes, want)
    np.testing.assert_array_equal(orc.impact_many(og, c[-1:], depth).nodes, c[::-1][1: 1 + max(depth, 0)])
    # the unbounded distance walk has no depth to stop at
    np.testing.assert_array_equal(orc.distances_many(og, c[:1], REACH4).nodes, c[1:])


def test_shortest_path_is_the_chain():
    s, og = shape("deep")
    for k in (255, 256, 257, 4100, gs.LONG_CHAIN):
        c = s.names[f"chain_{k}"]
        np.testing.assert_array_equal(orc.shortest_path(og, int(c[0]), int(c[-1])), c)
        assert orc.shortest_path(og, int(c[-1]), int(c[0])) is None            # directed
    c = s.names["chain_300"]
    np.testing.assert_array_equal(orc.shortest_path(og, int(c[0]), int(c[256])), c[:257])
    assert orc.shortest_path(og, int(c[0]), int(s.names["ghosts"][0])) is None
    assert orc.shortest_path(og, int(c[0]), int(s.names["chain_254"][3])) is None


def test_bidirectional_chain_and_comb():
    s, og = shape("deep")
    c = s.names["bichain"]
    mid = 150
    roots, root_off = np.asarray([c[mid]], np.int32), np.asarray([0, 1], np.int64)
    for direction in (1, 2, 3):
        t = orc.traverse_many(og, roots, root_off, direction=direction, max_depth=1000)
        # both neighbours at depth 1 (forward row: original edge to mid + 1, reversed copy to mid - 1), and so on outwards
        assert len(t.nodes) == 300 and t.nodes[0] == c[mid]
        np.testing.assert_array_equal(np.sort(t.aux[1:]), np.sort(np.abs(np.arange(300) - mid)[np.arange(300) != mid]))
        assert int(t.maxd[0]) == mid
    spine, leaf = s.names["comb_spine"], s.names["comb_leaf"]
    r = orc.reachable_many(og, spine[:1], UNBOUNDED, False)
    want = np.stack([spine[1:], leaf[:-1]], axis=1).ravel()
    np.testing.assert_array_equal(r.nodes[:-1], want)                         # level i = (spine i, leaf i - 1)
    assert r.nodes[-1] == leaf[-1]


def test_dependency_reach_min_hop_is_chain_depth_plus_two():
    s, og = shape("deep")
    rank = np.random.default_rng(0).permutation(og.n_nodes).astype(np.int32)
    agents = np.flatnonzero(og.node_type == gs.AGENT).astype(np.int32)
    np.testing.assert_array_equal(np.sort(agents), np.sort(s.names["agents"]))
    want = orc.dependency_reach(og, agents, REACH4, VULN_PKG, rank)
    pkgs = s.names["pkgs"]
    slot = {int(p): i for i, p in enumerate(want["pkg_ids"])}
    pm, po = want["pkg_minhop"], want["pkg_off"]
    for d, p in enumerate(pkgs):
        i = slot[int(p)]
        assert int(pm[i]) == d + 2
        assert int(po[i + 1] - po[i]) == 300
    vslot = {int(v): i for i, v in enumerate(want["vuln_ids"])}
    for d, v in zip(gs.FINDING_DEPTHS, s.names["vulns"]):
        assert int(want["vuln_minhop"][vslot[int(v)]]) == d + 2
        i = vslot[int(v)]
        np.testing.assert_array_equal(want["vuln_pkgs"][want["vuln_poff"][i]: want["vuln_poff"][i + 1]], [pkgs[d]])


@pytest.mark.parametrize("k", [257, 300, 4100])
def test_chain_subtree_rollup(k):
    """Bottleneck roll-up over one chain walk: node i (i >= 1) lies strictly inside the paths to the n - 1 - i nodes after it."""
    s, og = shape("deep")
    c = s.names[f"chain_{k}"]
    got = subtree_counts(og, c[:1])
    want = np.zeros(og.n_nodes, np.uint64)
    want[c[1:]] = (k - 1 - np.arange(1, k)).astype(np.uint64)
    np.testing.assert_array_equal(got, want)
    if k <= 300:
        np.testing.assert_array_equal(reference_bottleneck_counts(og, c[:1]), want)


def test_hub_rows_in_row_order():
    s, og = shape("wide")
    leaves, fhub, rhub = s.names["leaves"], s.names["fhub"], s.names["rhub"]
    assert og.n_nodes > gs.HUB_ROW and min(og.n_nodes + 4096, 1 << 16) == 65_536
    assert int(og.fwd_off[fhub + 1] - og.fwd_off[fhub]) == gs.HUB_ROW and int(og.rev_off[rhub + 1] - og.rev_off[rhub]) == gs.HUB_ROW
    r = orc.reachable_many(og, [fhub], 1, False)
    np.testing.assert_array_equal(r.nodes, leaves)
    imp = orc.impact_many(og, [rhub], 2)
    np.testing.assert_array_equal(imp.nodes, np.concatenate([leaves, [fhub]]))
    np.testing.assert_array_equal(imp.aux, np.concatenate([np.ones(gs.HUB_ROW, np.int32), [2]]))
    b = orc.bfs_many(og, [fhub], 5, False)
    np.testing.assert_array_equal(b.nodes, np.concatenate([leaves, [rhub]]))
    assert int(b.aux[-1]) == 0                                               # rhub's first discoverer is the first leaf


def test_repeated_neighbour_row():
    s, og = shape("wide")
    rep, x = s.names["rep"], s.names["x"]
    a, b = int(og.fwd_off[rep]), int(og.fwd_off[rep + 1])
    row, meta = og.fwd_nbr[a:b], og.fwd_meta[a:b]
    np.testing.assert_array_equal(np.flatnonzero(row == x), gs.REPEAT_AT)
    np.testing.assert_array_equal(meta[list(gs.REPEAT_AT)] & 0x1F, gs.REPEAT_RELS)
    assert meta[0] & orc.META_FIRSTPAIR and not (meta[list(gs.REPEAT_AT[1:])] & orc.META_FIRSTPAIR).any()
    assert (row == rep).sum() == 3                                           # self-loop, bidirectional self-loop and its reversed copy
    # x is discovered once, at its first occurrence; the fillers keep their row order around it
    r = orc.reachable_many(og, [rep], 1, False)
    np.testing.assert_array_equal(r.nodes, [v for i, v in enumerate(row) if v != rep and (v != x or i == 0)])
    # traversable only: x is first reached through a traversable repeat (position 0 is)
    assert orc.reachable_many(og, [rep], 1, True).nodes[0] == x
    rrep, y = s.names["rrep"], s.names["y"]
    a, b = int(og.rev_off[rrep]), int(og.rev_off[rrep + 1])
    np.testing.assert_array_equal(np.flatnonzero(og.rev_nbr[a:b] == y), gs.REPEAT_AT)


def test_clique_and_bipartite():
    s, og = shape("wide")
    cl, left, right = s.names["clique"], s.names["left"], s.names["right"]
    r = orc.reachable_many(og, cl[:1], 3, False)
    assert sorted(r.nodes.tolist()) == sorted(cl[1:].tolist()) and (r.aux == 1).all()
    r = orc.reachable_many(og, left[:1], 3, False)
    np.testing.assert_array_equal(r.nodes, np.concatenate([right, left[1:]]))
    np.testing.assert_array_equal(r.aux, np.concatenate([np.ones(200, np.int32), np.full(199, 2, np.int32)]))


def test_tiny_graphs():
    t = {k: (s, orc.build_csr(len(s.node_type), s.src, s.dst, s.rel, s.flags, s.node_type)) for k, s in gs.tiny().items()}
    s, og = t["n1"]
    assert og.n_nodes == 1 and len(s.src) == 0
    assert len(orc.reachable_many(og, [0], 5).nodes) == 0 and len(orc.distances_many(og, [0], REACH4).nodes) == 0
    s, og = t["n2_self_loop"]
    assert len(orc.reachable_many(og, [s.names["loop"]], 5).nodes) == 0       # a self-loop discovers nothing
    np.testing.assert_array_equal(orc.impact_many(og, [s.names["loop"]], 5).nodes, [])
    for n in (31, 32, 33):
        s, og = t[f"n{n}_ring"]
        ring = s.names["ring"]
        np.testing.assert_array_equal(orc.distances_many(og, ring[:1], 0xFFFFFFFF).nodes, ring[1:])
        np.testing.assert_array_equal(orc.impact_many(og, ring[:1], UNBOUNDED).aux[:1], [1])
    s, og = t["ghost_roots"]
    gh = s.names["ghosts"]
    assert (og.node_type[gh] == gs.GHOST).all()
    assert len(orc.reachable_many(og, gh, 9).nodes) == 0 and (orc.reachable_many(og, gh, 9).flags == 2).all()
    # the distance walk starts at ghosts too (the reference's _bfs_distances_along does not ask for a node record)
    d = orc.distances_many(og, gh[:1], 0xFFFFFFFF)
    np.testing.assert_array_equal(d.nodes, np.concatenate([s.names["real"], gh[2:]]))
