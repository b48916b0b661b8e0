"""Every walk kind on the deep, wide and tiny shapes of graph_shapes.py, bit for bit against the CPU oracle, with the storage-tier
hand-offs each shape exists for asserted from ``last_walk_tier_counts()``.

The walk keeps a query in one of five tiers (abb200.cu ``enqueue_tiers``): S1 (warp, shared memory, 256-entry queue, 8-bit depth),
the big block tier (36 864-entry queue), the mid block tier (shared-memory queue of up to 4 096 entries, 8-bit depth: it hands on at
level 255), G1 (warp, global bitmap, queue of min(n + 4096, 65 536)) and GX (whole graph).  The counters report S1's hand-offs
(``s1``, of which forecast-heavy ``s1_heavy``), the mid tier's (``mid``) and G1's (``g1``, to GX), summed here over the canonical and
the individual pass of a de-duplicated batch.  The big tier's own hand-offs are not reported: where a query goes through it (S1's
heavy hand-offs under the ``default`` / ``big-always`` / ``all-tiers`` / ``shrunk`` settings), only the later tiers' counters show
that it was handed on.

Every test sets its tier options and de-duplication explicitly and puts back what was there before.
"""

from __future__ import annotations

import numpy as np
import pytest

import graph_shapes as gs
from oracle import ocsf_oracle
from oracle import oracle as orc
from test_gpu_slice_consumers import pinned, subtree_counts
from test_gpu_tiers import CONFIGS

pytestmark = pytest.mark.gpu

REACH4 = (1 << 1) | (1 << 2) | (1 << 7) | (1 << 3)
VULN_PKG = (1 << 8) | (1 << 9)
DEEP = 1 << 30                    # a depth bound no walk here reaches
MID_DEPTH_CONFIGS = ("mid-only", "all-tiers", "big-never-routed")     # the mid tier is on with its full 4 096-entry queue
DEDUP = [pytest.param(True, id="dedup_on"), pytest.param(False, id="dedup_off")]

_graphs: dict = {}


def graph(name):
    """(shape, oracle graph, device graph, node rank) for "deep", "wide" or a ``tiny()`` name."""
    if name not in _graphs:
        from agent_bom_b200.engine import DeviceGraph
        from agent_bom_b200.graph import csr as csrmod

        s = getattr(gs, name)() if name in ("deep", "wide") else gs.tiny()[name]
        n = len(s.node_type)
        rank = np.random.default_rng(n).permutation(n).astype(np.int32)
        og = orc.build_csr(n, s.src, s.dst, s.rel, s.flags, s.node_type)
        dg = DeviceGraph.upload(csrmod.from_arrays(None, s.node_type, s.src, s.dst, s.rel, s.flags, node_rank=rank))
        _graphs[name] = (s, og, dg, rank)
    return _graphs[name]


def tiers(dg) -> dict:
    t = dg.last_walk_tier_counts()
    return {k: t["first"][k] + t["individual"][k] for k in t["first"]}


def assert_walk_equal(got, want, aux=None, shift=0, what="", maxd=True):
    """Node order (and parents / depths) of every slice, vectorised; the per-query loop only runs to name the first mismatch."""
    counts = np.diff(want.off)
    np.testing.assert_array_equal(got.count, counts.astype(np.int32), err_msg=f"counts {what}")
    idx = np.repeat(got.start.astype(np.int64) - want.off[:-1], counts) + np.arange(int(want.off[-1]))
    ok = np.array_equal(got.nodes[idx], want.nodes)
    if aux is not None:
        ok = ok and np.array_equal(getattr(got, aux)[idx] + shift, want.aux)
    if not ok:
        for q in range(len(counts)):
            a, b = int(want.off[q]), int(want.off[q + 1])
            np.testing.assert_array_equal(got.slice(q), want.nodes[a:b], err_msg=f"query {q} node order {what}")
            if aux is not None:
                np.testing.assert_array_equal(got.aux(q, aux) + shift, want.aux[a:b], err_msg=f"query {q} {aux} {what}")
    if maxd:
        np.testing.assert_array_equal(got.maxd, want.maxd, err_msg=f"maxd {what}")


def assert_traverse_equal(got, want, what=""):
    assert_walk_equal(got, want, aux="depth", what=what, maxd=False)
    np.testing.assert_array_equal(got.flags & 1, want.flags & 1, err_msg=f"truncated {what}")
    np.testing.assert_array_equal(got.ecount, np.diff(want.eoff), err_msg=f"edge counts {what}")
    idx = np.repeat(got.estart.astype(np.int64) - want.eoff[:-1], np.diff(want.eoff)) + np.arange(int(want.eoff[-1]))
    np.testing.assert_array_equal(got.edges[idx], want.edges, err_msg=f"recorded edges {what}")


def assert_context_equal(got, want):
    """Every per-finding array of ``DeviceGraph.finding_context`` and its flat source list against ``ocsf_oracle.finding_context``."""
    np.testing.assert_array_equal(got.count, want.count)
    np.testing.assert_array_equal(got.maxd, want.maxd)
    np.testing.assert_array_equal(got.flags & 2, want.flags & 2)
    np.testing.assert_array_equal(got.hist, want.hist)
    bc = want.bucket_counts()
    np.testing.assert_array_equal(got.bucket_counts, bc)
    per = bc.sum(axis=1).astype(np.int64)
    np.testing.assert_array_equal(got.start, np.cumsum(per) - per)
    flat = [x for lists in want.lists for x in lists]
    np.testing.assert_array_equal(got.source_nodes, np.concatenate(flat) if flat else np.zeros(0, np.int32))


def emitted(og, want, types: int):
    """The oracle's distance walk restricted to the entity types a type-filtered device walk emits (same order)."""
    keep = ((types >> np.minimum(og.node_type[want.nodes].astype(np.int64), 31)) & 1).astype(bool)
    q_of = np.repeat(np.arange(len(want.off) - 1), np.diff(want.off))
    off = np.zeros(len(want.off), np.int64)
    off[1:] = np.cumsum(np.bincount(q_of[keep], minlength=len(want.off) - 1))
    return orc.WalkResult(off=off, nodes=want.nodes[keep], aux=want.aux[keep], maxd=want.maxd, flags=want.flags)


# ── plain walks under every tier setting ─────────────────────────────────────────────────────────────────────────────────────
def plain_sources(s):
    """> 4 800 single sources: every position of the 300- and 4 100-node chains (the 300-chain twice, so that de-duplicated
    sources share a walk), the comb, heads and tails of every short chain, part of the bidirectional chain, ghosts, invalid ids."""
    nm = s.names
    n = len(s.node_type)
    short = [nm[f"chain_{k}"] for k in gs.CHAIN_LENGTHS]
    return np.concatenate([nm["chain_300"], nm["chain_300"][::3], nm["chain_4100"], nm["comb_spine"], nm["comb_leaf"][::10], nm["bichain"][::10],
                           [c[0] for c in short], [c[-1] for c in short], nm["ghosts"], [-1, n + 3]]).astype(np.int32)


_want: dict = {}


def plain_oracle(og, sources, kind, depth=None):
    key = (kind, depth)
    if key not in _want:
        if kind == "impact":
            _want[key] = orc.impact_many(og, sources, depth)
        elif kind == "bfs":
            _want[key] = orc.bfs_many(og, sources, DEEP, True)
        elif kind == "reachable":
            _want[key] = orc.reachable_many(og, sources, DEEP, False)
        else:
            _want[key] = orc.distances_many(og, sources, depth)
    return _want[key]


@pytest.mark.parametrize("dedup", DEDUP)
@pytest.mark.parametrize("config", list(CONFIGS))
def test_plain_walks_on_deep_chains(config, dedup):
    """impact at depths around 255, bfs with parents, reachable and unbounded distances (with and without a type filter) from
    every position of the 300- and 4 100-node chains: S1 hands every chain of 257+ levels on; with the mid tier on, it does too."""
    s, og, dg, _ = graph("deep")
    sources = plain_sources(s)
    mid_on = config in MID_DEPTH_CONFIGS
    with pinned(dg, dedup, config):
        for depth in (1, 4, 254, 255, 256, 257):
            want = plain_oracle(og, sources, "impact", depth)
            got = dg.impact_many(sources, depth)
            assert_walk_equal(got, want, what=f"impact d={depth}")
            np.testing.assert_array_equal(got.hist, want.hist)
            np.testing.assert_array_equal(got.flags & 2, want.flags & 2)
            assert (dg.last_walk_stats()["groups"] > 0) == dedup
            # a 256-level walk needs S1's 257th queue entry and its 256th level; a de-duplicated source's shared walk starts
            # one level down, so there it takes 257 levels
            if depth >= 257 or (depth == 256 and not dedup):
                t = tiers(dg)
                assert t["s1"] > 0 and (t["mid"] > 0 or not mid_on), t
        got = dg.bfs_many(sources, DEEP, True)
        assert_walk_equal(got, plain_oracle(og, sources, "bfs"), aux="parent", shift=-1, what="bfs")
        t = tiers(dg)
        assert t["s1"] > 0 and (t["mid"] > 0 or not mid_on), t
        got = dg.reachable_many(sources, DEEP, False)
        assert_walk_equal(got, plain_oracle(og, sources, "reachable"), what="reachable")
        assert (dg.last_walk_stats()["groups"] > 0) == dedup
        for mask, types in ((0xFFFFFFFF, 0xFFFFFFFF), (REACH4, (1 << gs.PACKAGE) | (1 << gs.TOOL))):
            want = plain_oracle(og, sources, "distances", mask)
            got = dg.walk(dg.spec_distances(mask, types), sources)
            assert (dg.last_walk_stats()["groups"] > 0) == dedup
            t = tiers(dg)
            assert t["s1"] > 0 and (t["mid"] > 0 or not mid_on), t
            assert_walk_equal(got, want if types == 0xFFFFFFFF else emitted(og, want, types), aux="depth", what=f"distances {mask:#x}")


@pytest.mark.parametrize("dedup", DEDUP)
@pytest.mark.parametrize("config", MID_DEPTH_CONFIGS)
def test_mid_tier_hands_on_at_level_255(config, dedup):
    """Walks of at most 600 queue entries (well inside the mid tier's queue) that are deeper than 255 levels: the mid tier hands
    them on because of its 8-bit depth, not its queue, and the depths past 255 come out right."""
    s, og, dg, _ = graph("deep")
    nm = s.names
    sources = np.concatenate([[nm[f"chain_{k}"][0] for k in (254, 255, 256, 257, 258)], nm["chain_300"], nm["chain_300"][:40], nm["comb_spine"],
                              nm["bichain"][:1]]).astype(np.int32)
    assert len(sources) >= 256
    want = orc.distances_many(og, sources, 0xFFFFFFFF)
    assert int(np.diff(want.off).max()) <= 600 and int(want.maxd.max()) > 255
    with pinned(dg, dedup, config):
        assert dg.get_option("mid_qcap") == 4096
        got = dg.walk(dg.spec_distances(0xFFFFFFFF), sources)
        t = tiers(dg)
        assert (dg.last_walk_stats()["groups"] > 0) == dedup
    assert t["mid"] > 0 and t["s1_heavy"] == 0, t
    assert_walk_equal(got, want, aux="depth")


def test_long_chain_plain_walks_reach_gx():
    """The 70 000-node chain is longer than G1's 65 536-entry queue: G1 hands it to GX, which walks it again from the start.
    A few queries per call (GX has 8 slots, each walks ~70 000 serial levels)."""
    s, og, dg, _ = graph("deep")
    c = s.names[f"chain_{gs.LONG_CHAIN}"]
    fwd = c[[0, 0, 1, 2, 3000, 4400, 10, 70]].astype(np.int32)
    rev = c[[-1, -1, -2, -4000, -4401]].astype(np.int32)
    with pinned(dg, False, "default"):
        for name, got, want, aux, shift in (
            ("reachable", lambda: dg.reachable_many(fwd, DEEP, True), lambda: orc.reachable_many(og, fwd, DEEP, True), None, 0),
            ("bfs", lambda: dg.bfs_many(fwd, DEEP, True), lambda: orc.bfs_many(og, fwd, DEEP, True), "parent", -1),
            ("distances", lambda: dg.walk(dg.spec_distances(REACH4), fwd), lambda: orc.distances_many(og, fwd, REACH4), "depth", 0),
            ("impact", lambda: dg.impact_many(rev, DEEP), lambda: orc.impact_many(og, rev, DEEP), None, 0),
        ):
            res = got()
            t = tiers(dg)
            assert t["s1"] > 0 and t["g1"] > 0, (name, t)
            assert_walk_equal(res, want(), aux=aux, shift=shift, what=name)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_hub_rows_every_tier(config):
    """100 000-entry rows: S1's forecast calls them heavy, and whatever tier takes them next (big tier or G1) cannot hold them,
    so G1 hands them to GX."""
    s, og, dg, _ = graph("wide")
    nm = s.names
    fwd = np.asarray([nm["fhub"], nm["fhub"], nm["rep"], nm["clique"][0], nm["left"][0], nm["leaves"][7]], np.int32)
    rev = np.asarray([nm["rhub"], nm["rrep"], nm["rhub"], nm["right"][3], nm["clique"][5]], np.int32)
    with pinned(dg, False, config):
        for name, got, want, aux, shift in (
            ("reachable", lambda: dg.reachable_many(fwd, 3, False), lambda: orc.reachable_many(og, fwd, 3, False), None, 0),
            ("reachable-trav", lambda: dg.reachable_many(fwd, 3, True), lambda: orc.reachable_many(og, fwd, 3, True), None, 0),
            ("bfs", lambda: dg.bfs_many(fwd, 4, False), lambda: orc.bfs_many(og, fwd, 4, False), "parent", -1),
            ("distances", lambda: dg.walk(dg.spec_distances(REACH4), fwd), lambda: orc.distances_many(og, fwd, REACH4), "depth", 0),
            ("impact", lambda: dg.impact_many(rev, 3), lambda: orc.impact_many(og, rev, 3), None, 0),
        ):
            res = got()
            t = tiers(dg)
            assert t["s1_heavy"] > 0 and t["g1"] > 0, (name, t)
            assert_walk_equal(res, want(), aux=aux, shift=shift, what=name)


@pytest.mark.parametrize("dedup", DEDUP)
def test_repeated_neighbours_clique_and_bipartite(dedup):
    """Rows that repeat one neighbour on both sides of each 32-entry boundary, self-loops, the clique and the bipartite block,
    in a batch large enough to be de-duplicated."""
    s, og, dg, _ = graph("wide")
    nm = s.names
    sources = np.concatenate([[nm["rep"]] * 3, nm["fill"][:50], nm["clique"], nm["left"], nm["right"][:50], [nm["x"], nm["y"], nm["rrep"]]]).astype(np.int32)
    rsources = np.concatenate([[nm["rrep"]] * 3, nm["fill"][:20], nm["clique"][:100], nm["right"], [nm["x"], nm["y"], nm["rep"]]]).astype(np.int32)
    with pinned(dg, dedup, "default"):
        for depth in (1, 2, 3):
            assert_walk_equal(dg.reachable_many(sources, depth, False), orc.reachable_many(og, sources, depth, False), what=f"reachable {depth}")
            assert_walk_equal(dg.reachable_many(sources, depth, True), orc.reachable_many(og, sources, depth, True), what=f"reachable trav {depth}")
            want = orc.impact_many(og, rsources, depth)
            got = dg.impact_many(rsources, depth)
            assert_walk_equal(got, want, what=f"impact {depth}")
            np.testing.assert_array_equal(got.hist, want.hist)
        for mask in (REACH4, 0xFFFFFFFF):
            assert_walk_equal(dg.walk(dg.spec_distances(mask), sources), orc.distances_many(og, sources, mask), aux="depth", what=f"distances {mask:#x}")
            assert (dg.last_walk_stats()["groups"] > 0) == dedup
        assert_walk_equal(dg.bfs_many(sources, 3, True), orc.bfs_many(og, sources, 3, True), aux="parent", shift=-1, what="bfs")


@pytest.mark.parametrize("name", ["n1", "n2_self_loop", "n31_ring", "n32_ring", "n33_ring", "ghost_roots"])
def test_tiny_graphs(name):
    s, og, dg, _ = graph(name)
    n = og.n_nodes
    sources = np.concatenate([np.arange(n), np.arange(n), [-1, n, n + 40]]).astype(np.int32)
    for depth in (0, 1, 2, 40):
        want = orc.impact_many(og, sources, depth)
        got = dg.impact_many(sources, depth)
        assert_walk_equal(got, want, what=f"impact {depth}")
        np.testing.assert_array_equal(got.hist, want.hist)
        np.testing.assert_array_equal(got.flags & 2, want.flags & 2)
        assert_walk_equal(dg.reachable_many(sources, depth, False), orc.reachable_many(og, sources, depth, False), what=f"reachable {depth}")
        assert_walk_equal(dg.bfs_many(sources, depth, True), orc.bfs_many(og, sources, depth, True), aux="parent", shift=-1, what=f"bfs {depth}")
    assert_walk_equal(dg.walk(dg.spec_distances(0xFFFFFFFF), sources), orc.distances_many(og, sources, 0xFFFFFFFF), aux="depth", what="distances")
    root_off = np.arange(len(sources) + 1, dtype=np.int64)
    for direction in (1, 2, 3):
        want = orc.traverse_many(og, sources, root_off, direction=direction, max_depth=40, max_nodes=2, max_edges=-1)
        got = dg.walk(dg.spec_traverse(direction, 40, 2, -1, False, 0, False, False, True), sources, root_off)
        assert_traverse_equal(got, want, what=f"traverse {direction}")


# ── non-plain walks: budgets, recorded edges, multiple roots, target stop (always S1 -> G1 -> GX) ──────────────────────────────
def traverse(dg, og, roots, root_off, *, direction, max_depth, max_nodes=-1, max_edges=-1, traversable_only=False, include_roots=True):
    want = orc.traverse_many(og, roots, root_off, direction=direction, max_depth=max_depth, max_nodes=max_nodes, max_edges=max_edges,
                             traversable_only=traversable_only, include_roots=include_roots)
    spec = dg.spec_traverse(direction, max_depth, max_nodes, max_edges, traversable_only, 0, False, False, include_roots)
    return dg.walk(spec, roots, root_off), want


def ragged(lists):
    roots = np.concatenate([np.asarray(x, np.int32) for x in lists]) if lists else np.zeros(0, np.int32)
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in lists])
    return roots, off


@pytest.mark.parametrize("direction", [1, 2, 3])
def test_traverse_records_edges_through_gx(direction):
    """traverse_subgraph with recorded edges over the whole 70 000-node chain (restarted in GX after G1 fills) and the short shapes."""
    s, og, dg, _ = graph("deep")
    nm = s.names
    c = nm[f"chain_{gs.LONG_CHAIN}"]
    start = {1: c[0], 2: c[-1], 3: c[35_000]}[direction]
    lists = [[start], [nm["chain_300"][0]], [nm["chain_300"][-1]], [nm["bichain"][150]], [nm["comb_spine"][0]], [nm["chain_4100"][2000]],
             [nm["ghosts"][0]], [], [nm["pkgs"][0]], [nm["vulns"][-1]]]
    roots, off = ragged(lists)
    with pinned(dg, False, "default"):
        for max_depth in (DEEP, 256):
            got, want = traverse(dg, og, roots, off, direction=direction, max_depth=max_depth)
            t = tiers(dg)
            assert_traverse_equal(got, want, what=f"direction {direction} depth {max_depth}")
            assert t["s1"] > 0 and (t["g1"] > 0) == (max_depth == DEEP), t
        got, want = traverse(dg, og, roots, off, direction=direction, max_depth=DEEP, traversable_only=True, include_roots=False)
        assert_traverse_equal(got, want, what="traversable only, roots not marked")


def test_multi_root_queries():
    """33, 257 and 300 roots per query (more than S1's queue holds), with duplicates, ghosts and invalid ids."""
    s, og, dg, _ = graph("deep")
    nm = s.names
    n = og.n_nodes
    rng = np.random.default_rng(3)
    pool = np.concatenate([nm["chain_4100"], nm["chain_300"], nm["comb_spine"], nm["bichain"]])
    lists = []
    for k in (33, 257, 300, 33, 257, 300):
        r = rng.choice(pool, size=k).astype(np.int32)
        r[::11] = r[0]                                               # duplicates
        r[5] = nm["ghosts"][0]
        r[7] = -1
        r[9] = n + 2
        lists.append(r)
    lists.append(nm["chain_300"][:257])
    roots, off = ragged(lists)
    with pinned(dg, False, "default"):
        for cfg in (dict(direction=1, max_depth=3), dict(direction=3, max_depth=300), dict(direction=2, max_depth=DEEP, include_roots=False),
                    dict(direction=3, max_depth=5, max_nodes=600), dict(direction=1, max_depth=DEEP, max_edges=1000)):
            got, want = traverse(dg, og, roots, off, **cfg)
            t = tiers(dg)
            assert t["s1"] > 0, (cfg, t)
            assert_traverse_equal(got, want, what=str(cfg))


@pytest.mark.parametrize("budget", ["max_nodes", "max_edges"])
def test_budgets_on_hubs_and_repeated_rows(budget):
    """Node and edge budgets at 32-entry chunk boundaries and at G1's 65 536-entry queue, on the 100 000-entry rows and the row that
    repeats one neighbour across chunk boundaries."""
    s, og, dg, _ = graph("wide")
    nm = s.names
    lists = [[nm["fhub"]], [nm["rhub"]], [nm["rep"]], [nm["rrep"]], [nm["x"]], [nm["clique"][0]], [nm["left"][0]], [nm["rep"], nm["x"], nm["rep"]]]
    roots, off = ragged(lists)
    values = (1, 31, 32, 33, 65_535, 65_536, 65_537) if budget == "max_nodes" else (31, 32, 33, 64, 65)
    with pinned(dg, False, "default"):
        for v in values:
            for direction, max_depth in ((1, 1), (2, 1), (3, 3)):
                got, want = traverse(dg, og, roots, off, direction=direction, max_depth=max_depth, **{budget: v})
                t = tiers(dg)
                assert t["s1_heavy"] > 0, t
                if budget == "max_nodes" and v == 65_537 and direction != 3:
                    assert t["g1"] > 0, t                                # 65 537 visited (root included) do not fit G1's queue
                assert_traverse_equal(got, want, what=f"{budget}={v} direction {direction}")
        got, want = traverse(dg, og, roots, off, direction=3, max_depth=2, max_nodes=70_000, max_edges=150_000)
        assert tiers(dg)["g1"] > 0
        assert_traverse_equal(got, want, what="both budgets")


def test_shortest_paths_along_the_chains():
    s, og, dg, _ = graph("deep")
    nm = s.names
    c300, c70k = nm["chain_300"], nm[f"chain_{gs.LONG_CHAIN}"]
    pairs = [(c300[0], c300[255]), (c300[0], c300[256]), (c300[0], c300[-1]), (c70k[0], c70k[-1]), (c70k[0], c70k[65_536]),
             (nm["chain_4100"][0], nm["chain_4100"][-1]), (c300[0], nm["ghosts"][0]), (c300[0], nm["chain_254"][3]), (c300[-1], c300[0]),
             (nm["chain_257"][0], nm["chain_257"][0]), (nm["agents"][4], nm["vulns"][-1]), (nm["bichain"][299], nm["bichain"][0])]
    a = np.asarray([p[0] for p in pairs], np.int32)
    b = np.asarray([p[1] for p in pairs], np.int32)
    with pinned(dg, False, "default"):
        res = dg.shortest_path_many(a, b)
        t = tiers(dg)
    assert t["s1"] > 0 and t["g1"] > 0, t
    for q in range(len(a)):
        want = orc.shortest_path(og, int(a[q]), int(b[q]))
        if a[q] == b[q]:
            assert list(want) == [int(a[q])]
            continue
        found = bool(res.flags[q] & 4)
        assert found == (want is not None), q
        if found:
            nodes, parent = res.slice(q), res.aux(q, "parent")
            i = len(nodes) - 1
            while nodes[i] != b[q]:
                i -= 1
            path = []
            while i >= 0:
                path.append(int(nodes[i]))
                i = int(parent[i])
            assert path[::-1] == [int(x) for x in want], q
    assert len(orc.shortest_path(og, int(c70k[0]), int(c70k[-1]))) == gs.LONG_CHAIN


# ── consumers of the walk ──────────────────────────────────────────────────────────────────────────────────────────────────
@pytest.mark.parametrize("config", ["default", "mid-only", "warp-tiers-only"])
@pytest.mark.parametrize("dedup", DEDUP)
def test_dependency_reach_past_255_hops(dedup, config):
    """All ten arrays against the oracle; the package chain's min-hop is its depth + 2, up to 302 (past the 8-bit depth of S1 and
    the mid tier).  The 300 agents share one server, so a de-duplicated batch walks once for all of them."""
    s, og, dg, rank = graph("deep")
    agents = np.flatnonzero(og.node_type == gs.AGENT).astype(np.int32)
    want = orc.dependency_reach(og, agents, REACH4, VULN_PKG, rank)
    with pinned(dg, dedup, config):
        got = dg.dependency_reach(agents, REACH4, VULN_PKG)
        stats, t = dg.last_walk_stats(), tiers(dg)
    assert (stats["groups"] > 0) == dedup and t["s1"] > 0, (stats, t)
    for k in ("pkg_ids", "pkg_off", "pkg_agents", "pkg_minhop", "vuln_ids", "vuln_poff", "vuln_pkgs", "vuln_aoff", "vuln_agents", "vuln_minhop"):
        np.testing.assert_array_equal(np.asarray(got[k]), np.asarray(want[k]), err_msg=k)
    slot = {int(p): i for i, p in enumerate(got["pkg_ids"])}
    np.testing.assert_array_equal([got["pkg_minhop"][slot[int(p)]] for p in s.names["pkgs"]], np.arange(2, 303))


def test_bottleneck_scores_on_chains_and_hubs():
    """Raw scores == the oracle's subtree roll-up, and on a lone chain the closed form: node i lies inside n - 1 - i paths (the
    70 000-node chain is checked against the closed form alone: the roll-up goes one level per numpy round)."""
    s, og, dg, _ = graph("deep")
    nm = s.names
    c70k = nm[f"chain_{gs.LONG_CHAIN}"]
    for sources in ([nm["chain_300"][0]], [nm["chain_4100"][0], nm["chain_257"][0], nm["comb_spine"][0], nm["chain_300"][0]], [c70k[0]]):
        src = np.asarray(sources, np.int32)
        with pinned(dg, False, "default"):
            got = dg.bottleneck_scores(src)
            t = tiers(dg)
        assert t["s1"] > 0 and (t["g1"] > 0) == (src[0] == c70k[0]), t
        if len(src) == 1:
            c = nm["chain_300"] if src[0] == nm["chain_300"][0] else c70k
            k = len(c)
            want = np.zeros(og.n_nodes, np.uint64)
            want[c[1:]] = (k - 1 - np.arange(1, k)).astype(np.uint64)
            np.testing.assert_array_equal(got, want)
        if src[0] != c70k[0]:
            np.testing.assert_array_equal(got, subtree_counts(og, src))
    s, og, dg, _ = graph("wide")
    nm = s.names
    src = np.asarray([nm["fhub"], nm["rep"], nm["clique"][0], nm["left"][0], nm["fhub"]], np.int32)
    with pinned(dg, False, "default"):
        got = dg.bottleneck_scores(src)
        t = tiers(dg)
    assert t["s1_heavy"] > 0 and t["g1"] > 0, t
    np.testing.assert_array_equal(got, subtree_counts(og, src))
    assert int(got[nm["leaves"][0]]) == 2                             # the first leaf discovers rhub, once per fhub source


@pytest.mark.parametrize("dedup", DEDUP)
def test_finding_context_below_the_package_chain(dedup):
    """Blast radius of findings 12..302 hops below 300 agents (impact walks deeper than S1 and the mid tier count)."""
    s, og, dg, _ = graph("deep")
    nm = s.names
    v = nm["vulns"]
    findings = np.concatenate([v, v, np.repeat(v[-1], 300), [nm["ghosts"][0], -1, og.n_nodes + 1], nm["pkgs"][::10]]).astype(np.int32)
    with pinned(dg, dedup, "mid-only"):
        for depth in (4, 255, 256, 300, 400):
            got = dg.finding_context(findings, depth)
            t = tiers(dg)
            assert_context_equal(got, ocsf_oracle.finding_context(og, findings, depth))
            if depth >= 300:
                assert t["s1"] > 0 and t["mid"] > 0, t


# ── a G1 slot used again after an overflow ─────────────────────────────────────────────────────────────────────────────────────
def assert_repeats_equal(got, sources, want, uniq, what=""):
    """Every query of ``sources`` (drawn from ``uniq``) against the oracle's slice of its source, one matrix compare per source."""
    for j, u in enumerate(uniq):
        qs = np.flatnonzero(sources == u)
        a, b = int(want.off[j]), int(want.off[j + 1])
        np.testing.assert_array_equal(got.count[qs], b - a, err_msg=f"counts {what}")
        idx = got.start[qs][:, None] + np.arange(b - a)[None, :]
        bad = np.flatnonzero((got.nodes[idx] != want.nodes[a:b][None, :]).any(axis=1))
        assert bad.size == 0, f"{what}: {bad.size} of {qs.size} walks from one source differ (first: query {qs[bad[0]]})"


@pytest.mark.parametrize("kind", ["reachable", "bfs_traversable"])
def test_g1_slot_reuse_after_overflow(kind):
    """Walks that overflow G1 first in a batch, then short G1 walks along the same chain; then short walks alone, three times as
    many as G1 has warp slots (40 per SM), so that every slot walks some.  A visited bit that an overflowing walk leaves set in its
    slot's bitmap shows up as a node missing from a later walk on that slot.  The unfiltered reachable walk takes the lean row loop,
    the traversable-only BFS the filtered one: each has its own overflow exit."""
    s, og, dg, _ = graph("deep")
    c = s.names[f"chain_{gs.LONG_CHAIN}"]
    if kind == "reachable":
        dev, ora = (lambda q, d: dg.reachable_many(q, d, False)), (lambda q, d: orc.reachable_many(og, q, d, False))
    else:
        dev, ora = (lambda q, d: dg.bfs_many(q, d, True)), (lambda q, d: orc.bfs_many(og, q, d, True))
    first = np.concatenate([np.full(8, c[0]), np.full(2000, c[65_000])]).astype(np.int32)
    uniq1 = np.asarray([c[0], c[65_000]], np.int32)
    short = np.repeat(c[[60_000, 62_000, 65_000]], 6000).astype(np.int32)       # 600-level walks inside the first walks' queue range
    uniq2 = np.asarray(c[[60_000, 62_000, 65_000]], np.int32)
    with pinned(dg, False, "default"):
        got = dev(first, DEEP)
        t = tiers(dg)
        assert t["g1"] == 8, t
        assert_repeats_equal(got, first, ora(uniq1, DEEP), uniq1, "overflowing batch")
        want = ora(uniq2, 600)
        for k in range(2):
            got = dev(short, 600)
            t = tiers(dg)
            assert t["s1"] == len(short) and t["g1"] == 0, t
            assert_repeats_equal(got, short, want, uniq2, f"short walks, call {k}")
