"""Parity tests proper: the CUDA engine (through the C ABI) against the CPU oracle and the golden fixtures.

Bit-exact bar: node ORDER (== the reference's discovery order), parents, depths,
recorded-edge order, histograms, truncation flags, exposure-path rows and
dependency-reach tuples must be identical arrays.  Needs a GPU.
"""

from __future__ import annotations

import numpy as np
import pytest

from golden_util import ALL_FIXTURES, edge_arrays, load, node_rank, rank_path_rows, seeded_graph
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

DYN = (1 << 26) | (1 << 27) | (1 << 28)
REACH4 = (1 << 1) | (1 << 2) | (1 << 7) | (1 << 3)
LATERAL = (1 << 13) | (1 << 14) | (1 << 15)
VULN_PKG = (1 << 8) | (1 << 9)


def device_graph(src, dst, rel, flags, node_type, rank=None):
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    h = csrmod.from_arrays(None, node_type, src, dst, rel, flags, node_rank=rank)
    return DeviceGraph.upload(h), h


_cache: dict = {}


def graphs_for(key):
    """(oracle graph, device graph, node_type) for a seeded-random spec or a golden fixture name."""
    if key in _cache:
        return _cache[key]
    if isinstance(key, str):
        doc = load(key)
        src, dst, rel, flags = edge_arrays(doc)
        nt = np.asarray(doc["node_types"], dtype=np.uint8)
        rank = node_rank(doc["node_ids"])
    else:
        n, e, seed = key
        src, dst, rel, flags, nt = seeded_graph(n, e, seed)
        rank = np.random.default_rng(seed + 1).permutation(n).astype(np.int32)
    og = orc.build_csr(len(nt), src, dst, rel, flags, nt)
    dg, h = device_graph(src, dst, rel, flags, nt, rank)
    _cache[key] = (og, dg, nt, rank, h)
    return _cache[key]


SEEDED = [(64, 300, 1), (2000, 12000, 2), (6000, 90000, 3), (30000, 400000, 4)]


def assert_slices_equal(gpu, ora, *, gpu_aux=None, ora_aux=True, aux_shift=0):
    assert len(gpu) == len(ora.off) - 1
    counts = np.diff(ora.off)
    np.testing.assert_array_equal(gpu.count, counts.astype(np.int32))
    for q in range(len(gpu)):
        a, b = int(ora.off[q]), int(ora.off[q + 1])
        np.testing.assert_array_equal(gpu.slice(q), ora.nodes[a:b], err_msg=f"query {q} node order")
        if gpu_aux is not None:
            np.testing.assert_array_equal(gpu.aux(q, gpu_aux) + aux_shift, ora.aux[a:b], err_msg=f"query {q} {gpu_aux}")


def test_csr_build_matches_oracle_model():
    """a1: the library's counting-sort CSR == numpy restatement of add_edge's adjacency lists."""
    for key in SEEDED[:3] + ["kat_probe", "estate_dense_40"]:
        og, _, _, _, h = graphs_for(key)
        for name in ("fwd_off", "fwd_nbr", "fwd_meta", "fwd_eid", "rev_off", "rev_nbr", "rev_meta", "rev_eid"):
            np.testing.assert_array_equal(getattr(h, name), getattr(og, name), err_msg=name)


@pytest.mark.parametrize("dedup", [True, False])
@pytest.mark.parametrize("key", SEEDED + ["estate_150", "estate_dense_40"])
def test_impact_many(key, dedup):
    og, dg, nt, _, _ = graphs_for(key)
    dg.set_dedup(dedup)
    rng = np.random.default_rng(7)
    n = og.n_nodes
    sources = np.concatenate([rng.integers(0, n, size=min(4000, 4 * n)), np.arange(min(n, 64)), [-1, n + 3]]).astype(np.int32)
    for depth in (4, 1, 0, 7):
        want = orc.impact_many(og, sources, depth)
        got = dg.impact_many(sources, depth)
        assert_slices_equal(got, want)
        np.testing.assert_array_equal(got.maxd, want.maxd)
        np.testing.assert_array_equal(got.hist, want.hist)
        np.testing.assert_array_equal(got.flags & 2, want.flags & 2)
    dg.set_dedup(True)


@pytest.mark.parametrize("key", SEEDED + ["estate_150", "estate_dense_40"])
def test_bfs_order_and_parents(key):
    og, dg, _, _, _ = graphs_for(key)
    rng = np.random.default_rng(11)
    n = og.n_nodes
    sources = np.concatenate([rng.integers(0, n, size=min(1500, 2 * n)), np.arange(min(n, 32))]).astype(np.int32)
    for depth, trav in ((4, True), (2, False), (6, True)):
        want = orc.bfs_many(og, sources, depth, trav)
        got = dg.bfs_many(sources, depth, trav)
        # device parents index the full queue (root at 0); the oracle's index the emitted slice (root = -1)
        assert_slices_equal(got, want, gpu_aux="parent", aux_shift=-1)


@pytest.mark.parametrize("key", SEEDED + ["estate_150"])
def test_reachable_from(key):
    og, dg, _, _, _ = graphs_for(key)
    rng = np.random.default_rng(13)
    sources = rng.integers(0, og.n_nodes, size=800).astype(np.int32)
    for depth, trav in ((6, False), (3, True)):
        assert_slices_equal(dg.reachable_many(sources, depth, trav), orc.reachable_many(og, sources, depth, trav))


@pytest.mark.parametrize("dedup", [True, False])
@pytest.mark.parametrize("key", SEEDED + ["estate_150", "estate_dense_40"])
def test_distances_unbounded_masked(key, dedup):
    """_bfs_distances_along: unbounded depth — on the big seeded graphs this exercises the overflow tiers."""
    og, dg, _, _, _ = graphs_for(key)
    dg.set_dedup(dedup)
    try:
        rng = np.random.default_rng(17)
        sources = rng.integers(0, og.n_nodes, size=300).astype(np.int32)
        for mask in (REACH4, 0xFFFFFFFF, LATERAL | REACH4):
            want = orc.distances_many(og, sources, mask)
            got = dg.walk(dg.spec_distances(mask), sources)
            assert_slices_equal(got, want, gpu_aux="depth")
            np.testing.assert_array_equal(got.maxd, want.maxd)
    finally:
        dg.set_dedup(True)


@pytest.mark.parametrize("key", SEEDED + ["estate_150", "estate_dense_40", "kat_probe"])
def test_traverse_subgraph_walks(key):
    og, dg, _, _, _ = graphs_for(key)
    rng = np.random.default_rng(19)
    n = og.n_nodes
    nq = 200
    sizes = rng.integers(1, 5, size=nq)
    root_off = np.zeros(nq + 1, dtype=np.int64)
    root_off[1:] = np.cumsum(sizes)
    roots = rng.integers(-1, n + 1, size=int(root_off[-1])).astype(np.int32)  # includes invalid and duplicate roots
    roots[::7] = roots[0]
    configs = [
        dict(direction=1, max_depth=4), dict(direction=2, max_depth=4), dict(direction=3, max_depth=3),
        dict(direction=3, max_depth=4, traversable_only=True), dict(direction=1, max_depth=5, rel_mask=REACH4),
        dict(direction=3, max_depth=2, rel_mask=LATERAL), dict(direction=3, max_depth=4, static=True), dict(direction=3, max_depth=4, dynamic=True),
        dict(direction=3, max_depth=4, include_roots=False), dict(direction=1, max_depth=3, include_roots=False),
        dict(direction=3, max_depth=4, max_nodes=3), dict(direction=3, max_depth=4, max_edges=4), dict(direction=3, max_depth=6, max_nodes=50, max_edges=300),
        dict(direction=2, max_depth=5, max_nodes=500, max_edges=10_000), dict(direction=3, max_depth=0), dict(direction=1, max_depth=1, max_nodes=1),
        dict(direction=3, max_depth=10, max_nodes=5000, max_edges=25_000),
    ]
    for cfg in configs:
        mask = cfg.get("rel_mask", 0)
        omask = mask or 0xFFFFFFFF
        if cfg.get("static"):
            omask &= ~DYN
        if cfg.get("dynamic"):
            omask &= DYN
        inc = cfg.get("include_roots", True)
        want = orc.traverse_many(og, roots, root_off, direction=cfg["direction"], max_depth=cfg["max_depth"], max_nodes=cfg.get("max_nodes", -1),
                                 max_edges=cfg.get("max_edges", -1), rel_mask=omask, traversable_only=cfg.get("traversable_only", False), include_roots=inc)
        spec = dg.spec_traverse(cfg["direction"], cfg["max_depth"], cfg.get("max_nodes", -1), cfg.get("max_edges", -1), cfg.get("traversable_only", False),
                                mask, cfg.get("static", False), cfg.get("dynamic", False), inc)
        got = dg.walk(spec, roots, root_off)
        assert_slices_equal(got, want, gpu_aux="depth")
        np.testing.assert_array_equal(got.flags & 1, want.flags & 1, err_msg=f"truncated {cfg}")
        np.testing.assert_array_equal(got.ecount, np.diff(want.eoff), err_msg=f"edge counts {cfg}")
        for q in range(nq):
            a, b = int(want.eoff[q]), int(want.eoff[q + 1])
            np.testing.assert_array_equal(got.edge_slice(q), want.edges[a:b], err_msg=f"edges q={q} {cfg}")


@pytest.mark.parametrize("key", SEEDED[:3] + ["estate_150"])
def test_shortest_path(key):
    og, dg, nt, _, _ = graphs_for(key)
    rng = np.random.default_rng(23)
    n = og.n_nodes
    a = rng.integers(0, n, size=300).astype(np.int32)
    b = rng.integers(0, n, size=300).astype(np.int32)
    res = dg.shortest_path_many(a, b)
    for q in range(len(a)):
        want = orc.shortest_path(og, int(a[q]), int(b[q]))
        if nt[a[q]] == 255 or nt[b[q]] == 255:
            assert want is None
            continue
        if a[q] == b[q]:
            assert list(want) == [int(a[q])]
            continue
        found = bool(res.flags[q] & 4)
        assert found == (want is not None)
        if found:
            nodes, parent = res.slice(q), res.aux(q, "parent")
            i = len(nodes) - 1
            while nodes[i] != b[q]:
                i -= 1
            path = []
            while i >= 0:
                path.append(int(nodes[i]))
                i = int(parent[i])
            assert path[::-1] == [int(x) for x in want]


@pytest.mark.parametrize("key", SEEDED + ALL_FIXTURES)
def test_exposure_path_rows(key):
    og, dg, nt, rank, _ = graphs_for(key)
    findings = np.flatnonzero((nt == 8) | (nt == 9)).astype(np.int32)
    extra = np.asarray([0, og.n_nodes - 1, -1], dtype=np.int32)  # non-findings / invalid ids yield no rows
    f = np.concatenate([findings, extra])
    want = orc.derived_paths(og, f, rank)
    got = dg.exposure_paths_many(f)
    np.testing.assert_array_equal(got.hops, want.hops)
    np.testing.assert_array_equal(got.rels, want.rels)
    np.testing.assert_array_equal(got.ncred, want.ncred)
    np.testing.assert_array_equal(got.ntool, want.ntool)
    assert int(got.off[-1]) == want.hops.shape[0]
    # the factorised form that crossed PCIe expands to the same rows
    nf = len(f)
    k = 0
    for i in range(nf):
        for l in range(int(got.link_off[i]), int(got.link_off[i + 1])):
            n = int(got.link_row_off[l + 1] - got.link_row_off[l])
            t0 = int(got.link_template[l])
            assert int(got.link_row_off[l]) == k
            np.testing.assert_array_equal(got.template[t0: t0 + n, 0], got.hops[k: k + n, 0])
            np.testing.assert_array_equal(got.template[t0: t0 + n, 2], got.ncred[k: k + n])
            assert (got.hops[k: k + n, 3] == f[i]).all()
            k += n
        if i > 200:
            break


@pytest.mark.parametrize("name", ALL_FIXTURES)
def test_derived_paths_vs_reference_golden(name):
    """End to end against the unmodified reference's ranked AttackPath list (api/routes/graph.py:686-786)."""
    doc = load(name)
    og, dg, _, rank, _ = graphs_for(name)
    rows = dg.exposure_paths_many(np.asarray(doc["findings"], dtype=np.int32))
    got = rank_path_rows(doc, rows, og)
    assert got == doc["cases"]["derived_paths"]


@pytest.mark.parametrize("name", ALL_FIXTURES)
def test_impact_vs_reference_golden(name):
    doc = load(name)
    _, dg, _, _, _ = graphs_for(name)
    cases = doc["cases"]["impact"]
    for depth in sorted({c["d"] for c in cases}):
        sub = [c for c in cases if c["d"] == depth]
        res = dg.impact_many([c["s"] for c in sub], depth)
        for q, c in enumerate(sub):
            assert sorted(int(x) for x in res.slice(q)) == c["nodes"]
            assert int(res.maxd[q]) == c["maxd"] and int(res.count[q]) == c["count"]
            assert res.hist_dict(q) == c["by_type"]


@pytest.mark.parametrize("name", ALL_FIXTURES)
def test_bfs_vs_reference_golden(name):
    doc = load(name)
    _, dg, _, _, _ = graphs_for(name)
    cases = doc["cases"]["bfs"]
    for key in sorted({(c["d"], c["t"]) for c in cases}):
        sub = [c for c in cases if (c["d"], c["t"]) == key]
        res = dg.bfs_many([c["s"] for c in sub], key[0], key[1])
        for q, c in enumerate(sub):
            nodes, parent = res.slice(q), res.aux(q, "parent")
            paths = []
            for i in range(len(nodes)):
                p = int(parent[i]) - 1
                paths.append(([c["s"]] if p < 0 else paths[p]) + [int(nodes[i])])
            assert paths == c["paths"]


@pytest.mark.parametrize("dedup", [True, False])
@pytest.mark.parametrize("key", SEEDED[:3] + ALL_FIXTURES)
def test_dependency_reach(key, dedup):
    og, dg, nt, rank, _ = graphs_for(key)
    dg.set_dedup(dedup)
    try:
        agents = np.flatnonzero(nt == 0).astype(np.int32)
        want = orc.dependency_reach(og, agents, REACH4, VULN_PKG, rank)
        got = dg.dependency_reach(agents, REACH4, VULN_PKG)
        for k in ("pkg_ids", "pkg_off", "pkg_agents", "pkg_minhop", "vuln_ids", "vuln_poff", "vuln_pkgs", "vuln_aoff", "vuln_agents", "vuln_minhop"):
            np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    finally:
        dg.set_dedup(True)


@pytest.mark.parametrize("dedup", [True, False])
@pytest.mark.parametrize("key", [SEEDED[2], "mesh_inventory", "estate_dense_40"])
def test_dependency_reach_device_merge_of_agent_shards(key, dedup):
    """a9 across ranks: per-shard device results merged by the CUDA path of dist.merge_dependency_reach (64-bit key sort on the
    device) == the numpy merge == the unsplit call."""
    from agent_bom_b200.dist import REACH_KEYS, merge_dependency_reach

    og, dg, nt, rank, _ = graphs_for(key)
    dg.set_dedup(dedup)
    try:
        agents = np.flatnonzero(nt == 0).astype(np.int32)
        whole = dg.dependency_reach(agents, REACH4, VULN_PKG)
        for cuts in ([0, len(agents) // 2, len(agents)], [0, 1, len(agents) // 3, len(agents) // 3, len(agents)]):
            parts = [dg.dependency_reach(agents[a:b], REACH4, VULN_PKG) for a, b in zip(cuts, cuts[1:])]
            on_device = merge_dependency_reach(parts, rank, "cuda:0")
            on_host = merge_dependency_reach(parts, rank)
            for k in REACH_KEYS:
                np.testing.assert_array_equal(np.asarray(on_device[k]), np.asarray(whole[k]), err_msg=k)
                np.testing.assert_array_equal(np.asarray(on_host[k]), np.asarray(whole[k]), err_msg=k)
    finally:
        dg.set_dedup(True)


def test_exposure_many_matches_separate_calls():
    og, dg, nt, _, _ = graphs_for("estate_dense_40")
    findings = np.flatnonzero((nt == 8) | (nt == 9)).astype(np.int32)
    w, p = dg.exposure_many(findings, 4)
    w2 = dg.impact_many(findings, 4)
    p2 = dg.exposure_paths_many(findings)
    for q in range(len(findings)):
        np.testing.assert_array_equal(w.slice(q), w2.slice(q))
    np.testing.assert_array_equal(w.hist, w2.hist)
    np.testing.assert_array_equal(p.hops, p2.hops)
    np.testing.assert_array_equal(p.rels, p2.rels)


def test_empty_and_ragged_batches():
    og, dg, _, _, _ = graphs_for(SEEDED[0])
    res = dg.impact_many(np.zeros(0, dtype=np.int32), 4)
    assert len(res) == 0 and res.nodes.shape[0] == 0
    rows = dg.exposure_paths_many(np.zeros(0, dtype=np.int32))
    assert rows.hops.shape == (0, 4)
    # a query with no roots at all
    spec = dg.spec_traverse(3, 4, -1, -1, False, 0, False, False, True)
    got = dg.walk(spec, np.asarray([1, 2], dtype=np.int32), np.asarray([0, 0, 2], dtype=np.int64))
    assert int(got.count[0]) == 0 and int(got.flags[0]) & 2


def test_whole_graph_walks_reach_the_last_tier():
    """Unbounded walks over a dense seeded graph outgrow the shared-memory and bounded-queue tiers (S1 -> G1 -> GX).  G1's queue
    (n + 4096 entries here) holds any walk of this graph, so it is G1's level forecast that hands them to GX; the 70 000-node chain
    of test_gpu_graph_shapes.py fills G1's queue instead."""
    og, dg, _, _, _ = graphs_for((30000, 400000, 4))
    rng = np.random.default_rng(29)
    sources = rng.integers(0, og.n_nodes, size=12).astype(np.int32)
    want = orc.distances_many(og, sources, 0xFFFFFFFF)
    assert int(np.diff(want.off).max()) > 20000          # really whole-graph
    for dedup in (True, False):
        dg.set_dedup(dedup)
        got = dg.walk(dg.spec_distances(0xFFFFFFFF), sources)
        t = dg.last_walk_tier_counts()["first"]
        assert t["s1"] == len(sources) and t["g1"] > 0, t
        assert_slices_equal(got, want, gpu_aux="depth")
    dg.set_dedup(True)
    spec = dg.spec_traverse(3, 12, -1, -1, False, 0, False, False, True)
    roots = sources[:4]
    root_off = np.arange(5, dtype=np.int64)
    want_t = orc.traverse_many(og, roots, root_off, direction=3, max_depth=12)
    got_t = dg.walk(spec, roots, root_off)
    t = dg.last_walk_tier_counts()["first"]
    assert t["s1"] == len(roots) and t["g1"] > 0, t
    assert_slices_equal(got_t, want_t, gpu_aux="depth")
    np.testing.assert_array_equal(got_t.ecount, np.diff(want_t.eoff))
