"""Semantic clusters on the device: every reference golden through ``semantic_clusters`` / ``semantic_clusters_view`` and through
``B200GraphStore`` (standalone and after ``save_graph``), a SQLite snapshot against the numpy oracle, seeded random graphs against
the oracle (one cluster holding every node over more than a million edges, more than 65,536 clusters, a graph without clusters,
an empty graph), and the tables freed with the graph."""

from __future__ import annotations

import gzip
import tempfile
from pathlib import Path

import numpy as np
import pytest

from clusters_golden import NAMES, case, graph, roundtrip
from oracle.clusters_oracle import ClusterOracle

from agent_bom_b200.graph import clusters as cl

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", NAMES)
def test_goldens_through_the_function(name):
    c = case(name)
    g = graph(name)
    for m in ("1", "2", "3"):
        got = cl.semantic_clusters(g, min_members=int(m))
        assert roundtrip([x.to_dict() for x in got]) == c["clusters"][m]["clusters"], f"min_members={m}"
        assert cl.semantic_cluster_stats(got) == c["clusters"][m]["stats"]
    for v in c["views"]:
        assert roundtrip(cl.semantic_clusters_view(g, **v["params"])) == v["body"], v["params"]


@pytest.mark.parametrize("name", NAMES)
def test_goldens_through_the_store(name):
    from agent_bom_b200.store import B200GraphStore

    c = case(name)
    g = graph(name)
    store = B200GraphStore()
    empty = store.semantic_clusters_view(tenant_id=c["tenant_id"], scan_id=c["scan_id"])
    assert empty["clusters"] == [] and empty["stats"]["cluster_count"] == 0
    store.save_graph(g)
    for v in c["views"]:
        assert roundtrip(store.semantic_clusters_view(tenant_id=c["tenant_id"], scan_id=c["scan_id"], **v["params"])) == v["body"], v["params"]
    with pytest.raises(ValueError, match="Unknown semantic cluster kind"):
        store.semantic_clusters_view(tenant_id=c["tenant_id"], kinds="nope")


def test_snapshot_graph_matches_oracle():
    from agent_bom_b200.graph import load_snapshot

    src = Path(__file__).resolve().parent / "golden" / "snapshot" / "graph.sqlite.gz"
    with tempfile.TemporaryDirectory() as td:
        db = Path(td) / "graph.sqlite"
        db.write_bytes(gzip.decompress(src.read_bytes()))
        for tenant, scan in (("default", "scan-a"), ("default", "scan-b"), ("acme", "scan-a")):
            g = load_snapshot(db, tenant_id=tenant, scan_id=scan)
            want_g = load_snapshot(db, tenant_id=tenant, scan_id=scan)
            want_g._dg = ClusterOracle(want_g.csr)
            assert len(g.nodes) > 0
            for m in (1, 2):
                assert roundtrip([x.to_dict() for x in cl.semantic_clusters(g, min_members=m)]) == \
                    roundtrip([x.to_dict() for x in cl.semantic_clusters(want_g, min_members=m)])
            assert roundtrip(cl.semantic_clusters_view(g, min_members=1)) == roundtrip(cl.semantic_clusters_view(want_g, min_members=1))


def random_case(seed, n_real, n_ghost, n_edges, k, *, all_cluster=False):
    from agent_bom_b200.graph import csr as csrmod

    rng = np.random.default_rng(seed)
    n = n_real + n_ghost
    src = rng.integers(0, n, n_edges).astype(np.int32)
    dst = np.where(rng.random(n_edges) < 0.05, src, rng.integers(0, n, n_edges)).astype(np.int32)    # some self loops
    rel = rng.integers(0, 32, n_edges).astype(np.uint8)                                               # 31: outside the enum
    flags = rng.integers(0, 4, n_edges).astype(np.uint8)                                              # traversable / bidirectional
    node_type = np.concatenate([rng.integers(0, 24, n_real), np.full(n_ghost, 255)]).astype(np.uint8)
    host = csrmod.from_arrays(None, node_type, src, dst, rel, flags, n_real=n_real, node_rank=rng.permutation(n).astype(np.int32))
    codes = np.full((n, 2), -1, np.int32)
    if k:
        if all_cluster:
            codes[:n_real, 0] = 0
            codes[:n_real, 1] = np.where(rng.random(n_real) < 0.8, rng.integers(1, k, n_real), -1)
        else:
            codes[:n_real, 0] = np.where(rng.random(n_real) < 0.7, rng.integers(0, k, n_real), -1)
            codes[:n_real, 1] = np.where(rng.random(n_real) < 0.5, rng.integers(0, k, n_real), -1)
            codes[codes[:, 1] == codes[:, 0], 1] = -1
    level = rng.integers(0, 5, n).astype(np.uint8)
    risk = np.round(rng.random(n) * 100.0, 3)
    etype = rng.integers(0, 64, n).astype(np.uint8)
    return host, codes, level, risk, etype


def check_against_oracle(host, k, codes, level, risk, etype):
    from agent_bom_b200.engine import DeviceGraph

    dg = DeviceGraph.upload(host)
    try:
        got = dg.build_clusters(k, codes, level, risk, etype)
        orc = ClusterOracle(host)
        want = orc.build_clusters(k, codes, level, risk, etype)
        for f in ("count", "max_risk", "hist", "type_mask", "rel_nnz"):
            assert np.array_equal(got[f], want[f]), f
        present = np.flatnonzero(want["count"] > 0)
        for sel in (present, present[::-1][:300], present[:1]):
            nm, npairs = int(want["count"][sel].sum()), int(want["rel_nnz"][sel].sum())
            gm, gr, gc = dg.fetch_clusters(sel, nm, npairs)
            wm, wr, wc = orc.fetch_clusters(sel, nm, npairs)
            assert np.array_equal(gm, wm) and np.array_equal(gr, wr) and np.array_equal(gc, wc)
        return got
    finally:
        dg.close()


def test_random_all_node_cluster_over_a_million_edges():
    host, codes, level, risk, etype = random_case(7, 200_000, 1_000, 1_200_000, 5_000, all_cluster=True)
    got = check_against_oracle(host, 5_000, codes, level, risk, etype)
    assert got["count"][0] == 200_000


def test_random_more_than_65536_clusters():
    host, codes, level, risk, etype = random_case(8, 300_000, 5_000, 600_000, 100_000)
    got = check_against_oracle(host, 100_000, codes, level, risk, etype)
    assert (got["count"] > 0).sum() > 65_536


def test_random_graph_without_clusters():
    host, codes, level, risk, etype = random_case(9, 5_000, 10, 20_000, 0)
    got = check_against_oracle(host, 0, codes, level, risk, etype)
    assert got["count"].shape == (0,)


def test_graph_whose_nodes_form_no_cluster_and_empty_graph():
    from agent_bom_b200.graph import UnifiedGraph, UnifiedNode

    g = UnifiedGraph(scan_id="s")
    g.add_node(UnifiedNode(id="m", entity_type="model", label="m"))
    assert cl.semantic_clusters(g, min_members=1) == []
    assert cl.semantic_clusters_view(g)["stats"]["cluster_count"] == 0
    assert cl.semantic_clusters_view(UnifiedGraph())["clusters"] == []


def test_cluster_tables_are_freed_with_the_graph():
    import torch

    from agent_bom_b200.engine import DeviceGraph

    host, codes, level, risk, etype = random_case(10, 2_000_000, 0, 4_000_000, 500_000)

    def cycle():
        dg = DeviceGraph.upload(host)
        dg.build_clusters(500_000, codes, level, risk, etype)
        dg.close()

    torch.cuda.mem_get_info()
    cycle()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
    free_after, _ = torch.cuda.mem_get_info()
    drop = free_before - free_after
    assert drop <= 8 << 20, f"two freed graphs kept {drop / 2**20:.1f} MiB of device memory"
