"""Snapshot lookups on the H100: every golden case through ``B200GraphStore`` with the graph entering the cache by topology-first loading
and by ``save_graph``, against the unmodified SQLite store (oracle/make_lookup_golden.py), ``impact`` against the reference engine;
seeded random graphs against the numpy oracle, one above 1 M edges with hubs of more than 10^5 incident entries, self loops and
ghost endpoints; lookups from threads on one graph; and the lookup table and result objects freed.
"""

from __future__ import annotations

import sqlite3
from types import SimpleNamespace

import numpy as np
import pytest
from oracle.lookup_oracle import LookupOracle
from test_store_lookup import CASES, IDS, call, db_path  # noqa: F401  (db_path: the module fixture)

from agent_bom_b200.engine import DeviceGraph
from agent_bom_b200.graph import csr as csrmod
from agent_bom_b200.graph.container import UnifiedGraph
from agent_bom_b200.graph.model import UnifiedEdge, UnifiedNode
from agent_bom_b200.graph.snapshot import load_snapshot, normalize_graph_tenant_id
from agent_bom_b200.store import B200GraphStore

pytestmark = pytest.mark.gpu


def check(got, case):
    """The SQLite store's answer; ``node_context.impact`` is the reference engine's walk on the saved graph (no golden walk meets the
    SQLite store's caps, so the two are equal), rows to ids that are not nodes included."""
    want = case["expected"]
    if case["method"] == "node_context" and want is not None:
        want = dict(want, impact=case["impact_engine"])
    assert got == want


@pytest.fixture(scope="module")
def loading_store(db_path):  # noqa: F811
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


def saved_graph(db, tenant: str, scan: str) -> UnifiedGraph:
    """The snapshot as an in-memory graph, rows in stored order, edges to ids that are not nodes included."""
    snap = load_snapshot(db, tenant_id=tenant, scan_id=scan)
    g = UnifiedGraph(scan_id=scan, tenant_id=normalize_graph_tenant_id(tenant), created_at=snap.created_at)
    for nid in snap.csr.node_ids:
        n = snap.nodes[nid]
        g.add_node(UnifiedNode(id=nid, entity_type=n.entity_type, label=n.label, status=n.status, risk_score=n.risk_score, severity=n.severity))
    conn = sqlite3.connect(str(db))
    try:
        for s, t, r, d, w, tr in conn.execute("SELECT source_id, target_id, relationship, direction, weight, traversable FROM graph_edges "
                                              "WHERE tenant_id = ? AND scan_id = ? ORDER BY rowid", (g.tenant_id, scan)):
            g.add_edge(UnifiedEdge(s, t, r, direction=d, weight=w, traversable=bool(tr)))
    finally:
        conn.close()
    g.attack_paths, g.interaction_risks = list(snap.attack_paths), list(snap.interaction_risks)
    return g


@pytest.fixture(scope="module")
def saving_store(db_path):  # noqa: F811
    s = B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None, save_graph=lambda _g: None), max_graphs=8)
    for tenant, scan in (("lookup", "est40"), ("", "kat-a"), ("", "kat-b")):
        s.save_graph(saved_graph(db_path, tenant, scan))
    return s


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_lookup_by_loading(loading_store, case):
    check(call(loading_store, case), case)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_lookup_by_save_graph(saving_store, case):
    check(call(saving_store, case), case)


def random_graph(seed: int, n_real: int, ghosts: int, m: int, hubs: int = 0, hub_deg: int = 0):
    rng = np.random.default_rng(seed)
    ids = list(dict.fromkeys(f"n:{rng.integers(1 << 40):x}{chr(0x1F600 + i % 40) if i % 13 == 0 else ''}" for i in range(n_real + ghosts + 64)))
    ids = ids[: n_real + ghosts]
    n = len(ids)
    src = rng.integers(0, n, m)
    dst = rng.integers(0, n, m)
    loops = rng.integers(0, n_real, m // 100)
    src[: loops.size] = loops
    dst[: loops.size] = loops
    for h in range(hubs):                       # hub h is the source of hub_deg edges and the target of hub_deg more
        a = loops.size + 2 * h * hub_deg
        src[a: a + hub_deg] = h
        dst[a + hub_deg: a + 2 * hub_deg] = h
    rel = rng.integers(0, 6, m)
    key = {}
    for i, k in enumerate(zip(src.tolist(), dst.tolist(), rel.tolist())):
        key.setdefault(k, i)
    keep = np.fromiter(key.values(), np.int64)
    src, dst, rel = src[keep].astype(np.int32), dst[keep].astype(np.int32), rel[keep]
    flags = rng.integers(0, 4, keep.size).astype(np.uint8)
    types = np.concatenate([rng.integers(0, 24, n_real), np.full(n - n_real, 255)]).astype(np.uint8)
    types[: n_real][rng.random(n_real) < 0.01] = 254
    csr = csrmod.from_arrays(ids, types, src, dst, np.where(rel < 4, rel, 31).astype(np.uint8), flags, n_real=n_real)
    erel = rel.astype(np.uint8)                 # ranks of six relationship strings
    sev = np.where(rng.random(n_real) < 0.02, 255, rng.integers(0, 9, n_real)).astype(np.uint8)
    return csr, sev, erel


@pytest.mark.parametrize("seed,n_real,ghosts,m,hubs,hub_deg", [(1, 3_000, 200, 12_000, 0, 0), (2, 50, 0, 400, 2, 40),
                                                                 (3, 400_000, 20_000, 1_300_000, 2, 110_000)])
def test_random_graphs_match_oracle(seed, n_real, ghosts, m, hubs, hub_deg):
    csr, sev, erel = random_graph(seed, n_real, ghosts, m, hubs, hub_deg)
    if hub_deg >= 100_000:
        deg = np.diff(csr.fwd_off.astype(np.int64)) + np.diff(csr.rev_off.astype(np.int64))
        assert deg[:hubs].min() >= 100_000
    dg, o = DeviceGraph.upload(csr), LookupOracle(csr)
    rng = np.random.default_rng(seed + 100)
    try:
        got, want = dg.build_lookup_table(n_real, sev, erel), o.build_lookup_table(n_real, sev, erel)
        for k in want:
            assert np.array_equal(got[k], want[k]), k
        sets = [np.arange(max(hubs, 1)), rng.integers(0, csr.n_nodes, 50), rng.integers(0, csr.n_nodes, 5_000), np.zeros(0, np.int64),
                np.concatenate([np.arange(hubs), np.arange(hubs)])]
        for s in sets:
            assert np.array_equal(dg.incident_edges(s), o.incident_edges(s))
        for u in list(range(hubs)) + rng.integers(0, csr.n_nodes, 30).tolist():
            assert np.array_equal(dg.context_edges(u), o.context_edges(u)), u
    finally:
        dg.close()


def test_context_needs_the_table_and_the_table_every_edge():
    csr, sev, erel = random_graph(4, 100, 0, 300)
    dg = DeviceGraph.upload(csr)
    try:
        with pytest.raises(RuntimeError):
            dg.context_edges(0)
        with pytest.raises(RuntimeError, match="relationship slots"):
            dg.build_lookup_table(csr.n_real, sev, erel[:-1])
        with pytest.raises(RuntimeError):
            dg.context_edges(0)
    finally:
        dg.close()


def test_concurrent_lookups_on_one_graph():
    from concurrent.futures import ThreadPoolExecutor

    csr, sev, erel = random_graph(5, 50_000, 1_000, 300_000, 1, 20_000)
    dg, o = DeviceGraph.upload(csr), LookupOracle(csr)
    rng = np.random.default_rng(6)
    try:
        dg.build_lookup_table(csr.n_real, sev, erel)
        o.build_lookup_table(csr.n_real, sev, erel)
        sets = [rng.integers(0, csr.n_nodes, int(k)) for k in rng.integers(1, 3_000, 24)]
        nodes = [0] + rng.integers(0, csr.n_nodes, 23).tolist()
        with ThreadPoolExecutor(8) as ex:
            edges = list(ex.map(dg.incident_edges, sets))
            ctx = list(ex.map(dg.context_edges, nodes))
        for s, e in zip(sets, edges):
            assert np.array_equal(e, o.incident_edges(s))
        for u, e in zip(nodes, ctx):
            assert np.array_equal(e, o.context_edges(u))
    finally:
        dg.close()


def test_table_and_results_are_freed():
    import torch

    csr, sev, erel = random_graph(7, 300_000, 0, 900_000, 1, 50_000)

    def cycle():
        dg = DeviceGraph.upload(csr)
        try:
            dg.build_lookup_table(csr.n_real, sev, erel)
            assert dg.lookup_table_bytes() >= csr.n_edges
            for _ in range(3):
                dg.incident_edges(np.arange(1_000))
                dg.context_edges(0)
        finally:
            dg.close()

    torch.cuda.mem_get_info()
    cycle()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20


def test_store_drops_its_tables_with_the_graph(db_path):  # noqa: F811
    import torch

    def cycle():
        s = B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))
        s.snapshot_stats(tenant_id="lookup", scan_id="est40")
        s.node_context(tenant_id="lookup", scan_id="est40", node_id="agent:agent-00007")
        s.edges_for_node_ids(tenant_id="lookup", scan_id="est40", node_ids={"agent:agent-00007"})
        g = s._graph("lookup", "est40")
        assert g._lookup is not None and g.device_graph.lookup_table_bytes() > 0
        s.node_context(tenant_id="", scan_id="kat-a", node_id="tool:t")       # builds the graph with the left-out rows
        assert s._graph("", "kat-a")._lookup._full_graph is not None
        del s, g

    import gc

    cycle()
    gc.collect()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
        gc.collect()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20
