"""Snapshot tables that live on a graph handle (semantic clusters, snapshot diff, lookup, node search, compliance) across rebuilds.

Each feature's table is built on one graph with inputs A, then a call the host argument checks reject must leave A served, then the
table is rebuilt with inputs B (other contents, and another size where the graph allows it) and, where the feature allows one, with an
empty input; every answer is checked against the feature's oracle, and the table's device bytes against a fresh graph built with the
same input.  A second thread reading ``*_table_bytes`` while the first rebuilds sees only A's or B's value, and free device memory
returns to its level across three upload / rebuild / close cycles.
"""

from __future__ import annotations

import threading

import numpy as np
import pytest
from oracle.clusters_oracle import ClusterOracle
from oracle.compliance_oracle import ComplianceOracle
from oracle.delta_oracle import DeltaOracle
from oracle.lookup_oracle import LookupOracle
from oracle.search_oracle import SearchOracle
from test_gpu_clusters import random_case
from test_gpu_compliance import random_table as compliance_inputs
from test_gpu_delta import pair
from test_gpu_search import random_table as search_inputs
from test_gpu_store_lookup import random_graph

from agent_bom_b200 import _lib
from agent_bom_b200.engine import DeviceGraph
from agent_bom_b200.graph import csr as csrmod
from agent_bom_b200.graph import delta
from agent_bom_b200.graph.search import MODE_ALL, MODE_FTS, MODE_LIKE, fold_table

pytestmark = pytest.mark.gpu


def one_node_graph() -> DeviceGraph:
    z = np.zeros(0, np.int32)
    return DeviceGraph.upload(csrmod.from_arrays(["n"], np.zeros(1, np.uint8), z, z, z.astype(np.uint8), z.astype(np.uint8), n_real=1))


def fresh_bytes(upload, build, table_bytes) -> int:
    dg = upload()
    try:
        build(dg)
        return table_bytes(dg)
    finally:
        dg.close()


def read_while_rebuilding(build_a, build_b, table_bytes, rounds: int = 6) -> set[int]:
    """Values ``table_bytes`` returns on a second thread while this one rebuilds B, A, B, ... from A."""
    build_a()
    seen: set[int] = set()
    done = threading.Event()

    def reader():
        while not done.is_set():
            seen.add(table_bytes())

    t = threading.Thread(target=reader)
    t.start()
    try:
        for r in range(rounds):
            (build_b if r % 2 == 0 else build_a)()
    finally:
        done.set()
        t.join()
    seen.add(table_bytes())
    return seen


# ── semantic clusters ──
def cluster_inputs(seed: int, k: int, n_real: int = 3_000, n_ghost: int = 100):
    _, codes, level, risk, etype = random_case(seed, n_real, n_ghost, 1, k)
    return k, codes, level, risk, etype


def check_clusters(dg, orc, inputs):
    got, want = dg.build_clusters(*inputs), orc.build_clusters(*inputs)
    for f in ("count", "max_risk", "hist", "type_mask", "rel_nnz"):
        assert np.array_equal(got[f], want[f]), f
    check_cluster_members(dg, orc, want)


def check_cluster_members(dg, orc, want):
    sel = np.flatnonzero(want["count"] > 0)
    nm, npairs = int(want["count"][sel].sum()), int(want["rel_nnz"][sel].sum())
    for g, w in zip(dg.fetch_clusters(sel, nm, npairs), orc.fetch_clusters(sel, nm, npairs)):
        assert np.array_equal(g, w)


def test_cluster_tables_across_rebuilds():
    host, *_ = random_case(1, 3_000, 100, 12_000, 1)
    a, b, empty = cluster_inputs(2, 40), cluster_inputs(3, 700), cluster_inputs(4, 0)
    dg, orc = DeviceGraph.upload(host), ClusterOracle(host)
    try:
        check_clusters(dg, orc, a)
        want_a = orc.build_clusters(*a)
        with pytest.raises(_lib.AbbError, match="out of range"):
            dg.fetch_clusters(np.array([a[0]]), 0, 0)
        with pytest.raises(_lib.AbbError, match="bad arguments"):
            _lib.check(_lib.load().abb_clusters_build_host(dg.handle, -1, None, None, None, None, None, None, None, None, None))
        check_cluster_members(dg, orc, want_a)
        check_clusters(dg, orc, b)
        check_clusters(dg, orc, empty)
        assert dg.fetch_clusters(np.zeros(0, np.int32), 0, 0)[0].size == 0
        with pytest.raises(_lib.AbbError, match="out of range"):
            dg.fetch_clusters(np.array([0]), 0, 0)
        check_clusters(dg, orc, a)
    finally:
        dg.close()


# ── snapshot diff ──
def delta_inputs():
    """The new graph of a seeded pair, its table, a table with other labels, codes, risk and weights (B), and the old graph's."""
    (co, to, no), (cn, tn, nn) = pair(21, 2_000, 6_000, 0.8, 40)
    rng = np.random.default_rng(22)
    nr = tn[0]
    labels = [f"label-{int(x)}-{'é' * int(x % 3)}" for x in rng.integers(0, 50, nr)]
    lb, loff = delta._pack(labels)
    tb = (nr, tn[1], tn[2], tn[3], lb, loff, rng.integers(0, 3, nr).astype(np.uint8), rng.integers(0, 3, nr).astype(np.uint8),
          rng.integers(0, 3, nr).astype(np.float64), tn[9], tn[10])
    union = sorted(set(no) | set(nn))
    relmaps = ([union.index(x) for x in no], [union.index(x) for x in nn])
    return co, to, cn, tn, tb, rng.integers(0, 2, cn.n_edges).astype(np.float64), relmaps


def test_delta_tables_across_rebuilds():
    co, to, cn, ta, tb, wb, (rm_o, rm_n) = delta_inputs()
    dgo, dgn = DeviceGraph.upload(co), DeviceGraph.upload(cn)
    oo, on = DeltaOracle(co), DeltaOracle(cn)
    try:
        dgo.build_delta_table(*to)
        oo.build_delta_table(*to)

        def check(table, weight):
            on.build_delta_table(*table, weight=weight)
            got, want = dgn.diff(dgo, rm_o, rm_n), on.diff(oo, rm_o, rm_n)
            for k in want:
                assert np.array_equal(got[k], want[k]), k

        dgn.build_delta_table(*ta)
        check(ta, None)
        bytes_a = dgn.delta_table_bytes()
        bad = list(ta)
        bad[9] = ta[9].copy()
        bad[9][0] = 64
        with pytest.raises(_lib.AbbError, match="out of range"):
            dgn.build_delta_table(*bad)
        assert dgn.delta_table_bytes() == bytes_a
        check(ta, None)
        dgn.build_delta_table(*tb, weight=wb)
        check(tb, wb)
        bytes_b = dgn.delta_table_bytes()
        assert bytes_b != bytes_a
        assert bytes_b == fresh_bytes(lambda: DeviceGraph.upload(cn), lambda g: g.build_delta_table(*tb, weight=wb), DeviceGraph.delta_table_bytes)
        seen = read_while_rebuilding(lambda: dgn.build_delta_table(*ta), lambda: dgn.build_delta_table(*tb, weight=wb), dgn.delta_table_bytes)
        assert seen <= {bytes_a, bytes_b}, seen
    finally:
        dgo.close()
        dgn.close()


# ── lookup ──
def test_lookup_tables_across_rebuilds():
    csr, sev, erel = random_graph(31, 3_000, 200, 12_000, 1, 300)
    rng = np.random.default_rng(32)
    a = (csr.n_real, sev, erel)
    # other relationship ranks: a relabelling, so parallel edges keep distinct ranks as a graph's relationship strings give them
    b = (csr.n_real // 2, rng.integers(0, 9, csr.n_real // 2).astype(np.uint8), rng.permutation(6).astype(np.uint8)[erel])
    empty = (0, np.zeros(0, np.uint8), rng.permutation(6).astype(np.uint8)[erel])
    nodes = [0] + rng.integers(0, csr.n_nodes, 20).tolist()
    dg, o = DeviceGraph.upload(csr), LookupOracle(csr)

    def check(inputs):
        got, want = dg.build_lookup_table(*inputs), o.build_lookup_table(*inputs)
        for k in want:
            assert np.array_equal(got[k], want[k]), k
        check_context()

    def check_context():
        for u in nodes:
            assert np.array_equal(dg.context_edges(u), o.context_edges(u)), u
        s = rng.integers(0, csr.n_nodes, 200)
        assert np.array_equal(dg.incident_edges(s), o.incident_edges(s))

    try:
        check(a)
        bytes_a = dg.lookup_table_bytes()
        bad = erel.copy()
        bad[0] = 64
        with pytest.raises(_lib.AbbError, match="out of range"):
            dg.build_lookup_table(csr.n_real, sev, bad)
        assert dg.lookup_table_bytes() == bytes_a
        check_context()
        check(b)
        bytes_b = dg.lookup_table_bytes()
        assert bytes_b == fresh_bytes(lambda: DeviceGraph.upload(csr), lambda g: g.build_lookup_table(*b), DeviceGraph.lookup_table_bytes)
        check(empty)
        assert dg.lookup_table_bytes() == fresh_bytes(lambda: DeviceGraph.upload(csr), lambda g: g.build_lookup_table(*empty), DeviceGraph.lookup_table_bytes)
        seen = read_while_rebuilding(lambda: dg.build_lookup_table(*a), lambda: dg.build_lookup_table(*b), dg.lookup_table_bytes)
        assert seen <= {bytes_a, bytes_b}, seen
    finally:
        dg.close()


# ── node search ──
SEARCH_SPECS = [dict(mode=MODE_ALL, patterns=[]), dict(mode=MODE_FTS, patterns=[b"agent"]), dict(mode=MODE_LIKE, patterns=[b"\xc3\xa9"]),
                dict(mode=MODE_LIKE, patterns=[b"tail"], offset=2, take=5), dict(mode=MODE_FTS, patterns=[b"needle0"])]


def test_search_tables_across_rebuilds():
    a, b = search_inputs(41, 3_000, 0, 6), search_inputs(42, 40, 2, 3)
    empty = (np.zeros(1, np.int64), b"", tuple(np.zeros(0, x.dtype) if isinstance(x, np.ndarray) else x for x in a[2]))
    dg, o = one_node_graph(), SearchOracle()

    def build(g, inputs):
        off, text, table = inputs
        g.build_search_table(fold_table(g.search_text(off, text)), *table)

    def check(inputs):
        off, text, table = inputs
        cps = dg.search_text(off, text)
        assert np.array_equal(cps, o.search_text(off, text))
        dg.build_search_table(fold_table(cps), *table)
        o.build_search_table(fold_table(cps), *table)
        check_search()

    def check_search():
        for spec in SEARCH_SPECS:
            got, want = dg.search(**spec), o.search(**spec)
            assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], spec

    try:
        check(a)
        bytes_a = dg.search_table_bytes()
        bad = list(a[2])
        bad[3] = bad[3].copy()
        bad[3][0] = bad[6]                     # entity-type code == n_types
        with pytest.raises(_lib.AbbError, match="out of range"):
            dg.build_search_table(fold_table(np.zeros(0, np.int64)), *bad)
        off = a[0].copy()
        off[2] = off[1] - 1
        with pytest.raises(_lib.AbbError, match="decrease"):
            dg.search_text(off, a[1])
        assert dg.search_table_bytes() == bytes_a
        check_search()
        check(b)
        bytes_b = dg.search_table_bytes()
        assert bytes_b == fresh_bytes(one_node_graph, lambda g: build(g, b), DeviceGraph.search_table_bytes)
        check(empty)
        assert dg.search_table_bytes() == fresh_bytes(one_node_graph, lambda g: build(g, empty), DeviceGraph.search_table_bytes)
        # with B's text stored, rebuilding only the table keeps the text: the bytes never read as "not built" in between
        check(b)
        fold = fold_table(dg.search_text(b[0], b[1]))
        b2 = (b[2][0][::-1].copy(),) + b[2][1:]
        dg.build_search_table(fold, *b[2])
        seen = read_while_rebuilding(lambda: dg.build_search_table(fold, *b[2]), lambda: dg.build_search_table(fold, *b2), dg.search_table_bytes)
        assert seen == {bytes_b}, seen
    finally:
        dg.close()


# ── compliance ──
def test_compliance_tables_across_rebuilds():
    a = compliance_inputs(51, 257, 40, 30, 7, 5, 0.3)
    b = compliance_inputs(52, 20_000, 3_000, 900, 150, 8, 0.5)
    empty = compliance_inputs(53, 0, 40, 30, 7, 5, 0.3)
    dg, o = one_node_graph(), ComplianceOracle()
    lib = _lib.load()

    def check(inputs):
        got, want = dg.compliance_table(*inputs), o.compliance_table(*inputs)
        for k in want:
            assert np.array_equal(got[k], want[k]), k

    def fetch_matches(want, n_fw):
        out = {"sev": np.empty((4, want["sev"].shape[1]), np.int64), "type": np.empty((4, want["type"].shape[1]), np.int64),
               "tag": np.empty((4, want["tag"].shape[1]), np.int64), "node_count": np.empty(n_fw, np.int64),
               "node_rows": np.empty(want["node_rows"].shape[0], np.int32)}
        _lib.check(lib.abb_compliance_fetch_host(dg.handle, *(out[k].ctypes.data for k in ("sev", "type", "tag", "node_count", "node_rows"))))
        for k in want:
            assert np.array_equal(out[k], want[k]), k

    try:
        check(a)
        want_a = o.compliance_table(*a)
        bytes_a = dg.compliance_table_bytes()
        bad = list(a)
        bad[4] = a[4].copy()
        bad[4][0] = a[5].shape[0]              # tag code == n_tags
        with pytest.raises(_lib.AbbError, match="out of range"):
            dg.compliance_table(*bad)
        assert dg.compliance_table_bytes() == bytes_a
        fetch_matches(want_a, a[6])
        check(b)
        bytes_b = dg.compliance_table_bytes()
        assert bytes_b == fresh_bytes(one_node_graph, lambda g: g.compliance_table(*b), DeviceGraph.compliance_table_bytes)
        check(empty)
        assert dg.compliance_table_bytes() == fresh_bytes(one_node_graph, lambda g: g.compliance_table(*empty), DeviceGraph.compliance_table_bytes)
        seen = read_while_rebuilding(lambda: dg.compliance_table(*a), lambda: dg.compliance_table(*b), dg.compliance_table_bytes)
        assert seen <= {bytes_a, bytes_b}, seen
    finally:
        dg.close()


# ── memory ──
def test_rebuilt_tables_are_freed_with_their_graphs():
    import torch

    host, *_ = random_case(61, 200_000, 1_000, 800_000, 1)
    clusters = [cluster_inputs(62, 5_000, 200_000, 1_000), cluster_inputs(63, 20_000, 200_000, 1_000), cluster_inputs(64, 0, 200_000, 1_000)]
    co, to, cn, ta, tb, wb, _ = delta_inputs()
    lk_csr, lk_sev, lk_erel = random_graph(65, 100_000, 1_000, 400_000)
    sa, sb = search_inputs(66, 100_000, 1, 6), search_inputs(67, 30_000, 0, 6)
    ca, cb = compliance_inputs(68, 200_000, 20_000, 900, 150, 8, 0.5), compliance_inputs(69, 0, 40, 30, 7, 5, 0.3)

    def cycle():
        graphs = [DeviceGraph.upload(host), DeviceGraph.upload(cn), DeviceGraph.upload(lk_csr), one_node_graph()]
        g_cl, g_dl, g_lk, g_sr = graphs
        try:
            for c in clusters:
                g_cl.build_clusters(*c)
            g_dl.build_delta_table(*ta)
            g_dl.build_delta_table(*tb, weight=wb)
            g_lk.build_lookup_table(lk_csr.n_real, lk_sev, lk_erel)
            g_lk.incident_edges(np.arange(1_000))
            g_lk.build_lookup_table(0, np.zeros(0, np.uint8), lk_erel)
            g_lk.context_edges(0)
            for off, text, table in (sa, sb):
                g_sr.build_search_table(fold_table(g_sr.search_text(off, text)), *table)
                g_sr.search(MODE_FTS, [b"agent"], take=50)
            g_sr.compliance_table(*ca)
            g_sr.compliance_table(*cb)
        finally:
            for g in graphs:
                g.close()

    torch.cuda.mem_get_info()
    cycle()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20
