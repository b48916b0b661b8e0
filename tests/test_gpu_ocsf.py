"""GPU: OCSF events with their device-computed graph context.

* Enriched events equal the reference's (tests/golden/ocsf/events.json.gz) on adopted graphs, the light builder's record and
  columnar graphs, SQLite snapshots and through ``B200GraphStore``; batch sizes and store pages do not change them.
* ``DeviceGraph.finding_context`` equals the CPU oracle on the golden graphs and on seeded graphs, with frontier de-duplication on
  and off and under every walk-tier setting, for query lists with invalid, ghost and duplicate ids and for an empty batch.
* What crosses PCIe is the documented per-finding arrays and the source lists, never the walk's node slices.
* M2 estate (every finding): counts and histograms equal ``impact_many``; a seeded sample's lists equal the oracle's.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import pytest

import ocsf_golden as og
from golden_util import seeded_graph
from oracle import ocsf_oracle
from oracle import oracle as orc
from test_gpu_tiers import CONFIGS

pytestmark = pytest.mark.gpu

GRAPH_CASES = og.graph_cases()
BUILDER_CASES = og.builder_cases()
SNAPSHOT_CASES = og.snapshot_cases()


def _without_data(evs):
    return [dict(ev, resources=[{k: v for k, v in r.items() if k != "data"} for r in ev["resources"]]) for ev in evs]


def check_enriched(graph, case, *, data=True, **kw):
    for v in og.versions():
        got = og.without_time(graph.to_ocsf_events(v, **kw) if not kw else list(graph.iter_ocsf_events(v, **kw)))
        want = og.events(case, v, True)
        if not data:     # the light builder does not record the reference builder's bookkeeping attributes (tests/test_ocsf.py)
            got, want = _without_data(got), _without_data(want)
        assert got == want


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_enriched_events_adopted(case):
    check_enriched(og.adopted(case), case)


@pytest.mark.parametrize("columnar", [False, True], ids=["records", "columnar"])
@pytest.mark.parametrize("case", BUILDER_CASES, ids=[c["name"] for c in BUILDER_CASES])
def test_enriched_events_light_builder(case, columnar):
    g = og.built(case, columnar)
    check_enriched(g, case, data=False)
    if columnar:
        assert not g.nodes._cache


@pytest.fixture(scope="module")
def snapshot_db(tmp_path_factory):
    return og.snapshot_db(tmp_path_factory.mktemp("ocsfsnap"))


@pytest.mark.parametrize("case", SNAPSHOT_CASES, ids=[c["name"] for c in SNAPSHOT_CASES])
def test_enriched_events_snapshot_and_store(snapshot_db, case):
    from agent_bom_b200.store import B200GraphStore

    check_enriched(og.loaded(case, snapshot_db), case)
    store = B200GraphStore(SimpleNamespace(_db_path=str(snapshot_db), load_graph=lambda **_kw: None))     # a SQLite-backed inner store
    kw = dict(tenant_id=case["tenant"], scan_id=case["snapshot_scan"])
    for v in og.versions():
        assert og.without_time(store.ocsf_events(**kw, product_version=v)) == og.events(case, v, True)
        assert og.without_time(store.ocsf_events(**kw, product_version=v, enrich_neighbors=False)) == og.events(case, v, False)
    full = og.events(case, "0.0.0", True)
    for offset, limit in ((0, 1), (3, 7), (len(full) - 2, None), (len(full), 5), (0, 0)):
        assert og.without_time(store.ocsf_events(**kw, offset=offset, limit=limit)) == full[offset: None if limit is None else offset + limit]
    assert store.ocsf_events(tenant_id=case["tenant"], scan_id="no-such-scan") == []


@pytest.mark.parametrize("name", ["estate_dense_40", "kat_ocsf"])
def test_batch_sizes_give_identical_events(name):
    case = next(c for c in GRAPH_CASES if c["name"] == name)
    g = og.adopted(case)
    for bs in (1, 7, 65536):
        check_enriched(g, case, batch_size=bs)


# ── FindingContext against the oracle ─────────────────────────────────────────────────────────────────────────────────────────
def assert_context_equal(got, want):
    """Every per-finding array, and the flat source list (finding-major, then bucket-major, row order) with its start offsets."""
    assert len(got) == len(want.count)
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


def queries(n_nodes, n_real, findings, rng):
    ghosts = np.arange(n_real, n_nodes, dtype=np.int32)[:5]
    dup = rng.choice(findings, size=min(40, len(findings))) if len(findings) else np.zeros(0, np.int32)
    return np.concatenate([findings, [-1, n_nodes + 3, -7], ghosts, dup, findings[:3]]).astype(np.int32)


_graphs: dict = {}


def golden_graph(name):
    if name not in _graphs:
        g = og.adopted(next(c for c in GRAPH_CASES if c["name"] == name))
        ograph, findings = og.oracle_of(g)
        _graphs[name] = (ograph, g.device_graph, findings, g.csr.n_nodes, g.csr.n_real)
    return _graphs[name]


def seeded(key):
    if key not in _graphs:
        from agent_bom_b200.engine import DeviceGraph
        from agent_bom_b200.graph import csr as csrmod

        n, e, seed = key
        src, dst, rel, flags, nt = seeded_graph(n, e, seed)
        ograph = orc.build_csr(len(nt), src, dst, rel, flags, nt)
        dg = DeviceGraph.upload(csrmod.from_arrays(None, nt, src, dst, rel, flags))
        findings = np.flatnonzero(np.isin(nt, (8, 9))).astype(np.int32)
        _graphs[key] = (ograph, dg, findings, n, n)
    return _graphs[key]


KEYS = ["kat_ocsf", "estate_dense_40", "estate_150", (2000, 12000, 2), (6000, 40000, 3)]
_oracle: dict = {}


def query_list(key):
    if ("q", key) not in _oracle:
        ograph, dg, findings, n_nodes, n_real = golden_graph(key) if isinstance(key, str) else seeded(key)
        rng = np.random.default_rng(31)
        q = queries(n_nodes, n_real, findings, rng)
        if isinstance(key, tuple):     # seeded graphs: also arbitrary nodes, whose rows hold every kind
            q = np.concatenate([q, rng.integers(0, n_nodes, size=1500).astype(np.int32)])
        _oracle[("q", key)] = q
    return _oracle[("q", key)]


def oracle_context(key, depth):
    """The oracle's answer for a key's query list, computed once for every tier / dedup setting."""
    if (key, depth) not in _oracle:
        ograph = (golden_graph(key) if isinstance(key, str) else seeded(key))[0]
        _oracle[(key, depth)] = ocsf_oracle.finding_context(ograph, query_list(key), depth)
    return _oracle[(key, depth)]


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("dedup", [True, False])
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_finding_context_matches_oracle(key, dedup, config):
    ograph, dg, findings, n_nodes, n_real = golden_graph(key) if isinstance(key, str) else seeded(key)
    try:
        dg.set_dedup(dedup)
        for k, v in CONFIGS[config].items():
            dg.set_option(k, v)
        q = query_list(key)
        for depth in (4, 6):
            assert_context_equal(dg.finding_context(q, depth), oracle_context(key, depth))
        empty = dg.finding_context(np.zeros(0, np.int32))
        assert len(empty) == 0 and empty.source_nodes.size == 0 and empty.d2h_bytes == 0
    finally:
        for k, v in CONFIGS["default"].items():
            dg.set_option(k, v)
        dg.set_dedup(True)


def expected_d2h(ctx) -> int:
    """count + maxd + flags (int32), the histogram as shipped, start (int64), bucket counts (int32 x 4), the source list (int32)."""
    n = len(ctx)
    hist = ctx.hist_packed.nbytes if ctx.hist_packed is not None else n * 24 * 4
    return 12 * n + hist + 8 * n + 16 * n + 4 * int(ctx.source_nodes.size)


def test_d2h_bytes_exclude_node_slices():
    ograph, dg, findings, n_nodes, n_real = seeded((2000, 12000, 2))
    rng = np.random.default_rng(5)
    for q in (findings[:100], rng.integers(0, n_nodes, size=5000).astype(np.int32)):      # dense and packed histograms
        for zero_copy in (0, 1):
            dg.set_option("zero_copy", zero_copy)
            ctx = dg.finding_context(q)
            assert ctx.d2h_bytes == expected_d2h(ctx) and ctx.h2d_bytes == 4 * len(q)
            imp = dg.impact_many(q)
            assert int(imp.count.sum()) > 0 and ctx.d2h_bytes < imp.d2h_bytes
            assert ctx.kernel_ms >= 0 and ctx.context_ms >= 0
    dg.set_option("zero_copy", 1)
    assert (len(q) >= 1024) == (ctx.hist_packed is not None)


# ── M2 estate ────────────────────────────────────────────────────────────────────────────────────────────────────────────────
def test_m2_every_finding():
    from agent_bom_b200 import estate
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    est = estate.generate(20_700, 2145, estate.BENCH_KNOBS, exact_rank=False)
    host = csrmod.from_arrays(None, est.node_type, est.src, est.dst, est.rel, est.flags, node_rank=est.node_rank)
    dg = DeviceGraph.upload(host)
    f = np.ascontiguousarray(est.findings, dtype=np.int32)
    ctx = dg.finding_context(f)
    imp = dg.impact_many(f)
    np.testing.assert_array_equal(ctx.count, imp.count)
    np.testing.assert_array_equal(ctx.maxd, imp.maxd)
    np.testing.assert_array_equal(ctx.hist, imp.hist)
    assert ctx.d2h_bytes == expected_d2h(ctx) and ctx.d2h_bytes < imp.d2h_bytes
    ograph = orc.build_csr(host.n_nodes, host.src, host.dst, host.rel, host.flags, host.node_type)
    sample = np.sort(np.random.default_rng(2026).choice(len(f), size=min(2000, len(f)), replace=False))
    for q in sample.tolist():
        want = ocsf_oracle.typed_sources(ograph, int(f[q]))
        for b in range(ocsf_oracle.N_BUCKETS):
            np.testing.assert_array_equal(ctx.sources(q, b), want[b])
    dg.close()
