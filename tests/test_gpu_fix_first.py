"""The fix-first view on the device.

* Golden parity: every view the unmodified reference's route returned (``tests/golden/fix_first/``) is returned again — on graphs
  adopted from the reference's records, through ``B200GraphStore.fix_first_view``, and on SQLite snapshots the reference wrote,
  loaded with ``load_snapshot``.
* Focused ranking at scale (M2 estate, every finding): matched counts and pages at several offsets equal a numpy stable sort of
  the expanded rows restricted to the focus; the NULL focus is the unfocused ranking; an empty focus matches nothing; a focus
  byte of every category on every node gives the unfocused order.
"""

from __future__ import annotations

import gzip

import numpy as np
import pytest

from fix_first_golden import adopted, cases, focus_kwargs, roundtrip

pytestmark = pytest.mark.gpu

GRAPH_CASES = cases()
SNAPSHOT_CASES = cases(with_graph=False)


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_views_equal_the_reference(case):
    from agent_bom_b200.graph import fix_first_view

    g = adopted(case)
    for vc in case["views"]:
        assert roundtrip(fix_first_view(g, **focus_kwargs(vc))) == roundtrip(vc["view"]), vc["focus"]


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_store_views_equal_the_reference(case):
    from agent_bom_b200.store import B200GraphStore

    store = B200GraphStore()
    store.save_graph(adopted(case))
    for vc in case["views"]:
        got = store.fix_first_view(tenant_id=case["tenant_id"], scan_id=case["scan_id"], **focus_kwargs(vc))
        assert roundtrip(got) == roundtrip(vc["view"]), vc["focus"]
    empty = store.fix_first_view(tenant_id=case["tenant_id"], scan_id="no-such-scan", cve="x")
    assert empty["cards"] == [] and empty["scan_id"] == "no-such-scan" and empty["focus"] == {"cve": "x", "package": "", "agent": ""}
    assert empty["summary"] == {"total_paths": 0, "matched_paths": 0, "returned_paths": 0, "highest_risk": 0.0, "covered_findings": 0,
                                "node_count": 0, "edge_count": 0}


@pytest.fixture(scope="module")
def snapshot_db(tmp_path_factory):
    from fix_first_golden import GOLD

    path = tmp_path_factory.mktemp("ffsnap") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD.parent / "snapshot" / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.mark.parametrize("case", SNAPSHOT_CASES, ids=[c["name"] for c in SNAPSHOT_CASES])
def test_snapshot_views_equal_the_reference(snapshot_db, case):
    from agent_bom_b200.graph import fix_first_view, load_snapshot

    g = load_snapshot(snapshot_db, tenant_id=case["tenant"], scan_id=case["scan_id"])
    assert g.scan_id == case["scan_id"]
    for vc in case["views"]:
        assert roundtrip(fix_first_view(g, **focus_kwargs(vc))) == roundtrip(vc["view"]), vc["focus"]


def test_view_caches_follow_the_graph():
    """The label index is built by the first focused call only, and a mutation drops every per-graph cache with the device graph."""
    from agent_bom_b200.graph import UnifiedNode, fix_first_view

    case = next(c for c in GRAPH_CASES if c["name"] == "kat_focus")
    g = adopted(case)
    fix_first_view(g)
    assert g._rank_inputs is not None and g._focus_index is None
    fix_first_view(g, agent="ci-bot")
    assert g._focus_index is not None
    g.add_node(UnifiedNode(id="agent:new", entity_type="agent", label="New"))
    assert g._rank_inputs is None and g._focus_index is None and g._edge_lookup is None and g._dg is None


# ── focused ranking at scale ──────────────────────────────────────────────────────────────────────────────────────────────────
@pytest.fixture(scope="module")
def m2():
    from agent_bom_b200 import estate
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    est = estate.generate(20_700, 2145, estate.BENCH_KNOBS, exact_rank=False)
    host = csrmod.from_arrays(None, est.node_type, est.src, est.dst, est.rel, est.flags, node_rank=est.node_rank)
    dg = DeviceGraph.upload(host)
    f = np.ascontiguousarray(est.findings)
    rows = dg.exposure_paths_many(f)
    n_rows = rows.hops.shape[0]
    base_of_sev = np.asarray([100.0, 80.0, 60.0, 40.0])        # severity rank * 20 (risk_score is 0 in the estates)
    base_vals, base_id = np.unique(base_of_sev[est.node_sev[f]], return_inverse=True)
    scores = np.empty((len(base_vals), 5, 15))
    for bi, b in enumerate(base_vals.tolist()):
        for nc in range(5):
            for nt in range(15):
                risk = b
                risk += min(10.0, nc * 3.0)
                risk += min(10.0, nt * 0.75)
                scores[bi, nc, nt] = round(min(100.0, risk), 2)
    levels = np.unique(scores)
    table = np.searchsorted(levels, scores).astype(np.uint32)
    ncu = np.zeros(host.n_nodes, dtype=np.int32); ntu = np.zeros(host.n_nodes, dtype=np.int32)
    ncu[rows.hops[:, 1]] = rows.ncred; ntu[rows.hops[:, 1]] = rows.ntool        # labels are unique per node in the estates
    risk = scores[np.repeat(base_id, np.diff(rows.off)), np.minimum(rows.ncred, 4), np.minimum(rows.ntool, 14)]
    nh = np.where(rows.hops[:, 2] >= 0, 4, 3)
    order = np.lexsort((np.arange(n_rows), -ntu[rows.hops[:, 1]], -ncu[rows.hops[:, 1]], -nh, -risk))
    args = (f, base_id.astype(np.int32), table, ncu, ntu)
    yield est, host, dg, rows, order, args
    dg.close()


def row_mask(rows, focus: np.ndarray, need: int) -> np.ndarray:
    from agent_bom_b200 import _lib

    h = rows.hops.astype(np.int64)
    vs = np.where(h[:, 2] >= 0, h[:, 2], h[:, 1])
    on_hops = (focus[h[:, 0]] | focus[h[:, 1]] | focus[vs]) & np.uint8(~_lib.FOCUS_CVE_FINDING & 0xFF)
    on_f = focus[h[:, 3]]
    got = on_hops | on_f | np.where(on_f & _lib.FOCUS_CVE_FINDING, _lib.FOCUS_CVE, 0).astype(np.uint8)
    return (got & need) == need


def test_focused_pages_match_a_host_sort(m2):
    from agent_bom_b200 import _lib

    est, host, dg, rows, order, args = m2
    h = rows.hops
    t = host.node_type
    agents, per_agent = np.unique(h[:, 0][t[h[:, 0]] == 0], return_counts=True)
    heavy_agent = int(agents[np.argmax(per_agent)])
    finds, per_find = np.unique(h[:, 3], return_counts=True)
    heavy_vuln = int(finds[np.argmax(per_find)])
    vs = h[:, 2][h[:, 2] >= 0]
    pkgs, per_pkg = np.unique(vs[t[vs] == 2], return_counts=True)
    rare_pkg = int(pkgs[np.argmin(per_pkg)])
    row_of_agent = int(np.flatnonzero(h[:, 0] == heavy_agent)[len(np.flatnonzero(h[:, 0] == heavy_agent)) // 2])
    agents_vuln = int(h[row_of_agent, 3])           # a finding the heavy agent reaches: the pair matches something
    C, CF, P, A = _lib.FOCUS_CVE, _lib.FOCUS_CVE_FINDING, _lib.FOCUS_PACKAGE, _lib.FOCUS_AGENT
    focus = np.zeros(host.n_nodes, dtype=np.uint8)
    focus[heavy_agent] |= A
    focus[heavy_vuln] |= C | CF
    focus[agents_vuln] |= CF                        # counts as CVE on the finding hop only
    focus[rare_pkg] |= P
    focus[int(h[0, 1])] |= CF                       # a server's CVE_FINDING bit is ignored
    n_rows = h.shape[0]
    for need in (A, C, P, C | A, P | A, C | P, C | P | A):
        mask = row_mask(rows, focus, need)
        want_order = order[mask[order]]
        m = int(mask.sum())
        for offset, limit in ((0, 20000), (m // 2, 5000), (max(0, m - 3000), 5000), (m + 5, 10)):
            page, rank, total, matched = dg.rank_exposure_paths_focused(*args, focus, need, offset, limit)
            assert (total, matched) == (n_rows, m), need
            want = want_order[offset: offset + limit]
            np.testing.assert_array_equal(page.hops, h[want])
            np.testing.assert_array_equal(page.rels, rows.rels[want])
    assert int(row_mask(rows, focus, A).sum()) > 1000 and 0 < int(row_mask(rows, focus, P).sum()) < 1000
    assert int(row_mask(rows, focus, C | A).sum()) > 0


def test_null_full_and_empty_focus(m2):
    from agent_bom_b200 import _lib

    est, host, dg, rows, order, args = m2
    n_rows = rows.hops.shape[0]
    all_cats = _lib.FOCUS_CVE | _lib.FOCUS_PACKAGE | _lib.FOCUS_AGENT
    every = np.full(host.n_nodes, 0x0F, dtype=np.uint8)
    for offset, limit in ((0, 20000), (n_rows // 2, 5000)):
        p0, r0, t0 = dg.rank_exposure_paths(*args, offset, limit)
        p1, r1, t1, m1 = dg.rank_exposure_paths_focused(*args, None, 0, offset, limit)
        p2, r2, t2, m2_ = dg.rank_exposure_paths_focused(*args, every, all_cats, offset, limit)
        assert t0 == t1 == t2 == m1 == m2_ == n_rows
        for p in (p1, p2):
            np.testing.assert_array_equal(p.hops, p0.hops)
            np.testing.assert_array_equal(p.rels, p0.rels)
            np.testing.assert_array_equal(p.ncred, p0.ncred)
            np.testing.assert_array_equal(p.ntool, p0.ntool)
        np.testing.assert_array_equal(r1, r0)
        np.testing.assert_array_equal(r2, r0)
        np.testing.assert_array_equal(p0.hops, rows.hops[order[offset: offset + limit]])
    nothing = np.zeros(host.n_nodes, dtype=np.uint8)
    page, rank, total, matched = dg.rank_exposure_paths_focused(*args, nothing, _lib.FOCUS_AGENT, 0, 25)
    assert (total, matched, page.hops.shape[0], rank.shape[0]) == (n_rows, 0, 0, 0)
    # limit 0 still reports the matched count
    _, _, _, matched = dg.rank_exposure_paths_focused(*args, every, _lib.FOCUS_AGENT, 0, 0)
    assert matched == n_rows
    with pytest.raises(_lib.AbbError):
        dg.rank_exposure_paths_focused(*args, every, 0x10, 0, 1)
