"""Snapshot diff on the H100: every golden pair through ``B200GraphStore.diff_snapshots`` and ``snapshot_diff`` against the reference's
``diff_snapshots`` (oracle/make_delta_golden.py); seeded random graph pairs against the Python oracle, one above 1 M edges with
heavy overlap and one with no shared id; diffs run concurrently against one graph; the union limit's error; the diff tables freed
with the graph; and ``compute_delta_alerts`` against the reference's alerts.
"""

from __future__ import annotations

import gzip
import json
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
from oracle.delta_oracle import DeltaOracle
from test_delta import ALERT_CASES, ALERT_IDS, alert_graphs, normalise_alerts

from agent_bom_b200 import _lib
from agent_bom_b200.engine import DeviceGraph
from agent_bom_b200.graph import csr as csrmod
from agent_bom_b200.graph import delta
from agent_bom_b200.graph.snapshot import load_snapshot
from agent_bom_b200.store import B200GraphStore

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden" / "delta"
CASES = json.loads(gzip.decompress((GOLD / "expected.json.gz").read_bytes()))
IDS = [f"{c['tenant'].strip() or '-'}:{c['old'] or 'blank'}>{c['new'] or 'blank'}" for c in CASES]


@pytest.fixture(scope="module")
def db_path(tmp_path_factory) -> Path:
    path = tmp_path_factory.mktemp("delta") / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLD / "graph.sqlite.gz").read_bytes()))
    return path


@pytest.fixture(scope="module")
def store(db_path) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None), max_graphs=4)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_diff_matches_reference(store, case):
    body = store.diff_snapshots(case["old"], case["new"], tenant_id=case["tenant"])
    assert json.loads(json.dumps(body)) == case["diff"]


@pytest.mark.parametrize("case", [c for c in CASES if c["old"] and c["new"] and "missing" not in (c["old"], c["new"])],
                         ids=lambda c: f"{c['tenant'].strip() or '-'}:{c['old']}>{c['new']}")
def test_snapshot_diff_matches_reference(db_path, case):
    old = load_snapshot(db_path, tenant_id=case["tenant"], scan_id=case["old"])
    new = load_snapshot(db_path, tenant_id=case["tenant"], scan_id=case["new"])
    timings: dict = {}
    body = delta.snapshot_diff(old, new, timings=timings)
    assert json.loads(json.dumps(body)) == case["diff"]
    assert set(timings) == {"device_s", "sql_s", "response_s"}


def pair(seed: int, n: int, m: int, overlap: float, ghosts: int = 0):
    """Two random graphs over string ids: the new one keeps a share of the old one's ids and edges and perturbs columns."""
    rng = np.random.default_rng(seed)
    pool = [f"n:{rng.integers(1 << 40):x}:{'é' if i % 7 == 0 else ''}{chr(0x1F600 + i % 50) if i % 11 == 0 else ''}" for i in range(int(n * (2 - overlap)) + 2 * ghosts)]
    pool = list(dict.fromkeys(pool))
    rels = ["uses", "depends_on", "hosts", "zz_custom", "affects", "aa_other"]

    def graph(ids, ghost_ids, keep_edges=None):
        allid = ids + ghost_ids
        nn, nr = len(allid), len(ids)
        if keep_edges is None:
            src = rng.integers(0, nn, m)
            dst = rng.integers(0, nn, m)
            rel = rng.integers(0, len(rels), m)
        else:
            src, dst, rel = keep_edges
        key = {}
        for i, (s, d, r) in enumerate(zip(src.tolist(), dst.tolist(), rel.tolist())):
            key.setdefault((s, d, r), i)
        idx = np.fromiter(key.values(), np.int64)
        src, dst, rel = src[idx], dst[idx], rel[idx]
        flags = rng.integers(0, 4, len(idx)).astype(np.uint8)
        codes = np.where(rel < 3, rel, 31).astype(np.uint8)
        types = np.concatenate([rng.integers(0, 25, nr).astype(np.uint8), np.full(nn - nr, 255, np.uint8)])
        types[types == 24] = 254
        csr = csrmod.from_arrays(allid, types, src.astype(np.int32), dst.astype(np.int32), codes, flags, n_real=nr)
        names = sorted(set(rels[r] for r in rel.tolist()))
        slot = {s: i for i, s in enumerate(names)}
        erel = np.asarray([slot[rels[r]] for r in rel.tolist()], np.uint8)
        ids_b, ioff = delta._pack(allid)
        labels = [f"l{int(x)}" for x in rng.integers(0, 3, nr)]
        lb, loff = delta._pack(labels)
        table = (nr, ids_b, ioff, np.argsort(csr.node_rank, kind="stable").astype(np.int32), lb, loff, rng.integers(0, 3, nr).astype(np.uint8),
                 np.where(rng.random(nr) < 0.02, 255, rng.integers(0, 3, nr)).astype(np.uint8), rng.integers(0, 3, nr).astype(np.float64), erel, flags)
        return csr, table, names, (src, dst, rel)

    old_ids = pool[:n]
    new_ids = pool[int(n * (1 - overlap)): int(n * (1 - overlap)) + n]
    gh = pool[len(pool) - 2 * ghosts:]
    co, to, no, (s, d, r) = graph(old_ids, gh[:ghosts])
    # the new graph reuses the old edges whose endpoints survive, re-indexed, and adds random ones
    pos = {x: i for i, x in enumerate(new_ids + gh[ghosts // 2: ghosts // 2 + ghosts])}
    all_old = old_ids + gh[:ghosts]
    ns = np.asarray([pos.get(all_old[x], -1) for x in s.tolist()])
    nd = np.asarray([pos.get(all_old[x], -1) for x in d.tolist()])
    keep = (ns >= 0) & (nd >= 0)
    extra = m - int(keep.sum())
    nn = len(pos)
    es = (np.concatenate([ns[keep], rng.integers(0, nn, extra)]), np.concatenate([nd[keep], rng.integers(0, nn, extra)]),
          np.concatenate([r[keep], rng.integers(0, 6, extra)]))
    cn, tn, nn_names, _ = graph(new_ids, gh[ghosts // 2: ghosts // 2 + ghosts], es)
    return (co, to, no), (cn, tn, nn_names)


def diff_both(old, new, weights: bool = False):
    (co, to, no), (cn, tn, nn) = old, new
    union = sorted(set(no) | set(nn))
    rm_o, rm_n = [union.index(x) for x in no], [union.index(x) for x in nn]
    rng = np.random.default_rng(5)
    wo = rng.integers(0, 2, co.n_edges).astype(np.float64) if weights else None
    wn = rng.integers(0, 2, cn.n_edges).astype(np.float64) if weights else None
    dgo, dgn = DeviceGraph.upload(co), DeviceGraph.upload(cn)
    oo, on = DeltaOracle(co), DeltaOracle(cn)
    try:
        dgo.build_delta_table(*to, weight=wo)
        dgn.build_delta_table(*tn, weight=wn)
        oo.build_delta_table(*to, weight=wo)
        on.build_delta_table(*tn, weight=wn)
        got = dgn.diff(dgo, rm_o, rm_n)
    finally:
        dgo.close()
        dgn.close()
    want = on.diff(oo, rm_o, rm_n)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    return got


@pytest.mark.parametrize("seed,n,m,overlap,ghosts,weights", [(1, 2_000, 6_000, 0.8, 50, False), (2, 3_000, 9_000, 0.5, 0, True), (3, 500, 2_000, 1.0, 20, True),
                                                              (4, 1_000, 3_000, 0.0, 0, False)])
def test_random_pairs_match_oracle(seed, n, m, overlap, ghosts, weights):
    got = diff_both(*pair(seed, n, m, overlap, ghosts), weights=weights)
    if overlap == 0.0:
        assert got["changed_new"].size == 0 and got["echanged_new"].size == 0
        assert got["nodes_added"].size == n and got["nodes_removed"].size == n


def test_million_edge_pair_with_heavy_overlap():
    got = diff_both(*pair(11, 200_000, 1_100_000, 0.95, 1_000), weights=True)
    assert got["echanged_new"].size > 0 and got["edges_added"].size > 0


def test_union_limit_error():
    (co, to, _), (cn, tn, _) = pair(7, 300, 600, 0.5)
    dgo, dgn = DeviceGraph.upload(co), DeviceGraph.upload(cn)
    try:
        dgo.build_delta_table(*to)
        dgn.build_delta_table(*tn)
        dgn.set_option("delta_union_limit", co.n_nodes)     # the union of the two id sets is larger
        with pytest.raises(_lib.AbbError, match="exceed the edge key's limit"):
            dgn.diff(dgo, list(range(6)), list(range(6)))
        dgn.set_option("delta_union_limit", 1 << 27)
        dgn.diff(dgo, list(range(6)), list(range(6)))
        with pytest.raises(_lib.AbbError):
            dgn.set_option("delta_union_limit", (1 << 27) + 1)
    finally:
        dgo.close()
        dgn.close()


def test_tables_are_freed_with_the_graph():
    import torch

    (co, to, _), (cn, tn, _) = pair(9, 400_000, 800_000, 0.9)

    def cycle():
        dgo, dgn = DeviceGraph.upload(co), DeviceGraph.upload(cn)
        try:
            dgo.build_delta_table(*to)
            dgn.build_delta_table(*tn)
            assert dgo.delta_table_bytes() > 8 * co.n_nodes
            dgn.diff(dgo, list(range(6)), list(range(6)))
        finally:
            dgo.close()
            dgn.close()

    torch.cuda.mem_get_info()
    cycle()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20


@pytest.mark.parametrize("case", ALERT_CASES, ids=ALERT_IDS)
def test_delta_alerts_match_reference(db_path, case):
    from agent_bom_b200.graph import compute_delta_alerts

    got = compute_delta_alerts(*alert_graphs(db_path, case))
    assert normalise_alerts(got) == normalise_alerts(case["alerts"])


def test_concurrent_diffs_against_one_new_graph():
    """Each diff's answer is its own: diffs of two old graphs against one shared new graph, run on threads, equal the serial ones."""
    from concurrent.futures import ThreadPoolExecutor

    (c1, t1, n1), (cn, tn, nn) = pair(21, 20_000, 80_000, 0.9, 100)
    (c2, t2, n2), _ = pair(22, 5_000, 10_000, 0.3, 0)
    graphs = [DeviceGraph.upload(c) for c in (c1, c2, cn)]
    try:
        for dg, t in zip(graphs, (t1, t2, tn)):
            dg.build_delta_table(*t)
        union = sorted(set(n1) | set(n2) | set(nn))
        rm = [[union.index(x) for x in names] for names in (n1, n2, nn)]
        serial = [graphs[2].diff(graphs[k], rm[k], rm[2]) for k in (0, 1)]
        assert serial[0]["edges_added"].size != serial[1]["edges_added"].size
        with ThreadPoolExecutor(8) as ex:
            futs = [(k, ex.submit(graphs[2].diff, graphs[k], rm[k], rm[2])) for _ in range(12) for k in (0, 1)]
            for k, f in futs:
                got = f.result()
                for key, want in serial[k].items():
                    assert np.array_equal(got[key], want), key
    finally:
        for dg in graphs:
            dg.close()
