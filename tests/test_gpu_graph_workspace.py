"""The graph handle's workspaces: the tuning options read and written through one table, the exposure tables built once per graph
and rebuilt only by a new graph, and one graph used from several threads at once (the library serialises the calls, and
abb_exposure_host splits each of its calls between two threads that must touch disjoint state).  Needs a GPU.
"""

from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_gpu_exposure_tables import ET_MISCONF, ET_VULN, batches, exposure_graph, expected_rows, rank_inputs, upload
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(2**63), 2**63 - 1
ERR_ARG = -2

# every writable option: the values set_option accepts and its message for the others (None: every value is accepted)
RANGES = {
    "mid_qcap": (32, 4096, "mid_qcap must be in [32, 4096]"),
    "big_qcap": (32, 36864, "big_qcap must be in [32, 36864]"),
    "chunks": (1, 64, "chunks must be in [1, 64]"),
    "chunk_min": (2, I64_MAX, "chunk_min must be >= 2"),
    "big_limit": (0, I64_MAX, "big_limit must be >= 0"),
    "nx_batch": (0, I64_MAX, "nx_batch must be >= 0"),
    "delta_union_limit": (0, 2**27, "delta_union_limit must be in [0, 2^27]"),
}
FLAGS = ("dedup", "zero_copy", "hist_pack")   # stored as value != 0
MASKED = {"block_tiers": 3}                   # stored as value & mask


@pytest.fixture(scope="module")
def graph():
    src, dst, rel, flags, nt, rank, special = exposure_graph()
    og = orc.build_csr(len(nt), src, dst, rel, flags, nt)
    return src, dst, rel, flags, nt, rank, special, og


def refused(dg, name, value, message):
    from agent_bom_b200 import _lib

    with pytest.raises(_lib.AbbError) as e:
        dg.set_option(name, value)
    assert e.value.code == ERR_ARG and message in str(e.value)


def test_every_option_round_trips_and_keeps_its_range(graph):
    dg = upload(graph)
    try:
        for name, (lo, hi, message) in RANGES.items():
            for v in (lo, hi):
                dg.set_option(name, v)
                assert dg.get_option(name) == v, name
            for bad in (lo - 1, hi + 1):
                if I64_MIN <= bad <= I64_MAX:
                    refused(dg, name, bad, message)
                    assert dg.get_option(name) == hi, name
        for name in FLAGS:
            for v, want in ((0, 0), (1, 1), (7, 1), (-1, 1), (0, 0)):
                dg.set_option(name, v)
                assert dg.get_option(name) == want, name
        for name, mask in MASKED.items():
            for v in (0, mask, 6, -1, I64_MAX, 2):
                dg.set_option(name, v)
                assert dg.get_option(name) == (v & mask), name
        refused(dg, "last_host_chunks", 1, "unknown option 'last_host_chunks'")
        assert dg.get_option("last_host_chunks") == 1
        refused(dg, "no_such_option", 1, "unknown option 'no_such_option'")
        assert dg.get_option("no_such_option") == -1
    finally:
        dg.close()


def launches(call):
    from agent_bom_b200 import _lib

    before = _lib.load().abb_launch_count()
    out = call()
    return int(_lib.load().abb_launch_count() - before), out


def check_host_rows(og, rank, f, rows):
    want, off = expected_rows(og, f, rank)
    np.testing.assert_array_equal(rows.off, off)
    np.testing.assert_array_equal(rows.hops, want.hops)
    np.testing.assert_array_equal(rows.rels, want.rels)
    np.testing.assert_array_equal(rows.ncred, want.ncred)
    np.testing.assert_array_equal(rows.ntool, want.ntool)


def test_exposure_tables_are_built_once_per_graph(graph):
    """The first call on a graph builds the graph-constant tables (more launches); later calls only gather from them.  A new
    graph after close() builds its own."""
    src, dst, rel, flags, nt, rank, special, og = graph
    f = batches(nt, special)[0]
    counts = []
    for _ in range(2):
        dg = upload(graph)
        try:
            per_graph = []
            for _ in range(3):
                k, rows = launches(lambda: dg.exposure_paths_many(f))
                check_host_rows(og, rank, f, rows)
                per_graph.append(k)
        finally:
            dg.close()
        first, second, third = per_graph
        assert first > second > 0 and second == third
        counts.append(per_graph)
    assert counts[0] == counts[1]


def snapshot_walk(w):
    return {"count": w.count.copy(), "maxd": w.maxd.copy(), "flags": w.flags.copy(), "hist": w.hist.copy(),
            "slices": [w.slice(q).copy() for q in range(len(w))]}


def snapshot_rows(p):
    return {k: getattr(p, k).copy() for k in ("off", "hops", "rels", "ncred", "ntool")}


def assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        if k == "slices":
            assert len(a[k]) == len(b[k]), what
            for q, (x, y) in enumerate(zip(a[k], b[k])):
                np.testing.assert_array_equal(x, y, err_msg=f"{what}: slice {q}")
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{what}: {k}")


def test_one_graph_used_from_several_threads(graph):
    """Four threads call exposure_many, finding_context, a de-duplicated impact walk and rank_exposure_paths on one graph while a
    fifth reads options and walk statistics; every result equals the same call made alone."""
    src, dst, rel, flags, nt, rank, special, og = graph
    n = len(nt)
    findings = np.flatnonzero((nt == ET_VULN) | (nt == ET_MISCONF)).astype(np.int32)
    sources = np.random.default_rng(12).integers(0, n, size=600).astype(np.int32)
    _node_base, base_id, table, ncu, ntu = rank_inputs(nt, findings)
    dg = upload(graph)
    try:
        def exposure():
            w, p = dg.exposure_many(findings, max_depth=4)
            walk = snapshot_walk(w)
            return {**{k if k == "slices" else "walk_" + k: v for k, v in walk.items()}, **snapshot_rows(p)}

        def context():
            c = dg.finding_context(findings, max_depth=4)
            return {"count": c.count.copy(), "maxd": c.maxd.copy(), "flags": c.flags.copy(), "start": c.start.copy(),
                    "bucket_counts": c.bucket_counts.copy(), "source_nodes": c.source_nodes.copy(), "hist": c.hist.copy()}

        def impact():
            return snapshot_walk(dg.impact_many(sources, max_depth=4))

        def ranked():
            page, rr, total = dg.rank_exposure_paths(findings, base_id, table, ncu, ntu, 0, 500)
            return {**snapshot_rows(page), "risk_rank": rr.copy(), "total": np.asarray([total])}

        calls = {"exposure_many": exposure, "finding_context": context, "impact_many": impact, "rank_exposure_paths": ranked}
        alone = {name: call() for name, call in calls.items()}
        impact()
        stats = dg.last_walk_stats()
        assert stats["queries"] == len(sources) and stats["eligible"] > 0     # the walk is de-duplicated
        assert alone["exposure_many"]["hops"].shape[0] > 0 and int(alone["rank_exposure_paths"]["total"][0]) > 0
        options = {name: dg.get_option(name) for name in ("dedup", "block_tiers", "chunks", "zero_copy")}
        iterations = 10

        def repeat(call):
            return [call() for _ in range(iterations)]

        def reader():
            seen = []
            for _ in range(iterations * 4):
                assert {name: dg.get_option(name) for name in options} == options
                ms = dg.last_walk_ms()
                assert ms == -1.0 or ms >= 0.0
                s = dg.last_walk_stats()
                assert s["queries"] in (len(findings), len(sources))
                seen.append(s["queries"])
            return seen

        with ThreadPoolExecutor(max_workers=len(calls) + 1) as pool:
            futures = {name: pool.submit(repeat, call) for name, call in calls.items()}
            read = pool.submit(reader)
            results = {name: fut.result() for name, fut in futures.items()}
            assert len(read.result()) == iterations * 4
        for name, runs in results.items():
            assert len(runs) == iterations
            for i, got in enumerate(runs):
                assert_same(alone[name], got, f"{name}, iteration {i}")
    finally:
        dg.close()
