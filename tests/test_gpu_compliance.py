"""Compliance posture on the H100: every golden case through ``B200GraphStore`` with the graph cached both by topology-first loading
and by ``save_graph``, against the unmodified SQLite store (oracle/make_compliance_golden.py), compared as JSON text; seeded random
tables against the numpy oracle (oracle/compliance_oracle.py), one with more than 10^6 tagged rows, more than 10^5 frameworks and
a framework tagging nearly every row; concurrent first calls on one graph and on two graphs; and the table's memory returned with
the graph.
"""

from __future__ import annotations

import json
import threading
from types import SimpleNamespace

import numpy as np
import pytest
from oracle.compliance_oracle import ComplianceOracle
from test_compliance import CASES, IDS, call, db_path  # noqa: F401  (db_path: the module fixture)
from test_gpu_store_lookup import saved_graph

from agent_bom_b200.engine import DeviceGraph
from agent_bom_b200.graph import csr as csrmod
from agent_bom_b200.store import B200GraphStore

pytestmark = pytest.mark.gpu
SCANS = (("compliance", "est40"), ("", "kat"), ("", "kat2"), ("errors", "bad-json"), ("errors", "bad-tag"), ("errors", "bad-list"))


def inner(db_path):  # noqa: F811
    return SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None, save_graph=lambda _g: None)


@pytest.fixture(scope="module")
def loading_store(db_path):  # noqa: F811
    return B200GraphStore(inner(db_path), max_graphs=8)


@pytest.fixture(scope="module")
def saving_store(db_path):  # noqa: F811
    s = B200GraphStore(inner(db_path), max_graphs=8)
    for tenant, scan in SCANS:
        s.save_graph(saved_graph(db_path, tenant, scan))
    return s


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_compliance_by_loading(loading_store, case):
    assert call(loading_store, case["kwargs"]) == json.dumps(case["expected"])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_compliance_by_save_graph(saving_store, case):
    assert call(saving_store, case["kwargs"]) == json.dumps(case["expected"])


# ── seeded random tables against the oracle ──
def graph_handle() -> DeviceGraph:
    z = np.zeros(0, np.int32)
    return DeviceGraph.upload(csrmod.from_arrays(["n"], np.zeros(1, np.uint8), z, z, z.astype(np.uint8), z.astype(np.uint8), n_real=1))


def random_table(seed: int, n: int, n_texts: int, n_tags: int, n_fw: int, max_tags: int, hot: float):
    """Interned inputs: ``hot`` of the texts carry a tag of framework 0 (so it tags about that share of the rows); tags repeat
    within a text now and then; every framework has a tag."""
    rng = np.random.default_rng(seed)
    tag_fw = np.concatenate([np.arange(n_fw), rng.integers(0, n_fw, n_tags - n_fw)]).astype(np.int32)
    rng.shuffle(tag_fw)
    fw0 = np.flatnonzero(tag_fw == 0)
    length = rng.integers(1, max_tags + 1, n_texts)
    tags = [rng.integers(0, n_tags, k) for k in length]
    for t in np.flatnonzero(rng.random(n_texts) < hot):
        tags[t][0] = rng.choice(fw0)
    for t in np.flatnonzero(rng.random(n_texts) < 0.05):
        tags[t] = np.concatenate([tags[t], tags[t][:1]])
    text_off = np.zeros(n_texts + 1, np.int64)
    text_off[1:] = np.cumsum([len(t) for t in tags])
    text_tags = np.concatenate(tags).astype(np.int32)
    n_sev, n_types = 6, 9
    return (rng.integers(0, n_texts, n).astype(np.int32), rng.integers(0, n_sev, n).astype(np.int32), rng.integers(0, n_types, n).astype(np.int32),
            text_off, text_tags, tag_fw, n_fw, n_sev, n_types)


@pytest.mark.parametrize("seed, n, n_texts, n_tags, n_fw, max_tags, hot", [
    (1, 1, 1, 1, 1, 1, 0.0),
    (2, 257, 40, 30, 7, 5, 0.3),
    (3, 20_000, 3_000, 900, 150, 8, 0.5),
    (4, 1_100_000, 250_000, 300_000, 120_000, 5, 0.98),        # > 10^6 rows, > 10^5 frameworks, framework 0 on ~98% of rows
])
def test_random_tables_match_oracle(seed, n, n_texts, n_tags, n_fw, max_tags, hot):
    args = random_table(seed, n, n_texts, n_tags, n_fw, max_tags, hot)
    want = ComplianceOracle().compliance_table(*args)
    dg = graph_handle()
    try:
        got = dg.compliance_table(*args)
        for key in ("sev", "type", "tag", "node_count", "node_rows"):
            assert np.array_equal(got[key], want[key]), key
        if hot > 0.9:
            assert want["node_count"][0] > 0.95 * n and want["node_count"].shape[0] > 100_000
    finally:
        dg.close()


# ── concurrency ──
def _first_calls(db_path, scans, threads: int):  # noqa: F811
    s = B200GraphStore(inner(db_path), max_graphs=8)
    for tenant, scan in scans:
        s._graph(tenant, scan)                           # graphs cached, compliance tables not yet built
    barrier = threading.Barrier(threads)
    out: dict[int, str] = {}

    def run(k):
        tenant, scan = scans[k % len(scans)]
        barrier.wait()
        out[k] = call(s, {"tenant_id": tenant, "scan_id": scan, "framework": ("", "owasp")[k % 2]})

    ts = [threading.Thread(target=run, args=(k,)) for k in range(threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for k in range(threads):
        tenant, scan = scans[k % len(scans)]
        want = next(c["expected"] for c in CASES if c["kwargs"] == {"tenant_id": tenant, "scan_id": scan, "framework": ("", "owasp")[k % 2]})
        assert out[k] == json.dumps(want)


def test_concurrent_first_calls_on_one_graph(db_path):  # noqa: F811
    _first_calls(db_path, [("", "kat")], 8)


def test_concurrent_first_calls_on_two_graphs(db_path):  # noqa: F811
    _first_calls(db_path, [("compliance", "est40"), ("", "kat")], 8)


# ── memory ──
def test_table_bytes_return_to_zero_with_the_graph(db_path):  # noqa: F811
    s = B200GraphStore(inner(db_path))
    s.compliance_summary(tenant_id="", scan_id="kat")
    g = s._graph("", "kat")
    assert g._compliance is not None and g.device_graph.compliance_table_bytes() > 0
    g._invalidate()
    assert g._compliance is None and g.device_graph.compliance_table_bytes() == 0


def test_store_drops_its_table_with_the_graph(db_path):  # noqa: F811
    import gc

    import torch

    def cycle():
        s = B200GraphStore(inner(db_path))
        s.compliance_summary(tenant_id="compliance", scan_id="est40")
        g = s._graph("compliance", "est40")
        assert g._compliance is not None and g.device_graph.compliance_table_bytes() > 0
        del s, g

    cycle()
    gc.collect()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
        gc.collect()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20
