"""Node search on the H100: every golden case through ``B200GraphStore`` with the graph cached both by topology-first loading and by
``save_graph``, against the unmodified SQLite store (oracle/make_search_golden.py); seeded random search tables against the numpy
oracle (oracle/search_oracle.py), one with more than 2^20 rows and matches and rows longer than 64 KB; concurrent calls on one
graph; and the table's memory returned with the graph.
"""

from __future__ import annotations

import random
from types import SimpleNamespace

import numpy as np
import pytest
from oracle.search_oracle import SEV_NULL, SearchOracle
from test_gpu_store_lookup import saved_graph
from test_search import CASES, IDS, call, db_path  # noqa: F401  (db_path: the module fixture)

from agent_bom_b200.engine import DeviceGraph
from agent_bom_b200.graph import csr as csrmod
from agent_bom_b200.graph.search import MODE_ALL, MODE_FTS, MODE_LIKE, fold_table
from agent_bom_b200.store import B200GraphStore

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def loading_store(db_path):  # noqa: F811
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))


@pytest.fixture(scope="module")
def saving_store(db_path):  # noqa: F811
    s = B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None, save_graph=lambda _g: None), max_graphs=8)
    for tenant, scan in (("search", "est40"), ("", "kat"), ("", "kat-noindex")):
        s.save_graph(saved_graph(db_path, tenant, scan))
    return s


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_search_by_loading(loading_store, case):
    assert call(loading_store, case) == case["expected"]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_store_search_by_save_graph(saving_store, case):
    assert call(saving_store, case) == case["expected"]


# ── seeded random tables against the oracle ──
WORDS = ["agent", "server", "cve-2024", "pkg:npm/x", "é", "naïve", "日本", "😀", "i̇stanbul", "straße", "ǆ", "x_y", "a.b:c", "́", "ｆｕｌｌ",
         "{\"k\": 1}", "claude-desktop", "osv", "σίσυφος", "éclair"]


def graph_handle() -> DeviceGraph:
    z = np.zeros(0, np.int32)
    return DeviceGraph.upload(csrmod.from_arrays(["n"], np.zeros(1, np.uint8), z, z, z.astype(np.uint8), z.astype(np.uint8), n_real=1))


def random_table(seed: int, n: int, long_rows: int = 0, words: int = 6):
    rng = random.Random(seed)
    rows = [" ".join(rng.choice(WORDS) + (str(rng.randrange(40)) if rng.random() < 0.5 else "") for _ in range(rng.randint(0, words)))
            for _ in range(n)]
    for k in range(long_rows):           # rows longer than 64 KB, a needle near the end
        rows[rng.randrange(n)] = " ".join(rng.choice(WORDS) for _ in range(12_000)) + f" needle{k} tail"
    enc = [r.encode() for r in rows]
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum([len(e) for e in enc])
    nr = np.random.default_rng(seed)
    sev = np.where(nr.random(n) < 0.05, SEV_NULL, nr.integers(-1, 6, n)).astype(np.int32)
    risk = nr.choice([0.0, -0.0, 1.5, 7.5, 9.8, np.nan, np.inf], n)
    label = nr.integers(0, max(n // 3, 1), n).astype(np.uint32)
    types = nr.integers(0, 7, n).astype(np.int32)
    cmp = np.where(nr.random(n) < 0.03, -1, nr.integers(0, 9, n)).astype(np.int32)
    src = np.where(cmp < 0, -1, nr.integers(0, 5, n)).astype(np.int32)
    return off, b"".join(enc), (sev, risk, label, types, cmp, src, 7, 9, 5)


def specs(seed: int, n: int, table) -> list[dict]:
    sev, risk, label = table[0], table[1], table[2]
    rng = np.random.default_rng(seed)
    out = [dict(mode=MODE_ALL, patterns=[]), dict(mode=MODE_FTS, patterns=[b"agent"]), dict(mode=MODE_FTS, patterns=[b"cve 2024", b"s"]),
           dict(mode=MODE_FTS, patterns=[b"needle0"]), dict(mode=MODE_LIKE, patterns=[b"\xc3\xa9"]), dict(mode=MODE_LIKE, patterns=[b""]),
           dict(mode=MODE_LIKE, patterns=[b"tail"]), dict(mode=MODE_FTS, patterns=[b"x y"]), dict(mode=MODE_FTS, patterns=[b"e"])]
    full = []
    for k, s in enumerate(out):
        for variant in range(3):
            d = dict(s, offset=int(rng.integers(0, 5)) * variant, take=int(rng.integers(-1, 60)))
            if variant >= 1:
                d.update(type_ok=rng.integers(0, 2, 7).astype(np.uint8), min_rank=int(rng.integers(-1, 4)))
                if s["mode"]:
                    d.update(cmp_ok=rng.integers(0, 2, 9).astype(np.uint8), src_ok=rng.integers(0, 2, 5).astype(np.uint8))
            if variant == 2:
                i = int(rng.integers(0, n))
                r = float(risk[i])
                d.update(offset=0, cursor=(int(sev[i]) if sev[i] != SEV_NULL else 0, None if r != r or k == 3 else r, int(label[i]) + 1, int(label[i]), i + 1))
            full.append(d)
    return full


def compare(dg, o, spec):
    got, want = dg.search(**spec), o.search(**spec)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], {k: v for k, v in spec.items() if k != "patterns"}


@pytest.mark.parametrize("seed,n,long_rows,words", [(1, 3_000, 0, 6), (2, 40, 2, 3), (3, 1_100_000, 3, 2)])
def test_random_tables_match_oracle(seed, n, long_rows, words):
    off, text, table = random_table(seed, n, long_rows, words)
    dg, o = graph_handle(), SearchOracle()
    try:
        cps = dg.search_text(off, text)
        assert np.array_equal(cps, o.search_text(off, text))
        fold = fold_table(cps)
        dg.build_search_table(fold, *table)
        o.build_search_table(fold, *table)
        if long_rows:
            assert int(np.diff(off).max()) > 64 << 10
        for spec in specs(seed, n, table)[:: 3 if n > 1 << 20 else 1]:       # the oracle is a Python loop per row
            compare(dg, o, spec)
        if n > 1 << 20:
            _, total, _ = dg.search(MODE_LIKE, [b""], take=10)
            assert total > 1 << 20
    finally:
        dg.close()


def test_concurrent_searches_on_one_graph():
    from concurrent.futures import ThreadPoolExecutor

    off, text, table = random_table(5, 50_000, 1)
    dg, o = graph_handle(), SearchOracle()
    try:
        fold = fold_table(dg.search_text(off, text))
        o.search_text(off, text)
        dg.build_search_table(fold, *table)
        o.build_search_table(fold, *table)
        work = specs(6, 50_000, table) * 3
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda s: dg.search(**s), work))
        for s, g in zip(work, got):
            want = o.search(**s)
            assert np.array_equal(g[0], want[0]) and g[1:] == want[1:]
    finally:
        dg.close()


def test_table_needs_text_and_is_freed_with_the_graph():
    import torch

    off, text, table = random_table(7, 200_000, 2)

    def cycle():
        dg = graph_handle()
        try:
            with pytest.raises(RuntimeError):
                dg.search(MODE_ALL, [])
            fold = fold_table(dg.search_text(off, text))
            assert dg.search_table_bytes() == 0
            dg.build_search_table(fold, *table)
            assert dg.search_table_bytes() > len(text)
            for _ in range(3):
                dg.search(MODE_FTS, [b"agent"], take=50)
            dg.search_text(off, text)                 # replacing the text drops the table until it is built again
            assert dg.search_table_bytes() == 0
        finally:
            dg.close()

    torch.cuda.mem_get_info()
    cycle()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20


def test_store_drops_its_table_with_the_graph(db_path):  # noqa: F811
    import gc

    import torch

    def cycle():
        s = B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None))
        s.search_nodes(tenant_id="search", scan_id="est40", query="agent")
        g = s._graph("search", "est40")
        assert g._search is not None and g.device_graph.search_table_bytes() > 0
        del s, g

    cycle()
    gc.collect()
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle()
        gc.collect()
    free_after, _ = torch.cuda.mem_get_info()
    assert free_before - free_after <= 4 << 20
