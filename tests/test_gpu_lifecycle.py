"""Edge lifecycle reads on the H100: ``B200GraphStore.active_edges_at`` and ``changed_edges_between_scans`` against every reference
golden (oracle/make_lifecycle_golden.py); seeded random multi-snapshot histories against the Python oracle at many timestamps; a
snapshot written by a second connection between two calls; the id limit's error; histories freed on eviction and on handle drop;
concurrent calls on one tenant; and ``diff_snapshots`` on the delta goldens, unchanged by the shared-pair extension.
"""

from __future__ import annotations

import gzip
import json
import shutil
import sqlite3
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
from oracle import lifecycle_oracle

from agent_bom_b200 import _lib
from agent_bom_b200.engine import EdgeHistory
from agent_bom_b200.graph import lifecycle
from agent_bom_b200.store import B200GraphStore

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
EXPECTED = json.loads(gzip.decompress((GOLD / "lifecycle" / "expected.json.gz").read_bytes()))
ACTIVE, CHANGES = EXPECTED["active"], EXPECTED["changes"]
CHANGE_IDS = [f"{c['db']}:{c['tenant'].strip() or '-'}:{c['old'] or 'blank'}>{c['new'] or 'blank'}" for c in CHANGES]
DELTA = json.loads(gzip.decompress((GOLD / "delta" / "expected.json.gz").read_bytes()))


def plain(body):
    return json.loads(json.dumps(body))


def store(db_path, **kw) -> B200GraphStore:
    return B200GraphStore(SimpleNamespace(_db_path=str(db_path), load_graph=lambda **_: None), **kw)


def ro(db_path) -> sqlite3.Connection:
    return sqlite3.connect(f"file:{db_path}?mode=ro", uri=True)


@pytest.fixture(scope="module")
def dbs(tmp_path_factory) -> dict[str, Path]:
    root = tmp_path_factory.mktemp("lifecycle")
    out = {}
    for name, src in (("lifecycle", GOLD / "lifecycle" / "graph.sqlite.gz"), ("delta", GOLD / "delta" / "graph.sqlite.gz")):
        out[name] = root / f"{name}.sqlite"
        out[name].write_bytes(gzip.decompress(src.read_bytes()))
    return out


def test_store_active_matches_reference(dbs):
    s = store(dbs["lifecycle"])
    for case in ACTIVE:
        assert plain(s.active_edges_at(case["at"], tenant_id=case["tenant"])) == case["edges"], (case["tenant"], case["at"])


@pytest.mark.parametrize("case", CHANGES, ids=CHANGE_IDS)
def test_store_changes_match_reference(dbs, case):
    body = store(dbs[case["db"]]).changed_edges_between_scans(case["old"], case["new"], tenant_id=case["tenant"])
    assert plain(body) == case["body"]


@pytest.mark.parametrize("case", DELTA, ids=[f"{c['tenant'].strip() or '-'}:{c['old'] or 'blank'}>{c['new'] or 'blank'}" for c in DELTA])
def test_diff_snapshots_unchanged(dbs, case):
    assert plain(store(dbs["delta"]).diff_snapshots(case["old"], case["new"], tenant_id=case["tenant"])) == case["diff"]


def stamp(day: int, hour: int = 0) -> str:
    return f"2026-05-{day:02d}T{hour:02d}:00:00+00:00"


def random_history(path: Path, tenant: str, seed: int, snapshots: int = 8, hot: int = 400, pool: int = 24_000, keep: float = 0.6) -> list[str]:
    """A seeded history written with plain SQL in the order a save writes it: ``hot`` keys with a version in every snapshot and a
    pool of keys present with probability ``keep``; ``valid_from`` empty, carried over or fresh; ``valid_to`` NULL, '' or a
    timestamp; two snapshots share a ``created_at``.  Returns the snapshot timestamps."""
    rng = np.random.default_rng(seed)
    ids = [f"n:{i:05d}{'é' if i % 7 == 0 else ''}{chr(0x1F600 + i % 40) if i % 13 == 0 else ''}{'ﬁ' if i % 17 == 0 else ''}" for i in range(3000)]
    rels = ["uses", "depends_on", "hosts", "zz_custom", "affects", "aa_other"]
    src, tgt, rel = rng.integers(0, len(ids), hot + pool), rng.integers(0, len(ids), hot + pool), rng.integers(0, len(rels), hot + pool)
    keys = sorted({(ids[s], ids[t], rels[r]) for s, t, r in zip(src.tolist(), tgt.tolist(), rel.tolist())})
    created = [stamp(1 + d) for d in range(snapshots)]
    created[3] = created[2]                              # a tie broken by scan id
    conn = sqlite3.connect(str(path))
    try:
        for k, at in enumerate(created):
            present = np.flatnonzero((np.arange(len(keys)) < hot) | (rng.random(len(keys)) < keep))
            vf_kind = rng.integers(0, 3, present.size)
            vt_kind = rng.integers(0, 6, present.size)
            rows = []
            for j, (i, a, b) in enumerate(zip(present.tolist(), vf_kind.tolist(), vt_kind.tolist())):
                s, t, r = keys[i]
                first = stamp(1 + int(rng.integers(0, snapshots)), int(rng.integers(0, 24)))
                vf = "" if a == 0 else (first if a == 1 else stamp(1 + int(rng.integers(0, snapshots + 1)), 12))
                vt = None if b < 3 else ("" if b == 3 else stamp(1 + int(rng.integers(0, snapshots + 1)), int(rng.integers(0, 24))))
                rows.append((s, t, r, first, at, vf, vt, f"r{k}", tenant))
            conn.executemany("INSERT OR REPLACE INTO graph_edges (source_id, target_id, relationship, first_seen, last_seen, valid_from, valid_to, "
                             "scan_id, tenant_id) VALUES (?, ?, ?, ?, ?, ?, ?, ?, ?)", rows)
            conn.execute("INSERT OR REPLACE INTO graph_snapshots VALUES (?, ?, ?, 0, ?, '{}')", (f"r{k}", tenant, at, len(rows)))
            conn.commit()
    finally:
        conn.close()
    return created


@pytest.fixture(scope="module")
def random_db(dbs, tmp_path_factory) -> tuple[Path, list[str]]:
    path = tmp_path_factory.mktemp("random") / "graph.sqlite"
    shutil.copy(dbs["lifecycle"], path)
    created = random_history(path, "rand", 11)
    random_history(path, "rand2", 12, snapshots=4, hot=100, pool=4000)
    return path, created


def test_random_history_matches_oracle(random_db):
    path, created = random_db
    s = store(path)
    conn = ro(path)
    try:
        rows = conn.execute("SELECT COUNT(*) FROM graph_edges WHERE tenant_id = 'rand'").fetchone()[0]
        assert rows > 100_000
        ats = sorted(set(created + [stamp(d, h) for d in (1, 3, 4, 6, 9) for h in (5, 12, 23)] + ["", "z", "2026-05", "2026-05-03T12"]))
        for at in ats:
            want = plain(lifecycle_oracle.active_edges_at(conn, at, "rand"))
            got = plain(s.active_edges_at(at, tenant_id="rand"))
            assert got == want, at
        hot_at = created[-1]
        assert len(s.active_edges_at(hot_at, tenant_id="rand")) > 1000
    finally:
        conn.close()


def test_second_writer_is_seen(random_db, tmp_path):
    src, _ = random_db
    path = tmp_path / "graph.sqlite"
    shutil.copy(src, path)
    s = store(path)
    at = "2026-06-01T00:00:00+00:00"
    first = plain(s.active_edges_at(at, tenant_id="rand2"))
    writer = sqlite3.connect(str(path))
    try:
        prev = writer.execute("SELECT source_id, target_id, relationship FROM graph_edges WHERE tenant_id = 'rand2' AND scan_id = 'r3'").fetchall()
        keep, drop = prev[: len(prev) // 2], prev[len(prev) // 2:]
        now = "2026-05-20T00:00:00+00:00"
        writer.executemany("INSERT OR REPLACE INTO graph_edges (source_id, target_id, relationship, first_seen, last_seen, valid_from, scan_id, tenant_id) "
                           "VALUES (?, ?, ?, ?, ?, ?, 'r9', 'rand2')", [(a, b, c, now, now, now) for a, b, c in keep + [("n:new", "n:newer", "uses")]])
        writer.executemany("UPDATE graph_edges SET valid_to = COALESCE(valid_to, ?) WHERE tenant_id = 'rand2' AND scan_id = 'r3' AND source_id = ? AND "
                           "target_id = ? AND relationship = ?", [(now, a, b, c) for a, b, c in drop])
        writer.execute("INSERT OR REPLACE INTO graph_snapshots VALUES ('r9', 'rand2', ?, 0, 0, '{}')", (now,))
        writer.commit()
    finally:
        writer.close()
    second = plain(s.active_edges_at(at, tenant_id="rand2"))
    assert second != first
    conn = ro(path)
    try:
        assert second == plain(lifecycle_oracle.active_edges_at(conn, at, "rand2"))
    finally:
        conn.close()


def test_id_limit_error(random_db):
    path, _ = random_db
    conn = ro(path)
    try:
        fp = lifecycle.fingerprint(conn, "rand2")
        n_ids = len(lifecycle.TenantHistory(conn, "rand2", fp).ids)
        with pytest.raises(_lib.AbbError, match="exceed the history key's limit"):
            lifecycle.TenantHistory(conn, "rand2", fp, id_limit=n_ids - 1)
        assert lifecycle.TenantHistory(conn, "rand2", fp, id_limit=n_ids).table.n_keys > 0
        with pytest.raises(_lib.AbbError):
            lifecycle.TenantHistory(conn, "rand2", fp, id_limit=(1 << 27) + 1)
    finally:
        conn.close()


def synthetic(n: int, seed: int) -> EdgeHistory:
    rng = np.random.default_rng(seed)
    cols = [rng.integers(0, 50_000, n), rng.integers(0, 50_000, n), rng.integers(0, 8, n)] + [rng.integers(0, 1000, n) for _ in range(3)]
    return EdgeHistory(*cols, 50_000, 8)


def test_histories_are_freed():
    import gc

    import torch

    torch.cuda.init()
    synthetic(1000, 0).active(500)                       # loads the kernels
    free0, _ = torch.cuda.mem_get_info()
    h = synthetic(4_000_000, 1)
    assert h.nbytes >= 16 * 4_000_000
    h.active(500)
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 >= 64 << 20
    del h
    gc.collect()
    free2, _ = torch.cuda.mem_get_info()
    assert abs(free0 - free2) < (4 << 20)


@pytest.fixture(scope="module")
def eviction_db(dbs, tmp_path_factory) -> Path:
    """A small tenant and one of 900 K rows (3 snapshots of 300 K keys): its device table is tens of MB, far above the driver's
    allocation granularity, so its release shows in the device's free memory."""
    path = tmp_path_factory.mktemp("eviction") / "graph.sqlite"
    shutil.copy(dbs["lifecycle"], path)
    random_history(path, "small", 13, snapshots=4, hot=100, pool=4000)
    conn = sqlite3.connect(str(path))
    try:
        for k in range(3):
            at = stamp(1 + k)
            conn.executemany("INSERT INTO graph_edges (source_id, target_id, relationship, first_seen, last_seen, scan_id, tenant_id) "
                             "VALUES (?, ?, 'uses', ?, ?, ?, 'big')", ((f"s:{i}", f"t:{i}", at, at, f"b{k}") for i in range(300_000)))
            conn.execute("INSERT INTO graph_snapshots VALUES (?, 'big', ?, 0, 300000, '{}')", (f"b{k}", at))
        conn.commit()
    finally:
        conn.close()
    return path


def test_eviction_frees_the_oldest(eviction_db):
    import gc
    import weakref

    import torch

    s = store(eviction_db, max_histories=1)
    s.active_edges_at("2027", tenant_id="small")
    gc.collect()
    free0, _ = torch.cuda.mem_get_info()
    assert s.active_edges_at("", tenant_id="big") == []      # builds the history; nothing is active at ''
    big = weakref.ref(next(iter(s._histories._entries.values())).table)
    size = big().nbytes
    assert size >= 16 * 900_000
    free1, _ = torch.cuda.mem_get_info()
    s.active_edges_at("2027", tenant_id="small")            # rebuilt; the big history is evicted
    gc.collect()
    free2, _ = torch.cuda.mem_get_info()
    assert len(s._histories) == 1 and big() is None
    assert free0 - free1 >= size // 2 and abs(free2 - free0) < (4 << 20)


def test_concurrent_calls_agree(random_db):
    path, _ = random_db
    s = store(path)
    ats = [stamp(d) for d in range(1, 6)] + [stamp(d, 12) for d in range(1, 6)]      # the 4-snapshot tenant: a few thousand rows per answer
    want = {at: plain(s.active_edges_at(at, tenant_id="rand2")) for at in ats}
    assert sum(map(len, want.values())) > 1000
    with ThreadPoolExecutor(8) as ex:
        got = list(ex.map(lambda at: (at, plain(s.active_edges_at(at, tenant_id="rand2"))), ats * 3))
    for at, body in got:
        assert body == want[at]
