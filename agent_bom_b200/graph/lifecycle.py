"""Edge versions active at a timestamp (``GET /v1/graph/edges/active?at=``) from a tenant's edge history on the device.

The reference's ``active_edges_at`` (``db/graph_store.py:775-796``) joins every edge row of every snapshot of the tenant to
``graph_snapshots``, builds a row dict for each row that passes its three timestamp tests and keeps the last one per
``(source, target, relationship)`` key in ``(created_at, scan_id)`` order.  Here (``csrc/lifecycle.cuh``):

- once per tenant history, one SQL pass reads the key, the three timestamps and the rowid of every joined row in that order; the
  host interns ids, relationships and timestamps into sorted dictionaries (UTF-8 byte order = ``str`` order = SQLite ``BINARY``)
  and the device sorts the rows by key, stably, into key segments;
- per call the host bisects ``at`` into the timestamp dictionary (``r`` strings are ``<= at``, so ``s <= at`` exactly when
  ``rank(s) < r``), one device thread per key finds the key's last active version, and only the winners' row indices come back;
- the winners' rows are read by rowid and built with the reference's row rule (``edge_history_row``), in key order.

A history is cached per (database, tenant) and keyed by a fingerprint of the tenant's ``graph_snapshots`` rows: every save ends
with an ``INSERT OR REPLACE`` there (a new rowid), so a snapshot written by another process is seen on the next call.  The
fingerprint check, a rebuild and the row reads run in one read transaction.
"""

from __future__ import annotations

import bisect
import sqlite3
import threading
from collections import OrderedDict
from typing import Any

import numpy as np

from .delta import edge_history_row
from .snapshot import normalize_graph_tenant_id

NONE_RANK = 0x7FFFFFFF          # lifecycle.cuh LC_NONE: an absent timestamp
_CHUNK = 500

_ROWS_SQL = ("SELECT ge.rowid, ge.source_id, ge.target_id, ge.relationship, COALESCE(NULLIF(ge.valid_from, ''), ge.first_seen), ge.valid_to, "
             "gs.created_at FROM graph_edges ge JOIN graph_snapshots gs ON gs.tenant_id = ge.tenant_id AND gs.scan_id = ge.scan_id "
             "WHERE ge.tenant_id = ? ORDER BY gs.created_at ASC, ge.scan_id ASC")


def fingerprint(conn, tenant: str) -> tuple:
    """The tenant's ``graph_snapshots`` rows as ``(rowid, scan_id, created_at)``: it changes with every save (an ``INSERT OR
    REPLACE`` gives a new rowid), re-save and deletion."""
    return tuple(conn.execute("SELECT rowid, scan_id, created_at FROM graph_snapshots WHERE tenant_id = ? ORDER BY rowid", (tenant,)).fetchall())


def _ranks(values, rank: dict) -> np.ndarray:
    return np.fromiter((rank[v] for v in values), np.int32, len(values))


def timestamp_rank(stamps: list[str], at: str) -> int:
    """``r``: how many dictionary strings are ``<= at``."""
    return bisect.bisect_right(stamps, at)


def make_history(codes: dict[str, np.ndarray], n_ids: int, n_rels: int, device: int, id_limit: int | None):
    """The device history of the coded rows (``engine.EdgeHistory``)."""
    from ..engine import EdgeHistory

    return EdgeHistory(codes["src"], codes["tgt"], codes["rel"], codes["created"], codes["valid_from"], codes["valid_to"], n_ids, n_rels,
                       device=device, id_limit=id_limit)


class TenantHistory:
    """One tenant's coded edge history: the host dictionaries, the rowid and key codes of every row, and its device table."""

    def __init__(self, conn, tenant: str, fp: tuple, *, device: int = 0, id_limit: int | None = None, timings: dict | None = None):
        import time

        t0 = time.perf_counter()
        rows = conn.execute(_ROWS_SQL, (tenant,)).fetchall()
        t1 = time.perf_counter()
        n = len(rows)
        rowid, src, tgt, rel, vf, vt, cr = (list(c) for c in zip(*rows)) if rows else ([] for _ in range(7))
        self.fingerprint = fp
        self.ids = sorted(set(src) | set(tgt))
        self.rels = sorted(set(rel))
        self.stamps = sorted({s for s in cr if s is not None} | {s for s in vf if s is not None} | {s for s in vt if s})
        id_rank = {s: i for i, s in enumerate(self.ids)}
        ts_rank = {s: i for i, s in enumerate(self.stamps)}
        ts_rank[None] = NONE_RANK
        vt_rank = dict(ts_rank)
        vt_rank[""] = NONE_RANK                  # '' valid_to: open, like NULL
        self.rowid = np.asarray(rowid, np.int64)
        self.src = _ranks(src, id_rank)
        self.tgt = _ranks(tgt, id_rank)
        self.rel = _ranks(rel, {s: i for i, s in enumerate(self.rels)})
        codes = {"src": self.src, "tgt": self.tgt, "rel": self.rel, "created": _ranks(cr, ts_rank), "valid_from": _ranks(vf, ts_rank),
                 "valid_to": _ranks(vt, vt_rank)}
        t2 = time.perf_counter()
        self.table = make_history(codes, len(self.ids), len(self.rels), device, id_limit)
        t3 = time.perf_counter()
        self.n_rows = n
        if timings is not None:
            timings.update(sql_s=t1 - t0, intern_s=t2 - t1, upload_s=t3 - t2)

    def key(self, i: int) -> tuple[str, str, str]:
        return self.ids[self.src[i]], self.ids[self.tgt[i]], self.rels[self.rel[i]]


class StaleHistory(Exception):
    """A winner's rowid no longer holds the row the history coded (rowids renumbered under an unchanged fingerprint)."""


def _hydrate(conn, hist: TenantHistory, winners: np.ndarray) -> list[dict[str, Any]]:
    rowids = hist.rowid[winners].tolist()
    cur = conn.cursor()
    cur.row_factory = sqlite3.Row
    by_rowid: dict[int, Any] = {}
    for a in range(0, len(rowids), _CHUNK):
        chunk = rowids[a: a + _CHUNK]
        for row in cur.execute(f"SELECT rowid, * FROM graph_edges WHERE rowid IN ({','.join('?' * len(chunk))})", chunk):
            by_rowid[row[0]] = row
    out = []
    for i, rid in zip(winners.tolist(), rowids):
        row = by_rowid.get(rid)
        if row is None or (row["source_id"], row["target_id"], row["relationship"]) != hist.key(i):
            raise StaleHistory(rid)
        out.append(edge_history_row(row))
    return out


class HistoryCache:
    """Tenant histories by (database, tenant), least recently used freed first beyond ``max_histories``."""

    def __init__(self, max_histories: int = 4, *, device: int = 0, id_limit: int | None = None):
        self.max_histories = max(1, int(max_histories))
        self.device = device
        self.id_limit = id_limit
        self._lock = threading.Lock()
        self._build_lock = threading.Lock()
        self._entries: "OrderedDict[tuple[str, str], TenantHistory]" = OrderedDict()

    def __len__(self) -> int:
        return len(self._entries)

    def clear(self) -> None:
        with self._lock:
            self._entries.clear()

    def get(self, conn, db_path: str, tenant: str, fp: tuple, *, force: bool = False, timings: dict | None = None) -> TenantHistory:
        """The history of ``fp``, built inside the caller's read transaction when the cached one is older (or ``force``)."""
        key = (str(db_path), tenant)
        with self._lock:
            h = self._entries.get(key)
            if h is not None and h.fingerprint == fp and not force:
                self._entries.move_to_end(key)
                return h
        with self._build_lock:
            with self._lock:
                h = self._entries.get(key)
                if h is not None and h.fingerprint == fp and not force:
                    self._entries.move_to_end(key)
                    return h
                self._entries.pop(key, None)     # the old history is freed once no call is inside it
            h = TenantHistory(conn, tenant, fp, device=self.device, id_limit=self.id_limit, timings=timings)
            with self._lock:
                self._entries[key] = h
                self._entries.move_to_end(key)
                while len(self._entries) > self.max_histories:
                    self._entries.popitem(last=False)
        return h


def active_edges_at(cache: HistoryCache, db_path, at, *, tenant_id: str = "", timings: dict | None = None) -> list[dict[str, Any]]:
    """The body of the reference ``active_edges_at(at, tenant_id=)`` over the SQLite database ``db_path``: the last version of each
    edge key whose snapshot and ``valid_from`` are ``<= at`` and whose ``valid_to`` is open or ``> at``, in key order.
    ``timings`` (optional) receives the seconds of each stage (``build`` stages only when the history was (re)built)."""
    import time

    if at is None or isinstance(at, (int, float)):
        return []        # SQLite: NULL compares to nothing, and a number sorts below every text
    if not isinstance(at, str):
        raise TypeError(f"at must be a string, not {type(at).__name__}")
    at.encode("utf-8")   # what binding the parameter would raise
    tenant = normalize_graph_tenant_id(tenant_id)
    conn = sqlite3.connect(f"file:{db_path}?mode=ro", uri=True, timeout=10)
    t: dict = {}
    try:
        conn.execute("BEGIN")          # the fingerprint, a rebuild and the row reads see one state of the database
        t0 = time.perf_counter()
        fp = fingerprint(conn, tenant)
        t["fingerprint_s"] = time.perf_counter() - t0
        if not fp:
            return []
        for attempt in (0, 1):
            build: dict = {}
            hist = cache.get(conn, db_path, tenant, fp, force=attempt > 0, timings=build)
            t.update(build)
            t0 = time.perf_counter()
            dev: dict = {}
            winners = hist.table.active(timestamp_rank(hist.stamps, at), dev)
            t["call_s"] = time.perf_counter() - t0
            t["device_ms"] = dev.get("device_ms", 0.0)
            t0 = time.perf_counter()
            try:
                out = _hydrate(conn, hist, winners)
            except StaleHistory:
                if attempt:
                    raise
                continue
            t["hydrate_s"] = time.perf_counter() - t0
            return out
    finally:
        conn.close()
        if timings is not None:
            timings.update(t)
    raise AssertionError("unreachable")
