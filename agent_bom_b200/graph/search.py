"""Node search and keyset pages served from the snapshot cache.

The reference's SQLite store answers ``search_nodes`` and ``page_nodes`` (reference ``api/graph_store.py:1242-1313,
1346-1468``) with an FTS5 ``MATCH`` (or a ``LIKE`` scan) over ``graph_node_search`` joined to ``graph_nodes``, a ``COUNT(*)`` of every
hit and a sort of every hit, per request.  Here each cached graph gets a search table once (``csrc/search.cuh``), built from the
scan's ``graph_node_search`` rows and one ``graph_nodes`` query, and a request is one device call: match, filter, cursor, count
and the page in sort order.  SQLite is asked only for the page's records, by primary key.

- FTS path (``q`` has a character ``isalnum()`` accepts and a ``[A-Za-z0-9_.:-]+`` token): each token is the phrase ``"tok"*``,
  the phrases ANDed.  unicode61 splits a token at ``_ . : -``; a phrase's folded tokens joined by one space, the last one a prefix,
  match a row exactly when they occur at a token start of the row's token text (its ``search_text`` tokenised and folded as
  unicode61 does, tokens joined by one space).  Every indexed column's text occurs, lowered, inside ``search_text`` at token
  boundaries, so matching ``search_text`` alone is matching the row (tests/test_search.py checks both against FTS5).  A phrase
  that tokenises to nothing matches nothing.
- LIKE path otherwise: ``search_text`` holds ``q.lower()`` as a plain substring (the reference escapes ``%``, ``_`` and ``\\``).
- How unicode61 folds each code point is asked of the SQLite library this process links (``unicode61_folds``), never restated.
- Order ``severity_id DESC, risk_score DESC, label, id`` with NULLs last; the cursor's keyset predicate keeps SQL's NULL rules.
"""

from __future__ import annotations

import base64
import json
import re
import sqlite3
import threading
from bisect import bisect_left, bisect_right
from collections import defaultdict
from typing import Any

import numpy as np

from .lookup import connect, node_records

MODE_ALL, MODE_FTS, MODE_LIKE = 0, 1, 2
CODEPOINTS = 0x110000
SEV_NULL = -(1 << 31)
_TOKEN = re.compile(r"[A-Za-z0-9_.:-]+")
_INT64 = (-(1 << 63), (1 << 63) - 1)
_lock = threading.Lock()
_folds: dict[int, int] = {}
_fold_lock = threading.Lock()


# ── unicode61, asked of SQLite ──
def unicode61_folds(codepoints) -> dict[int, int]:
    """How FTS5's default tokenizer (unicode61, remove_diacritics=1) treats each code point: -1 separator, 0 folds away, else the
    code point it folds to.  Each ``a<c>a`` is tokenised in an in-memory FTS5 table and its terms read back through fts5vocab:
    ``a``, ``a`` is a separator, ``a<f>a`` a fold to ``f``, ``aa`` a fold to nothing.  Answers are kept for the process."""
    cps = [int(c) for c in codepoints]
    with _fold_lock:
        todo = [c for c in cps if c not in _folds]
        if todo:
            terms: dict[int, list[str]] = defaultdict(list)
            probe = [c for c in todo if not 0xD800 <= c <= 0xDFFF]      # surrogates are not text
            conn = sqlite3.connect(":memory:")
            try:
                conn.execute("CREATE VIRTUAL TABLE p USING fts5(x)")
                conn.execute("CREATE VIRTUAL TABLE v USING fts5vocab(p, 'instance')")
                conn.executemany("INSERT INTO p(rowid, x) VALUES (?, ?)", [(c + 1, f"a{chr(c)}a") for c in probe])
                for term, doc in conn.execute("SELECT term, doc FROM v"):
                    terms[doc - 1].append(term)
            finally:
                conn.close()
            for c in todo:
                t = terms.get(c, ["a", "a"])
                if t == ["a", "a"]:
                    f = -1
                elif len(t) == 1 and 2 <= len(t[0]) <= 3 and t[0][0] == "a" and t[0][-1] == "a":
                    f = ord(t[0][1]) if len(t[0]) == 3 else 0
                else:
                    raise RuntimeError(f"unicode61 turns U+{c:04X} into {t!r}, not into one code point or none")
                _folds[c] = f
        return {c: _folds[c] for c in cps}


def fold_table(codepoints) -> np.ndarray:
    """Dense fold table [0x110000] for ASCII and ``codepoints`` (other entries -1)."""
    folds = unicode61_folds(list(range(128)) + [int(c) for c in codepoints])
    table = np.full(CODEPOINTS, -1, np.int32)
    table[np.fromiter(folds.keys(), np.int64, len(folds))] = np.fromiter(folds.values(), np.int32, len(folds))
    return table


def query_plan(query: str) -> tuple[int, list[bytes] | None]:
    """``(MODE_FTS, phrases)`` or ``(MODE_LIKE, [pattern])`` for ``q`` as the reference decides (:301-310, :1460); phrases are
    ``None`` when one of them tokenises to nothing (the search then matches nothing)."""
    tokens = [t.strip() for t in _TOKEN.findall(query) if t.strip()]
    if tokens and any(ch.isalnum() for ch in query):
        ascii_fold = unicode61_folds(range(128))
        phrases = []
        for tok in tokens:
            folded = "".join(" " if ascii_fold[ord(ch)] < 0 else chr(ascii_fold[ord(ch)]) if ascii_fold[ord(ch)] else "" for ch in tok)
            words = [w for w in folded.split(" ") if w]
            if not words:
                return MODE_FTS, None
            phrases.append(" ".join(words).encode())
        return MODE_FTS, phrases
    return MODE_LIKE, [query.lower().encode()]


# ── filters: the reference's LIKE clauses, evaluated once per distinct stored string ──
def _escape_like(text: str) -> str:
    return text.replace("\\", "\\\\").replace("%", "\\%").replace("_", "\\_")


def compliance_match(tags: str, prefix: str) -> bool:
    """``tags = p OR LIKE 'p-%' OR 'p %' OR '% p-%' OR '% p %'`` (:327-334): ``=`` compares the escaped prefix, the LIKE patterns
    match it literally.  There is no ``'% p'`` clause, so a last tag equal to ``p`` does not match unless it is the only one."""
    p = prefix.lower()
    return tags == _escape_like(p) or tags.startswith(p + "-") or tags.startswith(p + " ") or f" {p}-" in tags or f" {p} " in tags


def source_match(sources: str, source: str) -> bool:
    """``sources = d OR LIKE 'd %' OR '% d' OR '% d %'`` (:320-324)."""
    d = source.lower()
    return sources == _escape_like(d) or sources.startswith(d + " ") or sources.endswith(" " + d) or f" {d} " in sources


# ── cursors (:73-92) ──
def decode_cursor(cursor: str) -> tuple[int, float, str, str]:
    try:
        padded = cursor + "=" * (-len(cursor) % 4)
        values = json.loads(base64.urlsafe_b64decode(padded.encode()).decode())
        if not isinstance(values, list) or len(values) != 4:
            raise ValueError
        severity_id, risk_score, label, node_id = values
        return int(severity_id), float(risk_score), str(label), str(node_id)
    except Exception as exc:
        raise ValueError("Invalid graph cursor") from exc


def encode_cursor(node) -> str:
    key = [int(node.severity_id or 0), float(node.risk_score or 0.0), node.label or "", node.id]
    return base64.urlsafe_b64encode(json.dumps(key, separators=(",", ":"), ensure_ascii=True).encode()).decode().rstrip("=")


def _int64(value: int) -> int:
    if not _INT64[0] <= value <= _INT64[1]:
        raise OverflowError("Python int too large to convert to SQLite INTEGER")        # what binding it to SQLite raises
    return value


class SearchTable:
    """Per-graph search state: the scan's nodes in id order with their keys and interned strings, read once; the device table is
    built on first use.  ``lock`` guards the once-per-graph steps of this graph only."""

    def __init__(self, conn, tenant: str, scan_id: str):
        nodes = conn.execute("SELECT id, entity_type, label, severity_id, risk_score FROM graph_nodes WHERE tenant_id = ? AND scan_id = ?",
                             (tenant, scan_id)).fetchall()
        nodes.sort(key=lambda r: r[0])                   # Python str order = UTF-8 byte order = BINARY collation
        self.ids = [r[0] for r in nodes]
        index = {nid: i for i, nid in enumerate(self.ids)}
        n = len(self.ids)
        try:
            rows = conn.execute("SELECT node_id, compliance_tags, data_sources, search_text FROM graph_node_search WHERE tenant_id = ? AND scan_id = ?",
                                (tenant, scan_id)).fetchall()
        except sqlite3.OperationalError:                 # a database no SQLiteGraphStore opened has no index: nothing is found
            rows = []
        texts: list[bytes] = [b""] * n
        self.cmp_code = np.full(n, -1, np.int32)
        self.src_code = np.full(n, -1, np.int32)
        self.cmp_strings: list[str] = []
        self.src_strings: list[str] = []
        cmp_ix: dict[str, int] = {}
        src_ix: dict[str, int] = {}
        for node_id, tags, sources, text in rows:        # rowid order; the join drops rows of ids that are not nodes
            i = index.get(node_id, -1)
            if i < 0 or self.cmp_code[i] >= 0:
                continue
            tags, sources = tags or "", sources or ""
            self.cmp_code[i] = cmp_ix.setdefault(tags, len(cmp_ix))
            self.src_code[i] = src_ix.setdefault(sources, len(src_ix))
            texts[i] = (text or "").encode()
        self.cmp_strings, self.src_strings = list(cmp_ix), list(src_ix)
        self.text_off = np.zeros(n + 1, np.int64)
        self.text_off[1:] = np.cumsum([len(t) for t in texts])
        self.text = b"".join(texts)
        types: dict[str, int] = {}
        self.type_code = np.fromiter((types.setdefault(r[1], len(types)) for r in nodes), np.int32, n)
        self.types = list(types)
        sev = [r[3] for r in nodes]
        if any(s is not None and not SEV_NULL < s < (1 << 31) for s in sev):
            raise ValueError("severity_id outside the 32-bit range")
        self.severity = np.fromiter((SEV_NULL if s is None else s for s in sev), np.int32, n)
        self.risk = np.fromiter((np.nan if r[4] is None else r[4] for r in nodes), np.float64, n)
        self.labels = sorted({r[2] for r in nodes})
        rank = {lbl: k for k, lbl in enumerate(self.labels)}
        self.label_rank = np.fromiter((rank[r[2]] for r in nodes), np.uint32, n)
        self.lock = threading.Lock()
        self.ready = False

    def ensure_device(self, dg) -> None:
        with self.lock:
            if not self.ready:
                cps = dg.search_text(self.text_off, self.text)
                dg.build_search_table(fold_table(cps), self.severity, self.risk, self.label_rank, self.type_code, self.cmp_code, self.src_code,
                                      len(self.types), len(self.cmp_strings), len(self.src_strings))
                self.ready = True

    def cursor_args(self, key: tuple[int, float, str, str]):
        sev, risk, label, node_id = key
        lo = bisect_left(self.labels, label)
        eq = lo if lo < len(self.labels) and self.labels[lo] == label else -1
        return (_int64(sev), None if risk != risk else risk, bisect_right(self.labels, label), eq, bisect_right(self.ids, node_id))


def search_table(graph, conn, tenant: str) -> SearchTable:
    t = graph._search
    if t is None:
        with _lock:                       # only to give the graph its own lock: building one graph's table never waits on another's
            glock = graph.__dict__.setdefault("_search_lock", threading.Lock())
        with glock:
            t = graph._search
            if t is None:
                t = graph._search = SearchTable(conn, tenant, graph.scan_id)
    return t


def _page(graph, db_path, tenant: str, mode: int, patterns: list[bytes], entity_types, min_severity_rank, compliance_prefixes, data_sources,
          key, offset: int, limit: int):
    """``(nodes, total, next_cursor)`` of one request, as the reference pages (:1445-1451)."""
    conn = connect(db_path)
    try:
        table = search_table(graph, conn, tenant)
        dg = graph.device_graph
        table.ensure_device(dg)
        type_ok = np.fromiter((t in entity_types for t in table.types), np.uint8, len(table.types)) if entity_types else None
        cmp_ok = (np.fromiter((any(compliance_match(s, p) for p in compliance_prefixes) for s in table.cmp_strings), np.uint8, len(table.cmp_strings))
                  if compliance_prefixes else None)
        src_ok = (np.fromiter((any(source_match(s, d) for d in data_sources) for s in table.src_strings), np.uint8, len(table.src_strings))
                  if data_sources else None)
        take = limit + 1 if key is not None else limit   # SQLite: a negative LIMIT is no limit, a negative OFFSET is 0
        page, total, _ = dg.search(mode, patterns, type_ok, cmp_ok, src_ok, _int64(min_severity_rank) if min_severity_rank else None,
                                   None if key is None else table.cursor_args(key), 0 if key is not None else max(offset, 0), take if take >= 0 else -1)
        if total == 0:
            return [], 0, None
        has_more = len(page) > limit if key is not None else offset + limit < total
        ids = [table.ids[i] for i in page.tolist()[:limit]]
        recs = node_records(conn, tenant, graph.scan_id, ids)
    finally:
        conn.close()
    nodes = [recs[nid] for nid in ids if nid in recs]
    return nodes, total, (encode_cursor(nodes[-1]) if has_more and nodes else None)


def search_nodes(graph, db_path, tenant: str, *, query: str, entity_types=None, min_severity_rank: int = 0, compliance_prefixes=None,
                 data_sources=None, key=None, offset: int = 0, limit: int = 50) -> tuple[list, int, str | None]:
    """``search_nodes`` over ``graph`` (the resolved scan); ``key``: the decoded cursor or ``None``."""
    mode, patterns = query_plan(query)
    if patterns is None:
        return [], 0, None
    return _page(graph, db_path, tenant, mode, patterns, entity_types, min_severity_rank, compliance_prefixes, data_sources, key, offset, limit)


def page_nodes(graph, db_path, tenant: str, *, entity_types=None, min_severity_rank: int = 0, key=None, offset: int = 0,
               limit: int = 500) -> tuple[list, int, str | None]:
    """``page_nodes``' ``(nodes, total, next_cursor)`` over ``graph``: the same filters, order and cursor with no text predicate."""
    return _page(graph, db_path, tenant, MODE_ALL, [], entity_types, min_severity_rank, None, None, key, offset, limit)


def cursor_key(cursor: str | None) -> Any:
    return decode_cursor(cursor) if cursor else None
