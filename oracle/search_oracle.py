"""CPU restatement of the node search's device part (csrc/search.cuh) in numpy and Python strings.

``SearchOracle()`` answers ``search_text`` / ``build_search_table`` / ``search`` / ``search_table_bytes`` like ``engine.DeviceGraph``
does, so the host pipeline in ``agent_bom_b200/graph/search.py`` runs without a GPU (tests/test_search.py checks it against the
reference's goldens) and the device can be checked against it on seeded random snapshots (tests/test_gpu_search.py).

The token text is built here as ``str.translate`` with the fold table (separators to a space, code points that fold away deleted)
followed by a split at spaces that drops empty tokens, not by the device's per-row state machine.
"""

from __future__ import annotations

import numpy as np

SEV_NULL = -(1 << 31)


def token_text(raw: str, fold) -> str:
    table = {}
    for ch in set(raw):
        f = int(fold[ord(ch)])
        table[ord(ch)] = " " if f < 0 else (chr(f) if f else None)
    return " ".join(w for w in raw.translate(table).split(" ") if w)


def _desc_risk(risk: np.ndarray) -> np.ndarray:
    """Sort key of risk descending with NULL (NaN) last, -0.0 equal to 0.0."""
    r = np.where(risk == 0.0, 0.0, risk)
    return np.where(np.isnan(r), np.inf, -r)


class SearchOracle:
    def __init__(self):
        self.rows: list[str] = []
        self.table = None

    def search_text(self, text_off, text: bytes) -> np.ndarray:
        off = np.asarray(text_off, np.int64).tolist()
        self.rows = [text[a:b].decode() for a, b in zip(off[:-1], off[1:])]
        self.table = None
        return np.array(sorted({ord(c) for row in self.rows for c in row if ord(c) >= 0x80}), np.int64)

    def build_search_table(self, fold, severity, risk, label_rank, type_code, cmp_code, src_code, n_types, n_cmp, n_src) -> None:
        sev = np.asarray(severity, np.int64)
        risk = np.asarray(risk, np.float64)
        label = np.asarray(label_rank, np.int64)
        n = len(self.rows)
        order = np.lexsort((np.arange(n), label, _desc_risk(risk), np.where(sev == SEV_NULL, np.inf, -sev.astype(np.float64))))
        self.table = {"tok": [token_text(r, fold) for r in self.rows], "sev": sev, "risk": risk, "label": label, "type": np.asarray(type_code),
                      "cmp": np.asarray(cmp_code), "src": np.asarray(src_code), "order": order}

    def search_table_bytes(self) -> int:
        return 0 if self.table is None else 1

    def _cursor(self, i, cursor) -> bool:
        t = self.table
        cs, cr, label_gt, label_eq, id_gt = cursor
        s, r, lab = int(t["sev"][i]), float(t["risk"][i]), int(t["label"][i])
        if s == SEV_NULL:
            return False
        if s != cs:
            return s < cs
        if r != r or cr is None:
            return False
        if r != cr:
            return r < cr
        if lab >= label_gt:
            return True
        return lab == label_eq and i >= id_gt

    def search(self, mode, patterns, type_ok=None, cmp_ok=None, src_ok=None, min_rank=None, cursor=None, offset=0, take=-1):
        if self.table is None:
            raise RuntimeError("search table is not built")
        t = self.table
        pats = [p.decode() for p in patterns]
        total = 0
        selected = []
        for i in t["order"].tolist():
            if mode and t["cmp"][i] < 0:
                continue
            if type_ok is not None and not type_ok[t["type"][i]]:
                continue
            if min_rank is not None and (t["sev"][i] == SEV_NULL or t["sev"][i] < min_rank):
                continue
            if cmp_ok is not None and not cmp_ok[t["cmp"][i]]:
                continue
            if src_ok is not None and not src_ok[t["src"][i]]:
                continue
            if mode == 1 and not all((" " + t["tok"][i]).find(" " + p) >= 0 for p in pats):
                continue
            if mode == 2 and not all(p in self.rows[i] for p in pats):
                continue
            total += 1
            if cursor is None or self._cursor(i, cursor):
                selected.append(i)
        end = len(selected) if take < 0 else offset + take
        return np.asarray(selected[offset:end], np.int32), total, len(selected)
