"""CPU restatement of the compliance roll-up's device part (csrc/compliance.cuh) in numpy.

``ComplianceOracle()`` answers ``compliance_table`` / ``compliance_table_bytes`` like ``engine.DeviceGraph`` does, so the host
pipeline in ``agent_bom_b200/graph/compliance.py`` runs without a GPU (tests/test_compliance.py checks it against the reference's
goldens) and the device can be checked against it on seeded random tables (tests/test_gpu_compliance.py).

The pairs are expanded with ``np.repeat`` and each roll-up is ``np.unique`` over (framework, code) pairs, with the first row
taken as the minimum row of each group, not by a stable radix sort.
"""

from __future__ import annotations

import numpy as np

NODE_IDS = 100


def _runs(fw: np.ndarray, code: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """[4, runs] int64 (framework, code, pairs, first row) in (framework, code) order."""
    if fw.size == 0:
        return np.zeros((4, 0), np.int64)
    width = int(code.max()) + 1
    keys, inverse, counts = np.unique(fw * width + code, return_inverse=True, return_counts=True)
    first = np.full(keys.shape[0], np.iinfo(np.int64).max, np.int64)
    np.minimum.at(first, inverse, rows)
    return np.stack([keys // width, keys % width, counts, first]).astype(np.int64)


class ComplianceOracle:
    def __init__(self):
        self.table = None

    def compliance_table(self, row_text, row_sev, row_type, text_off, text_tags, tag_fw, n_fw, n_sev, n_types):
        row_text = np.asarray(row_text, np.int64)
        text_off = np.asarray(text_off, np.int64)
        text_tags = np.asarray(text_tags, np.int64)
        tag_fw = np.asarray(tag_fw, np.int64)
        length = (text_off[1:] - text_off[:-1])[row_text]
        rows = np.repeat(np.arange(row_text.shape[0], dtype=np.int64), length)
        start = np.repeat(text_off[row_text] - np.concatenate([[0], np.cumsum(length)[:-1]]), length) if rows.size else rows
        tag = text_tags[start + np.arange(rows.shape[0])] if rows.size else rows
        fw = tag_fw[tag] if rows.size else rows
        distinct = _runs(fw, rows, rows)                  # distinct (framework, row) pairs, framework then row order
        node_count = np.bincount(distinct[0], minlength=n_fw).astype(np.int64)
        rank = np.arange(distinct.shape[1]) - np.searchsorted(distinct[0], distinct[0])      # position within the framework
        tags = _runs(fw, tag, rows)
        tags[3] = -1                                        # the device keeps no first row for tags
        self.table = {"sev": _runs(fw, np.asarray(row_sev, np.int64)[rows], rows), "type": _runs(fw, np.asarray(row_type, np.int64)[rows], rows),
                      "tag": tags, "node_count": node_count, "node_rows": distinct[1][rank < NODE_IDS].astype(np.int32)}
        return {k: v.copy() for k, v in self.table.items()}

    def compliance_table_bytes(self) -> int:
        return 0 if self.table is None else 1
