"""CPU restatement of the semantic-cluster roll-ups (csrc/clusters.cuh) in numpy, with the device entry points' interface.

``ClusterOracle(csr)`` answers ``build_clusters`` / ``fetch_clusters`` like ``engine.DeviceGraph`` does, so the host pipeline in
``agent_bom_b200/graph/clusters.py`` can run on a machine without a GPU (tests/test_clusters.py checks it against the
reference's goldens) and the device can be checked against it on seeded random graphs (tests/test_gpu_clusters.py).
"""

from __future__ import annotations

import numpy as np

REL_OTHER = 31


class ClusterOracle:
    def __init__(self, csr):
        self.csr = csr
        self.n_nodes = csr.n_nodes
        self.tables = None

    def build_clusters(self, k: int, codes, level, risk, etype) -> dict[str, np.ndarray]:
        c = self.csr
        codes = np.asarray(codes, dtype=np.int64).reshape(-1, 2)
        node = np.repeat(np.arange(codes.shape[0], dtype=np.int64), 2)
        code = codes.reshape(-1)
        keep = code >= 0
        node, code = node[keep], code[keep]
        count = np.bincount(code, minlength=k).astype(np.int64)
        max_risk = np.zeros(k, np.float64)
        np.maximum.at(max_risk, code, np.asarray(risk, np.float64)[node])
        hist = np.zeros((k, 5), np.int64)
        np.add.at(hist, (code, np.asarray(level, np.int64)[node]), 1)
        type_mask = np.zeros(k, np.uint64)
        np.bitwise_or.at(type_mask, code, np.left_shift(np.uint64(1), np.asarray(etype, np.uint64)[node]))
        # members in id-string order: stable sort by (cluster, rank)
        order = np.lexsort((np.asarray(c.node_rank, np.int64)[node], code))
        members = node[order].astype(np.int32)
        mem_off = np.concatenate([[0], np.cumsum(count)])
        # relationship counts: each original edge once per distinct cluster among its endpoints, relationship 31 excluded
        e = np.flatnonzero(np.asarray(c.rel) != REL_OTHER)
        src, dst, rel = np.asarray(c.src, np.int64)[e], np.asarray(c.dst, np.int64)[e], np.asarray(c.rel, np.int64)[e]
        ends = np.stack([codes[src, 0], codes[src, 1], codes[dst, 0], codes[dst, 1]], axis=1)
        edge_id = np.repeat(np.arange(len(e), dtype=np.int64), 4)
        flat = ends.reshape(-1)
        ok = flat >= 0
        pairs = np.unique(np.stack([edge_id[ok], flat[ok]], axis=1), axis=0) if ok.any() else np.zeros((0, 2), np.int64)
        keys = (pairs[:, 1] << 5) | rel[pairs[:, 0]]
        ukeys, ucnt = np.unique(keys, return_counts=True)
        rel_nnz = np.bincount(ukeys >> 5, minlength=k).astype(np.int64)
        rel_off = np.concatenate([[0], np.cumsum(rel_nnz)])
        self.tables = (members, mem_off, (ukeys & 31).astype(np.uint8), ucnt.astype(np.int64), rel_off)
        return {"count": count, "max_risk": max_risk, "hist": hist, "type_mask": type_mask, "rel_nnz": rel_nnz}

    def fetch_clusters(self, sel, n_members: int, n_pairs: int):
        members, mem_off, rel, cnt, rel_off = self.tables
        sel = np.asarray(sel, dtype=np.int64)
        m = [members[mem_off[s]: mem_off[s + 1]] for s in sel]
        r = [np.arange(rel_off[s], rel_off[s + 1]) for s in sel]
        ri = np.concatenate(r) if r else np.zeros(0, np.int64)
        out_m = np.concatenate(m) if m else np.zeros(0, np.int32)
        assert out_m.shape[0] == n_members and ri.shape[0] == n_pairs
        return out_m.astype(np.int32), rel[ri], cnt[ri]
