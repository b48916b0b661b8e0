"""CPU restatement of the snapshot lookups' device part (csrc/lookup.cuh) in numpy over the host CSR.

``LookupOracle(csr)`` answers ``build_lookup_table`` / ``incident_edges`` / ``context_edges`` like ``engine.DeviceGraph`` does, and
``impact_of(graph, node_id)`` restates the reference engine's blast-radius walk (graph/container.py:230-279) over the host CSR, so the
host pipeline in ``agent_bom_b200/graph/lookup.py`` runs without a GPU (tests/test_store_lookup.py checks it against the reference's
goldens) and the device can be checked against it on seeded random graphs (tests/test_gpu_store_lookup.py).
"""

from __future__ import annotations

from collections import deque

import numpy as np

REVERSED = 0x80


class LookupOracle:
    def __init__(self, csr):
        self.csr = csr
        self.n_nodes = csr.n_nodes
        self.erel = None

    def build_lookup_table(self, n_real: int, severity, erel) -> dict[str, np.ndarray]:
        c = self.csr
        self.erel = np.asarray(erel, np.uint8)
        both = (c.src < n_real) & (c.dst < n_real)
        return {"type": np.bincount(c.node_type[:n_real], minlength=256).astype(np.int64),
                "severity": np.bincount(np.asarray(severity, np.uint8), minlength=256).astype(np.int64),
                "relationship": np.bincount(self.erel[both], minlength=64).astype(np.int64)}

    def _original_entries(self, u: int):
        """Edge ids of the entries of u's forward and reverse rows whose reversed bit is clear."""
        c = self.csr
        f = slice(int(c.fwd_off[u]), int(c.fwd_off[u + 1]))
        r = slice(int(c.rev_off[u]), int(c.rev_off[u + 1]))
        fe = c.fwd_eid[f][(c.fwd_meta[f] & REVERSED) == 0] >> 1
        re = c.rev_eid[r][(c.rev_meta[r] & REVERSED) == 0] >> 1
        return fe, re

    def incident_edges(self, nodes) -> np.ndarray:
        parts = [np.concatenate(self._original_entries(int(u))) for u in np.asarray(nodes).tolist()]
        return np.unique(np.concatenate(parts)).astype(np.int32) if parts else np.zeros(0, np.int32)

    def context_edges(self, node: int) -> np.ndarray:
        if self.erel is None:
            raise RuntimeError("lookup table is not built")
        c = self.csr
        e = np.unique(np.concatenate(self._original_entries(int(node)))).astype(np.int64)
        rank = c.node_rank.astype(np.int64)
        key = (rank[c.src[e]] << 33) | (rank[c.dst[e]] << 6) | self.erel[e].astype(np.int64)
        return e[np.argsort(key, kind="stable")].astype(np.int32)


def impact_of(graph, node_id: str, max_depth: int = 4) -> dict:
    """Reverse BFS from ``node_id``: a reverse row of the CSR is the reference's ``reverse_adjacency`` list of that node."""
    c = graph.csr
    u = c.idx(node_id)
    if not 0 <= u < c.n_real:
        return {"node_id": node_id, "affected_nodes": [], "affected_by_type": {}, "affected_count": 0, "max_depth_reached": 0}
    seen, queue, reached = {u}, deque([(u, 0)]), 0
    while queue:
        v, d = queue.popleft()
        if d >= max_depth:
            continue
        for w in c.rev_nbr[int(c.rev_off[v]): int(c.rev_off[v + 1])].tolist():
            if w not in seen:
                seen.add(w)
                queue.append((w, d + 1))
                reached = max(reached, d + 1)
    seen.discard(u)
    ids = [c.node_ids[i] for i in seen]
    by_type: dict[str, int] = {}
    for nid in ids:
        node = graph.nodes.get(nid)
        if node is not None:
            k = getattr(node.entity_type, "value", node.entity_type)
            by_type[k] = by_type.get(k, 0) + 1
    return {"node_id": node_id, "affected_nodes": sorted(ids), "affected_by_type": by_type, "affected_count": len(ids), "max_depth_reached": reached}
