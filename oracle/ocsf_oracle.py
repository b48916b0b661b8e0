"""CPU oracle of the OCSF export's graph context: numpy over the oracle CSR (oracle.build_csr).

Restates the neighbour half of the reference's ``UnifiedGraph.to_ocsf_events`` (graph/container.py:628-654): the sources of a
finding are ``reverse_adjacency[f]`` in list order — row f of the reverse CSR, reversed twins of bidirectional edges included,
duplicates kept — and the four lists keep the sources with a node record of type agent / server / package / credential.  The
blast-radius half (count, depth, type histogram) is ``oracle.impact_many``.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import oracle as orc

GHOST = 255
#: entity code -> bucket (agent, server, package, credential); 4 = not listed
BUCKET = np.full(256, 4, dtype=np.int8)
BUCKET[0], BUCKET[1], BUCKET[2], BUCKET[10] = 0, 1, 2, 3
N_BUCKETS = 4


@dataclass
class FindingContext:
    count: np.ndarray
    maxd: np.ndarray
    flags: np.ndarray
    hist: np.ndarray
    lists: list          # per finding: N_BUCKETS int32 arrays of source node indices, row order

    def sources(self, q: int, bucket: int) -> np.ndarray:
        return self.lists[q][bucket]

    def bucket_counts(self) -> np.ndarray:
        return np.asarray([[len(x) for x in per] for per in self.lists], dtype=np.int32).reshape(len(self.lists), N_BUCKETS)


def typed_sources(g: orc.OracleGraph, u: int) -> list[np.ndarray]:
    if not 0 <= u < g.n_nodes or int(g.node_type[u]) == GHOST:
        return [np.zeros(0, np.int32) for _ in range(N_BUCKETS)]
    row = g.rev_nbr[int(g.rev_off[u]): int(g.rev_off[u + 1])]
    b = BUCKET[g.node_type[row]]
    return [row[b == k].astype(np.int32) for k in range(N_BUCKETS)]


def finding_context(g: orc.OracleGraph, findings, max_depth: int = 4) -> FindingContext:
    f = np.ascontiguousarray(findings, dtype=np.int32)
    imp = orc.impact_many(g, f, max_depth)
    return FindingContext(count=np.diff(imp.off).astype(np.int32), maxd=imp.maxd, flags=imp.flags, hist=imp.hist,
                          lists=[typed_sources(g, int(u)) for u in f.tolist()])
