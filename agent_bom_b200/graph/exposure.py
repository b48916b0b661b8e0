"""Derived exposure / attack paths: device rows → ranked ``AttackPath`` records.

Drop-in for the reference's ``_derived_attack_paths``
(``/root/reference/src/agent_bom/api/routes/graph.py:686-786``).  The typed
pattern walk (finding ← vulnerable source ← server ← agent, with the server's
credential / tool fan-out and the per-hop relationships) runs in the CUDA
engine and returns integer rows in the reference's emission order; this module
does what needs Python objects and Python floats: labels, the risk formula
(``:677-683``, ``:762-771`` — same float expressions, same ``round``) and the
final stable descending sort (``:782-786``).
"""

from __future__ import annotations

import numpy as np

from .model import AttackPath
from .schema import ENTITY_CODE_GHOST, RELATIONSHIP_VALUES, SEVERITY_RANK

SUMMARY = ("Derived from graph topology: vulnerable package/server is reachable from an agent "
           "and inherits the server's credential/tool exposure.")
_REL_EXPOSES_CRED, _REL_PROVIDES_TOOL = 4, 3


def node_risk_100(node) -> float:
    """Reference ``_node_risk_100`` (api/routes/graph.py:677-683)."""
    risk = float(getattr(node, "risk_score", 0.0) or 0.0)
    if risk <= 10.0:
        risk *= 10.0
    if risk <= 0:
        risk = float(SEVERITY_RANK.get(str(getattr(node, "severity", "") or "").lower(), 0) * 20)
    return max(0.0, min(100.0, risk))


def server_exposure_labels(graph, server_idx: int) -> tuple[list[str], list[str]]:
    """Labels of the server's EXPOSES_CRED / PROVIDES_TOOL targets, in edge order, originals only (:740-749)."""
    c = graph.csr
    ids = c.node_ids
    creds, tools = [], []
    a, b = int(c.fwd_off[server_idx]), int(c.fwd_off[server_idx + 1])
    for nbr, meta in zip(c.fwd_nbr[a:b].tolist(), c.fwd_meta[a:b].tolist()):
        if meta & 0x80 or c.node_type[nbr] == ENTITY_CODE_GHOST:
            continue
        rel = meta & 0x1F
        if rel == _REL_EXPOSES_CRED:
            creds.append(graph.nodes[ids[nbr]].label)
        elif rel == _REL_PROVIDES_TOOL:
            tools.append(graph.nodes[ids[nbr]].label)
    return creds, tools


def materialize_attack_paths(graph, rows, *, sort: bool = True) -> list[AttackPath]:
    """Rows (emission order) → ``AttackPath`` list in the reference's final order (``sort=False``: rows are already ranked)."""
    ids = graph.csr.node_ids
    cache: dict[int, tuple[list[str], list[str]]] = {}
    out: list[AttackPath] = []
    hops_all, rels_all = rows.hops.tolist(), rows.rels.tolist()
    ncred, ntool = rows.ncred.tolist(), rows.ntool.tolist()
    for i, (a, srv, vs, f) in enumerate(hops_all):
        if srv not in cache:
            cache[srv] = server_exposure_labels(graph, srv)
        creds, tools = cache[srv]
        finding = graph.nodes[ids[f]]
        risk = node_risk_100(finding)
        risk += min(10.0, ncred[i] * 3.0)          # counts of the un-deduplicated label lists (:763-764)
        risk += min(10.0, ntool[i] * 0.75)
        hop_ids = [ids[a], ids[srv]] + ([ids[vs]] if vs >= 0 else []) + [ids[f]]
        out.append(AttackPath(
            source=ids[a], target=ids[f], hops=hop_ids, edges=[RELATIONSHIP_VALUES[r] if r < 31 else "other" for r in rels_all[i] if r >= 0],
            composite_risk=round(min(100.0, risk), 2), summary=SUMMARY, credential_exposure=sorted(set(creds)), tool_exposure=sorted(set(tools)),
            vuln_ids=[finding.label or finding.id],
        ))
    if sort:
        out.sort(key=lambda p: (p.composite_risk, len(p.hops), len(p.credential_exposure), len(p.tool_exposure)), reverse=True)
    return out


def _server_label_counts(graph) -> tuple[np.ndarray, np.ndarray]:
    """Per node: number of DISTINCT credential / tool labels among a server's EXPOSES_CRED / PROVIDES_TOOL targets
    (``len(sorted(set(labels)))``, api/routes/graph.py:777-778) — the last two components of the ranking key."""
    c = graph.csr
    n = c.n_nodes
    meta, nbr = c.fwd_meta, c.fwd_nbr
    rel = meta & 0x1F
    mask = ((meta & 0x80) == 0) & ((rel == _REL_EXPOSES_CRED) | (rel == _REL_PROVIDES_TOOL)) & (c.node_type[nbr] != ENTITY_CODE_GHOST)
    pos = np.flatnonzero(mask)
    ncu = np.zeros(n, dtype=np.int32)
    ntu = np.zeros(n, dtype=np.int32)
    if pos.size == 0:
        return ncu, ntu
    row = np.searchsorted(c.fwd_off.astype(np.int64), pos, side="right") - 1
    targets = nbr[pos]
    uniq_t, inv = np.unique(targets, return_inverse=True)
    ids = c.node_ids
    label_of: dict[str, int] = {}
    lab = np.asarray([label_of.setdefault(graph.nodes[ids[int(t)]].label, len(label_of)) for t in uniq_t], dtype=np.int64)[inv]
    kind = (rel[pos] == _REL_PROVIDES_TOOL).astype(np.int64)
    key = np.unique(((row.astype(np.int64) * 2 + kind) << 32) | lab)
    grp = key >> 32
    counts = np.bincount(grp, minlength=2 * n)
    return counts[0::2][:n].astype(np.int32), counts[1::2][:n].astype(np.int32)


class RankInputs:
    """What the device ranking needs besides the topology, for one finding list: finding indices, per finding the index of its
    base risk, the dense-rank table of every rounded score, and per server the distinct credential / tool label counts."""

    __slots__ = ("idx", "base_id", "table", "ncu", "ntu")

    def __init__(self, graph, finding_ids):
        self.idx = np.asarray([graph.csr.idx(f) for f in finding_ids], dtype=np.int32)
        base = np.asarray([node_risk_100(graph.nodes[f]) for f in finding_ids], dtype=np.float64)
        base_vals, base_id = np.unique(base, return_inverse=True) if len(base) else (np.zeros(1), np.zeros(0, dtype=np.int64))
        scores = np.empty((len(base_vals), 5, 15), dtype=np.float64)
        for bi, b in enumerate(base_vals.tolist()):
            for nc in range(5):
                for nt in range(15):
                    risk = b
                    risk += min(10.0, nc * 3.0)
                    risk += min(10.0, nt * 0.75)
                    scores[bi, nc, nt] = round(min(100.0, risk), 2)
        levels = np.unique(scores)
        self.base_id = base_id.astype(np.int32)
        self.table = np.searchsorted(levels, scores).astype(np.uint32)
        self.ncu, self.ntu = _server_label_counts(graph)


def rank_inputs(graph) -> RankInputs:
    """The ranking inputs of every finding node, built once per graph (millions of ``node_risk_100`` calls and a label
    de-duplication over every credential / tool edge at L) and dropped with the device graph."""
    if getattr(graph, "_rank_inputs", None) is None:
        graph._rank_inputs = RankInputs(graph, graph.finding_ids())
    return graph._rank_inputs


def ranked_attack_paths(graph, offset: int = 0, limit: int = 100, finding_ids=None) -> tuple[list[AttackPath], int]:
    """One page of the derived attack paths in the reference's order, ranked on the device (nothing but the page is materialised).

    The score itself stays host arithmetic: every distinct (base risk, min(#creds,4), min(#tools,14)) combination is
    evaluated with the reference's float expression and Python ``round`` (api/routes/graph.py:762-771); the device only
    compares the dense ranks of those values."""
    if graph.attack_paths:
        paths = list(graph.attack_paths)
        return paths[offset: offset + limit], len(paths)
    ri = rank_inputs(graph) if finding_ids is None else RankInputs(graph, finding_ids)
    rows, _rank, total = graph.device_graph.rank_exposure_paths(ri.idx, ri.base_id, ri.table, ri.ncu, ri.ntu, offset, limit)
    return materialize_attack_paths(graph, rows, sort=False), total


def exposure_path_rows(graph, finding_ids=None):
    """Device rows for the given findings (default: every finding node, in ``graph.nodes`` order)."""
    if finding_ids is None:
        finding_ids = graph.finding_ids()
    idx = np.asarray([graph.csr.idx(f) for f in finding_ids], dtype=np.int32)
    return graph.device_graph.exposure_paths_many(idx)


def derived_attack_paths(graph) -> list[AttackPath]:
    """Materialised paths win when present (:695-696); otherwise derive them from topology on the device."""
    if graph.attack_paths:
        return list(graph.attack_paths)
    return materialize_attack_paths(graph, exposure_path_rows(graph))
