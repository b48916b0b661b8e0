"""The fix-first graph view: "what should I inspect first?", ranked on the device.

Same object as the reference route ``GET /v1/graph/views/fix-first`` (``api/routes/graph.py:1110-1166``): the derived (or
persisted) attack paths that match an optional ``cve`` / ``package`` / ``agent`` focus (``_path_matches_focus``, ``:448-476``),
in the AttackPath ranking order, the top ``limit`` turned into cards (``_fix_first_card_for_path``, ``:411-445``, with the
helpers ``:255-410``) plus a summary.

Derived paths never exist on the host as a whole: the focus becomes one byte per node (``node_focus``; the bit table is in
``csrc/paths.cuh``), the device ranks only the rows whose hops carry every requested category, and only the returned page is
materialised.  Persisted paths (``graph.attack_paths``) are few and already objects; they are filtered and sorted here with the
same predicate and key.  Pinned card for card by ``tests/test_fix_first.py`` and ``tests/test_gpu_fix_first.py`` on views the
unmodified reference produced (``tests/golden/fix_first/``).
"""

from __future__ import annotations

from typing import Any
from urllib.parse import quote

import numpy as np

from .. import _lib
from .envelope import EdgeIndex, exposure_path_for_attack_path, finding_ids_for_nodes
from .exposure import materialize_attack_paths, rank_inputs
from .schema import ENTITY_CODE, enum_value

MAX_LIMIT = 25
_AGENT_TYPES = frozenset({"agent", "user", "group", "service_account"})
_SERVER_TYPES = frozenset({"server", "container", "cloud_resource"})
_PACKAGE_TYPES = frozenset({"package"})
_FINDING_TYPES = frozenset({"vulnerability", "misconfiguration"})
_AGENT_CODES = np.asarray(sorted(ENTITY_CODE[t] for t in _AGENT_TYPES), dtype=np.uint8)
_PACKAGE_CODE = ENTITY_CODE["package"]
_FINDING_CODES = np.asarray(sorted(ENTITY_CODE[t] for t in _FINDING_TYPES), dtype=np.uint8)
_DANGEROUS_TOOL_WORDS = ("shell", "exec", "run", "command", "subprocess", "filesystem")


def norm(value: str) -> str:
    return value.strip().lower()


def _rank_key(p):
    return (p.composite_risk, len(p.hops), len(p.credential_exposure), len(p.tool_exposure))


# ── card helpers (api/routes/graph.py:255-445) ───────────────────────────────────────────────────────────────────────────────
def node_labels_for_types(nodes: dict[str, Any], hops: list[str], types: frozenset[str]) -> list[str]:
    """``label or id`` of the hops with one of the entity types, in hop order, first of each case-insensitive label only."""
    out, seen = [], set()
    for hop in hops:
        node = nodes.get(hop)
        if node is None or enum_value(node.entity_type) not in types:
            continue
        label = node.label or node.id
        if label.lower() not in seen:
            seen.add(label.lower())
            out.append(label)
    return out


def risk_reasons(path, findings: list[str]) -> list[dict[str, str]]:
    reasons = []
    if path.composite_risk >= 90:
        reasons.append({"kind": "critical_reach", "label": "Critical reach", "detail": "Composite risk is at or above the release-blocking threshold."})
    elif path.composite_risk >= 70:
        reasons.append({"kind": "high_reach", "label": "High reach",
                        "detail": "Composite risk is high enough to prioritize before broad topology review."})
    if path.credential_exposure:
        reasons.append({"kind": "credential_exposure", "label": "Credential exposure",
                        "detail": f"{len(path.credential_exposure)} credential signal(s) sit on this path."})
    if path.tool_exposure:
        dangerous = sum(1 for t in path.tool_exposure if any(w in t.lower() for w in _DANGEROUS_TOOL_WORDS))
        detail = (f"{dangerous} execution/file-capable tool(s) are reachable." if dangerous
                  else f"{len(path.tool_exposure)} tool(s) are reachable from the affected agent/server.")
        reasons.append({"kind": "tool_reach", "label": "Tool reach", "detail": detail})
    if findings:
        reasons.append({"kind": "finding", "label": "Finding in chain",
                        "detail": f"{len(findings)} vulnerability or misconfiguration finding(s) anchor this path."})
    if not reasons:
        reasons.append({"kind": "topology", "label": "Connected exposure",
                        "detail": "The graph found a connected exposure path that should be reviewed before full expansion."})
    return reasons[:4]


def next_actions(path, findings: list[str], agents: list[str]) -> list[dict[str, str]]:
    actions = []
    if findings:
        actions.append({"title": "Validate lead finding", "detail": "Open the first finding and confirm the root cause before expanding the graph.",
                        "href": f"/findings?cve={quote(findings[0])}"})
    if agents:
        actions.append({"title": "Inspect exposed identity", "detail": "Review the agent, user, or service account that can trigger this path.",
                        "href": f"/agents?name={quote(agents[0])}"})
    if path.credential_exposure:
        actions.append({"title": "Contain credentials", "detail": "Rotate, scope, or remove exposed credentials before widening blast-radius analysis.",
                        "href": "/mesh"})
    elif path.tool_exposure:
        actions.append({"title": "Review reachable tools", "detail": "Check whether the tool permissions turn this finding into a real incident path.",
                        "href": "/mesh"})
    actions.append({"title": "Expand topology", "detail": "Open the full lineage graph only when neighboring context is needed.", "href": "/graph"})
    return actions[:4]


def fix_first_card(graph, path, rank: int, edges=None) -> dict[str, Any]:
    """One ranked card; ``edges`` may be the graph's ``EdgeIndex`` (built once per graph) or the plain edge list."""
    nodes = graph.nodes
    findings = finding_ids_for_nodes(nodes, path.hops, path.vuln_ids)
    agents = node_labels_for_types(nodes, path.hops, _AGENT_TYPES)
    on_path = [nodes[h] for h in path.hops if h in nodes]
    title = [findings[0] if findings else "Exposure path"]
    if agents:
        title.append(f"via {agents[0]}")
    if path.tool_exposure:
        title.append(f"with {path.tool_exposure[0]}")
    return {
        "id": f"{path.source}::{path.target}::{'->'.join(path.hops)}",
        "rank": rank,
        "title": " ".join(title),
        "summary": path.summary or "Review this path before opening the full topology graph.",
        "attack_path": path.to_dict(),
        "exposure_path": exposure_path_for_attack_path(path, nodes_by_id=nodes, edges=graph.edges if edges is None else edges, rank=rank,
                                                       scan_id=graph.scan_id),
        "nodes": [n.to_dict() for n in on_path],
        "sequence_labels": [n.label for n in on_path],
        "risk_reasons": risk_reasons(path, findings),
        "next_actions": next_actions(path, findings, agents),
        "affected": {
            "agents": agents,
            "servers": node_labels_for_types(nodes, path.hops, _SERVER_TYPES),
            "packages": node_labels_for_types(nodes, path.hops, _PACKAGE_TYPES),
            "findings": findings,
            "credentials": list(path.credential_exposure),
            "tools": list(path.tool_exposure),
        },
    }


# ── focus ─────────────────────────────────────────────────────────────────────────────────────────────────────────────────────
def path_matches_focus(graph, path, *, cve: str = "", package: str = "", agent: str = "") -> bool:
    """Host form of the focus predicate, for persisted paths (any hop list, hops without a node record allowed)."""
    cve_n, package_n, agent_n = norm(cve), norm(package), norm(agent)
    if not (cve_n or package_n or agent_n):
        return True
    nodes = graph.nodes
    if cve_n and cve_n not in {norm(nodes[h].label) for h in path.hops if h in nodes} \
            and cve_n not in {norm(v) for v in finding_ids_for_nodes(nodes, path.hops, path.vuln_ids)}:
        return False
    if package_n and package_n not in {norm(v) for v in node_labels_for_types(nodes, path.hops, _PACKAGE_TYPES)}:
        return False
    if agent_n and agent_n not in {norm(v) for v in node_labels_for_types(nodes, path.hops, _AGENT_TYPES)}:
        return False
    return True


class FocusIndex:
    """Node indices by ``norm(label)`` and by ``norm(label or id)``: a focused request then costs O(matching nodes)."""

    __slots__ = ("by_label", "by_label_or_id")

    def __init__(self, graph):
        idx = graph.csr.idx
        self.by_label: dict[str, list[int]] = {}
        self.by_label_or_id: dict[str, list[int]] = {}
        for nid, node in graph.nodes.items():
            i = idx(nid)
            self.by_label.setdefault(norm(node.label), []).append(i)
            self.by_label_or_id.setdefault(norm(node.label or node.id), []).append(i)


def focus_index(graph) -> FocusIndex:
    """Built on the first focused request and kept with the device graph (an unfocused view never pays for it)."""
    if getattr(graph, "_focus_index", None) is None:
        graph._focus_index = FocusIndex(graph)
    return graph._focus_index


def node_focus(graph, *, cve: str = "", package: str = "", agent: str = "") -> tuple[np.ndarray | None, int]:
    """(``_lib.FOCUS_*`` bits per node, categories every matching row needs); ``(None, 0)`` without a focus."""
    cve_n, package_n, agent_n = norm(cve), norm(package), norm(agent)
    if not (cve_n or package_n or agent_n):
        return None, 0
    c = graph.csr
    ix = focus_index(graph)
    focus = np.zeros(c.n_nodes, dtype=np.uint8)
    need = 0

    def hits(table: dict[str, list[int]], key: str, codes=None) -> np.ndarray:
        i = np.asarray(table.get(key, ()), dtype=np.int64)
        return i if codes is None else i[np.isin(c.node_type[i], codes)]

    if cve_n:
        need |= _lib.FOCUS_CVE
        focus[hits(ix.by_label, cve_n)] |= _lib.FOCUS_CVE                                  # any hop's bare label
        focus[hits(ix.by_label_or_id, cve_n, _FINDING_CODES)] |= _lib.FOCUS_CVE            # a finding-typed hop's label or id
        focus[hits(ix.by_label_or_id, cve_n)] |= _lib.FOCUS_CVE_FINDING                    # the path's vuln_ids entry
    if package_n:
        need |= _lib.FOCUS_PACKAGE
        focus[hits(ix.by_label_or_id, package_n, [_PACKAGE_CODE])] |= _lib.FOCUS_PACKAGE
    if agent_n:
        need |= _lib.FOCUS_AGENT
        focus[hits(ix.by_label_or_id, agent_n, _AGENT_CODES)] |= _lib.FOCUS_AGENT
    return focus, need


class CsrEdgeIndex(EdgeIndex):
    """``EdgeIndex.first_edge`` answered from the graph's CSR: the forward row of ``a`` holds every edge ``a -> b`` and the reversed
    copy of every bidirectional ``b -> a``, each with its position in ``graph.edges``, so the first edge of the pair is the smallest
    position among the row's entries for ``b``.  Nothing is built per graph: a card page needs a handful of pairs, while an
    ``EdgeIndex`` would turn every edge of a columnar or snapshot graph into a record."""

    __slots__ = ("_graph",)

    def __init__(self, graph):
        self._graph = graph

    def first_edge(self, source, target):
        c = self._graph.csr
        a, b = c.idx(source), c.idx(target)
        if a < 0 or b < 0:
            return None
        lo, hi = int(c.fwd_off[a]), int(c.fwd_off[a + 1])
        eids = c.fwd_eid[lo:hi][c.fwd_nbr[lo:hi] == b]
        return self._graph.edges[int(eids.min()) >> 1] if eids.size else None


def edge_lookup(graph) -> EdgeIndex:
    if getattr(graph, "_edge_lookup", None) is None:
        graph._edge_lookup = CsrEdgeIndex(graph)
    return graph._edge_lookup


# ── the view ──────────────────────────────────────────────────────────────────────────────────────────────────────────────────
def ranked_focus_page(graph, *, cve: str = "", package: str = "", agent: str = "", offset: int = 0, limit: int = 8):
    """(page of AttackPaths in ranking order, total paths, matched paths)."""
    if graph.attack_paths:
        available = list(graph.attack_paths)
        ranked = sorted((p for p in available if path_matches_focus(graph, p, cve=cve, package=package, agent=agent)), key=_rank_key, reverse=True)
        return ranked[offset: offset + limit], len(available), len(ranked)
    if not graph.nodes:
        return [], 0, 0
    ri = rank_inputs(graph)
    if ri.idx.size == 0:
        return [], 0, 0
    focus, need = node_focus(graph, cve=cve, package=package, agent=agent)
    rows, _rank, total, matched = graph.device_graph.rank_exposure_paths_focused(ri.idx, ri.base_id, ri.table, ri.ncu, ri.ntu, focus, need, offset, limit)
    return materialize_attack_paths(graph, rows, sort=False), total, matched


def fix_first_view(graph, *, cve: str = "", package: str = "", agent: str = "", limit: int = 8) -> dict[str, Any]:
    """The fix-first view model of one graph (the reference route's response body)."""
    if not 1 <= int(limit) <= MAX_LIMIT:
        raise ValueError(f"limit must be between 1 and {MAX_LIMIT}, got {limit}")
    page, total, matched = ranked_focus_page(graph, cve=cve, package=package, agent=agent, limit=int(limit))
    edges = edge_lookup(graph) if page else None
    cards = [fix_first_card(graph, p, i + 1, edges) for i, p in enumerate(page)]
    covered = {f for card in cards for f in card["affected"]["findings"]}
    return {
        "scan_id": graph.scan_id,
        "tenant_id": graph.tenant_id,
        "created_at": graph.created_at,
        "cards": cards,
        "summary": {
            "total_paths": total,
            "matched_paths": matched,
            "returned_paths": len(cards),
            "highest_risk": cards[0]["attack_path"]["composite_risk"] if cards else 0.0,
            "covered_findings": len(covered),
            "node_count": len(graph.nodes),
            "edge_count": len(graph.edges),
        },
        "focus": {"cve": cve, "package": package, "agent": agent},
    }
