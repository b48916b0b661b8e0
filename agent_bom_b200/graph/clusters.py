"""Semantic graph clusters (``GET /v1/graph/clusters``) with the roll-ups computed on the device.

Drop-in for the reference's ``build_semantic_clusters`` / ``semantic_cluster_stats``
(``/root/reference/src/agent_bom/graph/semantic_clusters.py:81-135``) and the body of its route
(``api/routes/graph.py:1485-1528``).  The reference scans every edge once per cluster; here the host interns each node's
cluster keys once per graph (``ClusterTable``: the key rules restated below, in the reference's first-appearance order) and
the device builds every cluster's member count, risk roll-up, members in id order and relationship counts in one pass over
the graph (``csrc/clusters.cuh``).  Only the clusters a caller returns cross PCIe and become Python objects.
"""

from __future__ import annotations

import re
import threading
from collections import Counter
from dataclasses import dataclass, field
from typing import Any, Iterable

import numpy as np

from .schema import ENTITY_VALUES, REL_CODE_OTHER, RELATIONSHIP_VALUES, SEVERITY_RANK, enum_value

SEMANTIC_CLUSTER_KINDS = (
    "package_family",
    "cve_family",
    "agent_fleet",
    "server_fleet",
    "credential_family",
    "tool_capability",
    "source_environment",
)
#: severity levels in histogram order (the keys of ``risk_summary``)
LEVELS = ("critical", "high", "medium", "low", "none")
_RISK_SEVERITY = ((90.0, 0), (70.0, 1), (40.0, 2), (1.0, 3))
_CVE = re.compile(r"CVE-(\d{4})-", flags=re.IGNORECASE)
_CWE = re.compile(r"CWE-(\d+)", flags=re.IGNORECASE)
_SLUG = re.compile(r"[^a-z0-9]+")
_DIMENSIONS = ("ecosystem", "cloud_provider", "agent_type", "surface", "environment")
_EMPTY_DIMS: dict[str, str] = {}
_build_lock = threading.Lock()


@dataclass(slots=True)
class SemanticClusterExpansion:
    mode: str = "members"
    member_ids: list[str] = field(default_factory=list)
    collapse_id: str = ""
    reversible: bool = True

    def to_dict(self) -> dict[str, Any]:
        return {"mode": self.mode, "member_ids": self.member_ids, "collapse_id": self.collapse_id, "reversible": self.reversible}


@dataclass(slots=True)
class SemanticCluster:
    id: str
    kind: str
    label: str
    layer: str
    entity_types: list[str]
    count: int
    member_ids: list[str]
    max_risk: float
    severity: str
    risk_summary: dict[str, int]
    relationship_counts: dict[str, int]
    expansion: SemanticClusterExpansion

    def to_dict(self) -> dict[str, Any]:
        return {
            "id": self.id, "kind": self.kind, "label": self.label, "layer": self.layer, "entity_types": self.entity_types, "count": self.count,
            "member_ids": self.member_ids, "max_risk": self.max_risk, "severity": self.severity, "risk_summary": self.risk_summary,
            "relationship_counts": self.relationship_counts, "expansion": self.expansion.to_dict(),
        }


# ── the reference's key rules (semantic_clusters.py:138-232), over plain fields ──
def _string_attr(attrs, *keys: str) -> str:
    for key in keys:
        value = attrs.get(key)
        if isinstance(value, str) and value.strip():
            return value.strip()
    return ""


def _slug(value: str) -> str:
    return _SLUG.sub("-", value.lower()).strip("-") or "unknown"


def _package_name(nid: str, label: str, attrs) -> str:
    raw = _string_attr(attrs, "name", "package_name", "package") or label or nid
    if "@" in raw and not raw.startswith("@"):
        raw = raw.split("@", 1)[0]
    return raw.replace("pkg:", "").strip() or "unknown"


def _cve_family(nid: str, label: str, attrs) -> str:
    raw = " ".join([nid, label, *(str(value) for value in attrs.values() if isinstance(value, str))])
    match = _CVE.search(raw)
    if match:
        return f"CVE {match.group(1)}"
    cwe = _CWE.search(raw)
    if cwe:
        return f"CWE {cwe.group(1)}"
    return "unclassified findings"


def _credential_family(nid: str, label: str, attrs) -> str:
    provider = _string_attr(attrs, "provider", "cloud_provider", "service")
    if provider:
        return provider
    text = (label or nid).upper()
    for token in ("AWS", "AZURE", "GCP", "OPENAI", "ANTHROPIC", "GITHUB", "SNOWFLAKE"):
        if token in text:
            return token
    return "generic"


def _tool_capability(nid: str, label: str) -> str:
    text = (label or nid).lower()
    if any(token in text for token in ("shell", "exec", "command")):
        return "execution"
    if any(token in text for token in ("read", "file", "fs")):
        return "file access"
    if any(token in text for token in ("http", "fetch", "web")):
        return "network access"
    return "general"


def cluster_keys(entity_type: str, nid: str, label: str, attrs, dims, data_sources) -> list[tuple[str, str, str, str]]:
    """``_cluster_keys_for_node`` (semantic_clusters.py:138-171): ``dims`` is a mapping of the ``NodeDimensions`` fields."""
    get = dims.get
    keys: list[tuple[str, str, str, str]] = []
    environment = get("environment", "") or _string_attr(attrs, "environment", "env", "workspace", "account")
    source = data_sources[0] if data_sources else _string_attr(attrs, "source", "provider")
    if environment or source:
        env_key = environment or source
        source_part = f" / {source}" if source and source != env_key else ""
        keys.append(("source_environment", "infra", f"{env_key}:{source}", f"{env_key}{source_part}"))
    if entity_type == "package":
        ecosystem = get("ecosystem", "") or _string_attr(attrs, "ecosystem", "package_ecosystem") or "unknown"
        package_name = _package_name(nid, label, attrs)
        keys.append(("package_family", "package", f"{ecosystem}:{package_name}", f"{ecosystem} / {package_name}"))
    elif entity_type == "vulnerability":
        family = _cve_family(nid, label, attrs)
        keys.append(("cve_family", "finding", family, family))
    elif entity_type == "agent":
        fleet = get("agent_type", "") or environment or source or _string_attr(attrs, "fleet", "agent_type", "kind") or "agents"
        keys.append(("agent_fleet", "orchestration", fleet, f"{fleet} agents"))
    elif entity_type == "server":
        fleet = get("surface", "") or environment or source or _string_attr(attrs, "fleet", "server_type", "kind") or "servers"
        keys.append(("server_fleet", "mcp_server", fleet, f"{fleet} servers"))
    elif entity_type == "credential":
        family = _credential_family(nid, label, attrs)
        keys.append(("credential_family", "identity", family, f"{family} credentials"))
    elif entity_type == "tool":
        capability = _string_attr(attrs, "capability", "category", "tool_type") or _tool_capability(nid, label)
        keys.append(("tool_capability", "tool", capability, f"{capability} tools"))
    return keys


def cluster_risk(risk_score, severity) -> float:
    """``_node_risk_100`` of the cluster rule (semantic_clusters.py:255-261): clamped at 0 and rounded to 3 places."""
    risk = float(risk_score or 0.0)
    if risk <= 10.0:
        risk *= 10.0
    if risk <= 0 and severity:
        risk = float(SEVERITY_RANK.get(severity.lower(), 0) * 20)
    return round(min(100.0, max(0.0, risk)), 3)


def cluster_level(severity, risk100: float) -> int:
    """Index into ``LEVELS`` of ``_node_severity`` (:243-252): a named severity wins, else the ROUNDED risk's threshold."""
    sev = (severity or "").lower()
    if sev in ("critical", "high", "medium", "low"):
        return LEVELS.index(sev)
    for threshold, level in _RISK_SEVERITY:
        if risk100 >= threshold:
            return level
    return 4


def _dims_of(node):
    """``node.dimensions`` as a mapping: reference records carry a ``NodeDimensions``, snapshot rows a dict, ours none."""
    dims = getattr(node, "dimensions", None)
    if dims is None:
        return _EMPTY_DIMS
    if isinstance(dims, dict):
        return dims
    return {f: getattr(dims, f, "") for f in _DIMENSIONS}


class ClusterTable:
    """Per graph: every node's cluster codes (int32 [n, 2], -1 = none), its severity level, rounded risk and entity-type index,
    and per cluster (in first-appearance order) its kind, layer, key and label.  ``other_rel`` holds the relationship counts of
    edges whose relationship is outside the enum, per cluster (the device skips them).  After ``ensure_device`` the device's
    per-cluster summaries and the clusters' full ranking order are attached."""

    def __init__(self, graph):
        csr = graph.csr
        n, n_real = csr.n_nodes, csr.n_real
        self.codes = np.full((n, 2), -1, dtype=np.int32)
        self.level = np.full(n, 4, dtype=np.uint8)
        self.risk = np.zeros(n, dtype=np.float64)
        self.etype = np.zeros(n, dtype=np.uint8)
        self.kind: list[str] = []
        self.layer: list[str] = []
        self.key: list[str] = []
        self.label: list[str] = []
        self.type_names: list[str] = []
        self._intern: dict[tuple[str, str, str, str], int] = {}
        self._types: dict[str, int] = {}
        self._risk_memo: dict[tuple, tuple[float, int]] = {}
        cols = getattr(graph, "_cols", None)
        if cols is not None and not isinstance(graph.nodes, dict):
            self._from_columns(cols, n_real)
        else:
            if hasattr(graph, "hydrate_nodes"):
                graph.hydrate_nodes(list(graph.nodes))
            self._from_records(graph.nodes.values())
        self._intern = self._types = self._risk_memo = None
        self.other_rel = self._other_relationships(graph)
        self.summary: dict[str, np.ndarray] | None = None
        self.order: np.ndarray | None = None
        self._dg = None

    @property
    def n_clusters(self) -> int:
        return len(self.kind)

    def _node(self, i: int, et: str, nid: str, label: str, attrs, dims, data_sources, risk_score, severity) -> None:
        for j, k in enumerate(cluster_keys(et, nid, label, attrs, dims, data_sources)):
            c = self._intern.get(k)
            if c is None:
                c = self._intern[k] = len(self.kind)
                self.kind.append(k[0]); self.layer.append(k[1]); self.key.append(k[2]); self.label.append(k[3])
            self.codes[i, j] = c
        t = self._types.get(et)
        if t is None:
            if len(self.type_names) == 64:
                raise ValueError("semantic clusters support at most 64 distinct entity types per graph")
            t = self._types[et] = len(self.type_names)
            self.type_names.append(et)
        self.etype[i] = t
        memo_key = (risk_score, severity)
        rl = self._risk_memo.get(memo_key)
        if rl is None:
            r = cluster_risk(risk_score, severity)
            rl = self._risk_memo[memo_key] = (r, cluster_level(severity, r))
        self.risk[i], self.level[i] = rl

    def _from_records(self, nodes) -> None:
        for i, node in enumerate(nodes):
            self._node(i, enum_value(node.entity_type), node.id, node.label, node.attributes or {}, _dims_of(node), node.data_sources,
                       node.risk_score, node.severity)

    def _from_columns(self, cols, n_real: int) -> None:
        """Columnar graphs: read the columns, never a node record (no dimensions; the first data source is always present)."""
        attrs, more = cols.attrs, cols.more_sources
        names = list(ENTITY_VALUES) + ["other"] * (256 - len(ENTITY_VALUES))
        for i in range(n_real):
            src = cols.sources[i]
            ds = [src, *more[i]] if i in more else (src,)
            self._node(i, names[cols.types[i]], cols.ids[i], cols.labels[i], attrs.get(i) or {}, _EMPTY_DIMS, ds, cols.risk[i], cols.severity[i])

    def _other_relationships(self, graph) -> dict[int, Counter]:
        csr = graph.csr
        out: dict[int, Counter] = {}
        for e in np.flatnonzero(csr.rel == REL_CODE_OTHER).tolist():
            name = enum_value(graph.edges[e].relationship)
            for c in set(self.codes[csr.src[e]].tolist()) | set(self.codes[csr.dst[e]].tolist()):
                if c >= 0:
                    out.setdefault(c, Counter())[name] += 1
        return out

    def ensure_device(self, graph) -> None:
        """Build the device tables and the ranking order once per device graph."""
        dg = graph.device_graph
        if self._dg is dg:
            return
        s = self.summary = dg.build_clusters(self.n_clusters, self.codes, self.level, self.risk, self.etype)
        # the reference's final sort, (-max_risk, -count, kind, label), stable over first-appearance order
        label_rank = {lab: r for r, lab in enumerate(sorted(set(self.label)))}
        kind_rank = {k: r for r, k in enumerate(sorted(SEMANTIC_CLUSTER_KINDS))}
        lr = np.fromiter((label_rank[lab] for lab in self.label), dtype=np.int64, count=self.n_clusters)
        kr = np.fromiter((kind_rank[k] for k in self.kind), dtype=np.int64, count=self.n_clusters)
        self.order = np.lexsort((np.arange(self.n_clusters), lr, kr, -s["count"], -s["max_risk"])).astype(np.int32)
        self._dg = dg

    def materialise(self, graph, sel: np.ndarray) -> list[SemanticCluster]:
        """``SemanticCluster`` objects of the selected clusters, in selection order; only their members and pairs are copied back."""
        s = self.summary
        sel = np.asarray(sel, dtype=np.int32)
        device_nnz = s["rel_nnz"][sel]
        counts = s["count"][sel]
        members, rel, rel_cnt = graph.device_graph.fetch_clusters(sel, int(counts.sum()), int(device_nnz.sum()))
        ids = graph.csr.node_ids
        out: list[SemanticCluster] = []
        mo = ro = 0
        for i, c in enumerate(sel.tolist()):
            cnt, nnz = int(counts[i]), int(device_nnz[i])
            member_ids = [ids[u] for u in members[mo: mo + cnt].tolist()]
            rels = {RELATIONSHIP_VALUES[r]: v for r, v in zip(rel[ro: ro + nnz].tolist(), rel_cnt[ro: ro + nnz].tolist())}
            mo += cnt
            ro += nnz
            rels.update(self.other_rel.get(c, {}))
            hist = s["hist"][c].tolist()
            mask = int(s["type_mask"][c])
            cluster_id = f"cluster:{self.kind[c]}:{_slug(self.key[c])}"
            out.append(SemanticCluster(
                id=cluster_id, kind=self.kind[c], label=self.label[c], layer=self.layer[c],
                entity_types=sorted(self.type_names[t] for t in range(len(self.type_names)) if mask >> t & 1),
                count=cnt, member_ids=member_ids, max_risk=float(s["max_risk"][c]),
                severity=next((LEVELS[k] for k in range(4) if hist[k]), "none"),
                risk_summary=dict(zip(LEVELS, hist)), relationship_counts=dict(sorted(rels.items())),
                expansion=SemanticClusterExpansion(member_ids=member_ids, collapse_id=cluster_id),
            ))
        return out


def cluster_table(graph) -> ClusterTable:
    """The graph's key table, built once (under a lock: store calls arrive on worker threads) and dropped with the device graph
    or when a node merge changes what the keys read."""
    table = getattr(graph, "_clusters", None)
    if table is None:
        with _build_lock:
            table = getattr(graph, "_clusters", None)
            if table is None:
                table = graph._clusters = ClusterTable(graph)
    return table


def _ranked(graph, min_members: int) -> tuple[ClusterTable | None, np.ndarray]:
    if not graph.nodes:
        return None, np.zeros(0, np.int32)
    table = cluster_table(graph)
    with _build_lock:
        table.ensure_device(graph)
    order = table.order
    return table, order[table.summary["count"][order] >= min_members]


def semantic_clusters(graph, *, min_members: int = 2) -> list[SemanticCluster]:
    """``build_semantic_clusters(graph.nodes.values(), graph.edges, min_members=...)``: every cluster, in the reference's order."""
    table, sel = _ranked(graph, int(min_members))
    return [] if table is None else table.materialise(graph, sel)


def semantic_cluster_stats(clusters: Iterable[SemanticCluster]) -> dict[str, int]:
    """Reference ``semantic_cluster_stats`` (semantic_clusters.py:127-135)."""
    cluster_list = list(clusters)
    member_ids = {member_id for cluster in cluster_list for member_id in cluster.member_ids}
    by_kind = Counter(cluster.kind for cluster in cluster_list)
    return {"cluster_count": len(cluster_list), "member_count": len(member_ids), **{f"{kind}_count": by_kind.get(kind, 0) for kind in SEMANTIC_CLUSTER_KINDS}}


def parse_kinds(kinds) -> set[str]:
    """The route's ``kinds`` parameter (comma-separated, or an iterable of names); ``ValueError`` with the route's 400 text."""
    if kinds:
        parts = kinds.split(",") if isinstance(kinds, str) else list(kinds)
        selected = {kind.strip() for kind in parts if kind.strip()}
    else:
        selected = set(SEMANTIC_CLUSTER_KINDS)
    unknown = selected - set(SEMANTIC_CLUSTER_KINDS)
    if unknown:
        raise ValueError(f"Unknown semantic cluster kind(s): {', '.join(sorted(unknown))}")
    return selected


def semantic_clusters_view(graph, *, kinds=None, min_members: int = 2, limit: int = 250) -> dict[str, Any]:
    """The body of ``GET /v1/graph/clusters`` (reference api/routes/graph.py:1485-1528) for a loaded graph.

    Raises ``ValueError`` for unknown kinds (the route's 400 detail) and for ``min_members`` outside 1-100 or ``limit`` outside
    1-1000 (the route's query bounds).  Only the returned clusters are copied back from the device and materialised."""
    if not 1 <= int(min_members) <= 100:
        raise ValueError("min_members must be in [1, 100]")
    if not 1 <= int(limit) <= 1000:
        raise ValueError("limit must be in [1, 1000]")
    selected = parse_kinds(kinds)
    table, order = _ranked(graph, int(min_members))
    clusters: list[SemanticCluster] = []
    if table is not None and len(order):
        kind_ok = np.asarray([k in selected for k in SEMANTIC_CLUSTER_KINDS])
        kind_idx = {k: i for i, k in enumerate(SEMANTIC_CLUSTER_KINDS)}
        if not kind_ok.all():
            ck = np.fromiter((kind_idx[k] for k in table.kind), dtype=np.int64, count=table.n_clusters)
            order = order[kind_ok[ck[order]]]
        clusters = table.materialise(graph, order[: int(limit)])
    return {
        "scan_id": graph.scan_id,
        "tenant_id": graph.tenant_id,
        "created_at": graph.created_at,
        "clusters": [cluster.to_dict() for cluster in clusters],
        "stats": semantic_cluster_stats(clusters),
        "available_kinds": list(SEMANTIC_CLUSTER_KINDS),
    }
