"""OCSF events of the graph's findings, with their blast-radius context computed on the device.

Restates the reference's SIEM export, ``UnifiedGraph.to_ocsf_events`` (``/root/reference/src/agent_bom/graph/container.py:628-654``)
and ``UnifiedNode.to_ocsf_event`` (``graph/node.py:179-219``), for every node-record family the engine holds: the light
records of ``graph/model.py``, columnar graphs (read from their columns, no record is made), snapshot records (their JSON
columns are read once per batch) and adopted reference records.

The reference builds each event's ``graph_context`` with one ``sources_of`` and one depth-4 ``impact_of`` per finding.  Here a
batch of findings is one ``DeviceGraph.finding_context`` call: the impact walk's count and type histogram plus the typed
in-neighbour lists come back, the walk's node slices stay on the device, and labels are read by node index from a label column.
"""

from __future__ import annotations

import time
from typing import Any, Iterator

import numpy as np

from .. import _lib
from . import csr as csrmod
from .schema import FINDING_CODES, enum_value

#: OCSF (category_uid, class_uid) per entity kind: inventory -> Discovery / Device Inventory Info, identity -> IAM / Account
#: Change, vulnerability -> Findings / Vulnerability Finding, misconfiguration -> Findings / Compliance Finding; the
#: organisational provider / environment kinds and anything unknown have none.
_INVENTORY, _IDENTITY = (5, 4001), (3, 3001)
OCSF_CLASS: dict[str, tuple[int, int]] = {
    **{k: _INVENTORY for k in ("agent", "server", "package", "tool", "model", "dataset", "container", "cloud_resource", "credential", "fleet", "cluster")},
    **{k: _IDENTITY for k in ("org", "account", "user", "group", "role", "policy", "service_account", "service_principal", "federated_identity")},
    "vulnerability": (2, 2001),
    "misconfiguration": (2, 2003),
    "provider": (0, 0),
    "environment": (0, 0),
}
#: OCSF 1.1 severity_id of a severity string (lower-cased) and the display name of each id
SEVERITY_ID = {"critical": 5, "high": 4, "medium": 3, "low": 2, "info": 1, "informational": 1, "none": 0, "unknown": 0}
SEVERITY_NAME = {5: "Critical", 4: "High", 3: "Medium", 2: "Low", 1: "Informational", 0: "Unknown"}
FINDING_KINDS = frozenset({"vulnerability", "misconfiguration"})
OCSF_SCHEMA_VERSION = "1.1.0"

_SCALARS = (str, int, float, bool)
_CONTEXT_KEYS = ((_lib.CTX_AGENT, "affected_agents"), (_lib.CTX_SERVER, "affected_servers"), (_lib.CTX_PACKAGE, "affected_packages"),
                 (_lib.CTX_CREDENTIAL, "exposed_credentials"))


def _event(node_id: str, kind: str, label: str, severity: str, attributes: dict, tags: list, product_version: str, *, category_uid: int = 0,
           class_uid: int = 0, type_uid: int = 0, severity_id: int = 0) -> dict[str, Any]:
    """One event.  Stored classification values win when non-zero; otherwise they are derived from the entity kind and the
    severity string, as the reference's record constructor does."""
    cat, cls = OCSF_CLASS.get(kind, (0, 0))
    category_uid = category_uid or cat
    class_uid = class_uid or cls
    type_uid = type_uid or class_uid * 100 + 1
    if not severity_id and severity:
        severity_id = SEVERITY_ID.get(severity.lower(), 0)
    event: dict[str, Any] = {
        "class_uid": class_uid,
        "category_uid": category_uid,
        "type_uid": type_uid,
        "activity_id": 1,
        "activity_name": "Create",
        "severity_id": severity_id,
        "severity": SEVERITY_NAME.get(severity_id, "Unknown"),
        "status_id": 1,
        "status": "New",
        "time": int(time.time() * 1000),
        "message": f"{kind}:{label}",
        "metadata": {"product": {"name": "agent-bom", "vendor_name": "msaad00", "version": product_version}, "version": OCSF_SCHEMA_VERSION},
        "resources": [{"type": kind, "name": label, "uid": node_id, "data": {k: v for k, v in attributes.items() if isinstance(v, _SCALARS)}}],
    }
    if class_uid == 2001:
        event["finding_info"] = {"title": label, "uid": node_id, "types": [kind]}
    if tags:
        event["compliance"] = {"standards": tags}
    return event


def ocsf_event(node, product_version: str = "0.0.0") -> dict[str, Any]:
    """``UnifiedNode.to_ocsf_event`` for any node record (light, snapshot, adopted reference record)."""
    return _event(node.id, enum_value(node.entity_type), node.label, getattr(node, "severity", "") or "", getattr(node, "attributes", None) or {},
                  getattr(node, "compliance_tags", None) or [], product_version, category_uid=getattr(node, "category_uid", 0) or 0,
                  class_uid=getattr(node, "class_uid", 0) or 0, type_uid=getattr(node, "type_uid", 0) or 0, severity_id=getattr(node, "severity_id", 0) or 0)


def _columns(graph):
    """The column store of a columnar graph whose records have not been materialised, else None."""
    from .columnar import _NodeView

    return graph._cols if isinstance(graph.nodes, _NodeView) else None


def _column_event(cols, i: int, product_version: str) -> dict[str, Any]:
    return _event(cols.ids[i], _kind(cols.types[i]), cols.labels[i], cols.severity[i], cols.attrs.get(i) or {}, [], product_version)


def _kind(code: int) -> str:
    from .schema import ENTITY_VALUES

    return ENTITY_VALUES[code] if code < len(ENTITY_VALUES) else "other"


def label_column(graph) -> list[str]:
    """``node.label`` of every real node by node index (columnar graphs: the label column itself)."""
    cols = _columns(graph)
    if cols is not None:
        return cols.labels
    nodes = graph.nodes
    return [nodes[nid].label for nid in graph.csr.node_ids[: graph.csr.n_real]]


def finding_indices(graph) -> np.ndarray:
    """Node indices of the findings, in ``nodes`` insertion order."""
    c = graph.csr
    return np.flatnonzero(np.isin(c.node_type[: c.n_real], FINDING_CODES)).astype(np.int32)


def _blast_by_type(graph, ctx, q: int, idx: int, has_other: bool) -> dict[str, int]:
    by_type = ctx.hist_dict(q)
    # entity kinds outside the enum are not in the device histogram: tally them from the walk's slice, as impact_of does
    if has_other and sum(by_type.values()) < int(ctx.count[q]):
        return graph.impact_of(graph.csr.node_ids[idx])["affected_by_type"]
    return by_type


def iter_ocsf_events(graph, product_version: str = "0.0.0", *, enrich_neighbors: bool = True, batch_size: int = 65536, offset: int = 0,
                     limit: int | None = None) -> Iterator[dict[str, Any]]:
    """OCSF events of the graph's findings in ``nodes`` order — the page [offset, offset+limit) of them (``limit=None``: to the
    end); one device call per ``batch_size`` findings of the page when enriching.  Without enrichment nothing is uploaded and no
    device is needed."""
    from .snapshot import SnapshotGraph

    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    offset = max(0, int(offset))
    stop = None if limit is None else offset + max(0, int(limit))
    cols = _columns(graph)
    if not enrich_neighbors:
        if cols is not None:
            page = [i for i, code in enumerate(cols.types) if _kind(code) in FINDING_KINDS][offset:stop]
            for i in page:
                yield _column_event(cols, i, product_version)
            return
        page = [n for n in graph.nodes.values() if enum_value(n.entity_type) in FINDING_KINDS][offset:stop]
        for a in range(0, len(page), batch_size):
            batch = page[a: a + batch_size]
            if isinstance(graph, SnapshotGraph):
                graph.hydrate_nodes([n.id for n in batch])
            for n in batch:
                yield ocsf_event(n, product_version)
        return
    findings = finding_indices(graph)[offset:stop]
    if not findings.size:
        return
    labels = label_column(graph)
    ids = graph.csr.node_ids
    has_other = bool((graph.csr.node_type == csrmod.ENTITY_CODE_OTHER).any())
    dg = graph.device_graph
    for a in range(0, int(findings.size), batch_size):
        idx = findings[a: a + batch_size]
        ctx = dg.finding_context(idx)
        if cols is None and isinstance(graph, SnapshotGraph):
            graph.hydrate_nodes([ids[i] for i in idx.tolist()])
        for q, i in enumerate(idx.tolist()):
            event = _column_event(cols, i, product_version) if cols is not None else ocsf_event(graph.nodes[ids[i]], product_version)
            context = {key: [labels[s] for s in ctx.sources(q, b).tolist()] for b, key in _CONTEXT_KEYS}
            context["blast_radius"] = int(ctx.count[q])
            context["blast_by_type"] = _blast_by_type(graph, ctx, q, i, has_other)
            event["graph_context"] = context
            yield event
