"""Fixture of the OCSF export goldens (``oracle/make_ocsf_golden.py`` → ``tests/golden/ocsf/events.json.gz``): graphs replayed from
the reference's node records and edge stream, the builder-identity reports and SQLite snapshots they came from, and the
reference's ``to_ocsf_events`` on each of them (without ``time``)."""

from __future__ import annotations

import copy
import gzip
import json
from functools import lru_cache
from pathlib import Path
from types import SimpleNamespace

GOLDEN = Path(__file__).resolve().parent / "golden"
SEP = "|#|"


@lru_cache(maxsize=None)
def doc() -> dict:
    return json.loads(gzip.decompress((GOLDEN / "ocsf" / "events.json.gz").read_bytes()))


def versions() -> list[str]:
    return doc()["versions"]


def graph_cases() -> list[dict]:
    """Cases that carry their graph (the snapshots and the builder reports are replayed from their sources instead)."""
    return [c for c in doc()["cases"] if "nodes" in c]


def snapshot_cases() -> list[dict]:
    return [c for c in doc()["cases"] if "snapshot_scan" in c]


def builder_cases() -> list[dict]:
    return [c for c in doc()["cases"] if "builder" in c]


def expand(stored: dict, version: str, enriched: bool) -> list[dict]:
    """The reference's events of one run, rebuilt from their stored form: the un-enriched events of the first product version
    and each event's ``graph_context`` (the generator checks this equals every run of the reference)."""
    out = []
    for ev, ctx in zip(stored["plain"], stored["graph_context"]):
        ev = copy.deepcopy(ev)
        ev["metadata"]["product"]["version"] = version
        if enriched:
            ev["graph_context"] = copy.deepcopy(ctx)
        out.append(ev)
    return out


def events(case: dict, version: str, enriched: bool) -> list[dict]:
    return expand(case["events"], version, enriched)


class OcsfRecordNode:
    """A reference node record replayed with the fields its OCSF event reads (classification, severity id, tags, attributes).
    Non-finding nodes are stored with id, entity type and label only; the rest take the record defaults."""

    __slots__ = ("id", "entity_type", "label", "severity", "risk_score", "attributes", "category_uid", "class_uid", "type_uid", "severity_id",
                 "compliance_tags", "data_sources", "_dict")

    def __init__(self, rec: dict):
        self.id, self.entity_type, self.label = rec["id"], rec["entity_type"], rec["label"]
        self.severity, self.risk_score, self.attributes = rec.get("severity", ""), rec.get("risk_score", 0.0), rec.get("attributes", {})
        self.category_uid, self.class_uid = rec.get("category_uid", 0), rec.get("class_uid", 0)
        self.type_uid, self.severity_id = rec.get("type_uid", 0), rec.get("severity_id", 0)
        self.compliance_tags, self.data_sources = rec.get("compliance_tags", []), rec.get("data_sources", [])
        self._dict = rec

    def to_dict(self) -> dict:
        return copy.deepcopy(self._dict)


def reference_graph(case: dict):
    """A reference-shaped graph object for ``UnifiedGraph.from_graph``."""
    from agent_bom_b200.graph import UnifiedEdge

    nodes = {n["id"]: OcsfRecordNode(n) for n in case["nodes"]}
    edges = [UnifiedEdge(**e) for e in case["edges"]]
    return SimpleNamespace(nodes=nodes, edges=edges, attack_paths=[], interaction_risks=[], scan_id=case["scan_id"], tenant_id=case["tenant_id"],
                           created_at=case["created_at"])


def adopted(case: dict, device: int = 0):
    from agent_bom_b200.graph import UnifiedGraph

    return UnifiedGraph.from_graph(reference_graph(case), device=device)


@lru_cache(maxsize=None)
def _identity_docs() -> dict:
    docs = json.loads(gzip.decompress((GOLDEN / "identity" / "builder_identity.json.gz").read_bytes()))
    return {d["label"]: d for d in docs}


def built(case: dict, columnar: bool, device: int = 0):
    """The light builder's graph (records or columns) of the report the case's reference graph was built from."""
    from agent_bom_b200.graph import build_unified_graph_from_report

    d = _identity_docs()[case["builder"]]
    caps, creds = d["tool_caps"], set(d["cred_keys"])
    g = build_unified_graph_from_report(json.loads(json.dumps(d["report"])), classify_tool=lambda n, desc: caps.get(n + SEP + desc, []),
                                        is_credential_key=lambda k: k in creds, columnar=columnar)
    g.device = device
    return g


def snapshot_db(tmp_path: Path) -> Path:
    path = tmp_path / "graph.sqlite"
    path.write_bytes(gzip.decompress((GOLDEN / "snapshot" / "graph.sqlite.gz").read_bytes()))
    return path


def loaded(case: dict, db: Path, device: int = 0):
    from agent_bom_b200.graph import load_snapshot

    return load_snapshot(db, tenant_id=case["tenant"], scan_id=case["snapshot_scan"], device=device)


def without_time(evs, t0_ms: int | None = None, t1_ms: int | None = None) -> list[dict]:
    """Events as the fixture stores them: ``time`` dropped (checked to be integer milliseconds inside [t0, t1] when given),
    JSON round trip."""
    out = []
    for ev in evs:
        ev = dict(ev)
        t = ev.pop("time")
        assert isinstance(t, int)
        if t0_ms is not None:
            assert t0_ms <= t <= t1_ms
        out.append(ev)
    return json.loads(json.dumps(out))


def oracle_of(graph):
    """The oracle CSR of a graph (its host CSR's edge stream) and its findings in ``nodes`` order."""
    from agent_bom_b200.graph.ocsf import finding_indices
    from oracle import oracle as orc

    c = graph.csr
    return orc.build_csr(c.n_nodes, c.src, c.dst, c.rel, c.flags, c.node_type), finding_indices(graph)


def oracle_context(graph, ctx, q: int, labels) -> dict:
    """The ``graph_context`` block the reference builds, restated from an oracle / device context (label column by node index)."""
    from agent_bom_b200.graph.schema import ENTITY_VALUES

    keys = ("affected_agents", "affected_servers", "affected_packages", "exposed_credentials")
    out = {k: [labels[int(s)] for s in ctx.sources(q, b)] for b, k in enumerate(keys)}
    out["blast_radius"] = int(ctx.count[q])
    out["blast_by_type"] = {ENTITY_VALUES[t]: int(c) for t, c in enumerate(ctx.hist[q]) if c}
    return out
