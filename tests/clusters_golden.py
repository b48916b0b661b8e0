"""Fixtures of the semantic-cluster goldens (``oracle/make_clusters_golden.py`` → ``tests/golden/clusters/*.json.gz``): the graphs
rebuilt from the reference's node / edge records (or, for ``light_40``, rebuilt with this package's builder), and the reference's
per-node keys, clusters and route bodies on them."""

from __future__ import annotations

import gzip
import json
from functools import lru_cache
from pathlib import Path
from types import SimpleNamespace

GOLD = Path(__file__).resolve().parent / "golden" / "clusters"
NAMES = ("kat_clusters", "light_40", "estate_dense_40", "estate_150")
LIGHT_AGENTS = 40


def decode(packed: dict) -> dict:
    """Expand a fixture's compact form (``oracle/make_clusters_golden.encode``) into the reference's objects: per-node keys,
    cluster dicts with ``member_ids`` and ``expansion``, route bodies, node and edge records."""
    ids = packed["node_ids"]
    endpoints = ids + packed.get("ghost_ids", [])
    table = packed["key_table"]

    def cluster(c):
        member_ids = [ids[i] for i in c["member_ids"]]
        d = {**c, "member_ids": member_ids}
        d["expansion"] = {"mode": "members", "member_ids": member_ids, "collapse_id": c["id"], "reversible": True}
        return d

    clusters = [cluster(c) for c in packed["cluster_list"]]
    out = {k: packed[k] for k in ("name", "scan_id", "tenant_id", "created_at", "risk", "severity")}
    out["keys"] = [[list(table[k]) for k in ks] for ks in packed["keys"]]
    out["clusters"] = {m: {"clusters": [clusters[i] for i in v["index"]], "stats": v["stats"]} for m, v in packed["clusters"].items()}
    out["views"] = [{"params": v["params"], "body": {**v["body"], "clusters": [clusters[i] for i in v["body"]["clusters"]]}} for v in packed["views"]]
    if "nodes" in packed:
        out["nodes"] = [{"id": nid, **n} for nid, n in zip(ids, packed["nodes"])]
        out["edges"] = [{"source": endpoints[s], "target": endpoints[t], "relationship": rel, "direction": "bidirectional" if bidir else "directed",
                         "traversable": trav} for s, t, rel, bidir, trav in packed["edges"]]
    return out


@lru_cache(maxsize=None)
def case(name: str) -> dict:
    return decode(json.loads(gzip.decompress((GOLD / f"{name}.json.gz").read_bytes())))


class RecordNode:
    """A reference node record replayed; ``dimensions`` as the snapshot's dict, as an object, or absent."""

    def __init__(self, rec: dict, dims_form: str):
        self.id, self.entity_type, self.label = rec["id"], rec["entity_type"], rec["label"]
        self.severity, self.risk_score = rec["severity"], rec["risk_score"]
        self.attributes, self.data_sources = rec["attributes"], rec["data_sources"]
        dims = rec["dimensions"] or {}
        if dims_form == "dict":
            self.dimensions = dict(dims)
        elif dims_form == "object":
            self.dimensions = SimpleNamespace(**{f: dims.get(f, "") for f in ("ecosystem", "cloud_provider", "agent_type", "surface", "environment")})


def light_graph(*, columnar: bool = False, device: int = 0):
    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report

    g = build_unified_graph_from_report(estate.generate(LIGHT_AGENTS, 2145, estate.BENCH_KNOBS).report_json(), columnar=columnar, device=device)
    g.scan_id, g.tenant_id, g.created_at = "light-scan", "default", "2026-05-01T00:00:00+00:00"
    return g


def graph(name: str, *, dims_form: str = "dict", device: int = 0):
    """The golden's graph as a ``UnifiedGraph`` (records adopted as they are)."""
    from agent_bom_b200.graph import UnifiedEdge, UnifiedGraph

    c = case(name)
    if "nodes" not in c:
        return light_graph(device=device)
    nodes = {n["id"]: RecordNode(n, dims_form) for n in c["nodes"]}
    edges = [UnifiedEdge(**e) for e in c["edges"]]
    ref = SimpleNamespace(nodes=nodes, edges=edges, attack_paths=[], interaction_risks=[], scan_id=c["scan_id"], tenant_id=c["tenant_id"],
                          created_at=c["created_at"])
    return UnifiedGraph.from_graph(ref, device=device)


def roundtrip(obj):
    return json.loads(json.dumps(obj, sort_keys=True))
