"""Fixture of the fix-first view goldens (``oracle/make_fix_first_golden.py`` → ``tests/golden/fix_first/views.json.gz``): graphs
rebuilt from the reference's node / edge records, and the reference's views and focus verdicts on them."""

from __future__ import annotations

import copy
import gzip
import json
from functools import lru_cache
from pathlib import Path
from types import SimpleNamespace

GOLD = Path(__file__).resolve().parent / "golden" / "fix_first"


@lru_cache(maxsize=None)
def doc() -> dict:
    return json.loads(gzip.decompress((GOLD / "views.json.gz").read_bytes()))


def cases(*, with_graph: bool = True) -> list[dict]:
    return [c for c in doc()["cases"] if ("nodes" in c) == with_graph]


class RecordNode:
    """A reference node record replayed: the fields the engine reads, and the reference's own ``to_dict``."""

    __slots__ = ("id", "entity_type", "label", "severity", "risk_score", "attributes", "_dict")

    def __init__(self, rec: dict):
        self.id, self.entity_type, self.label = rec["id"], rec["entity_type"], rec["label"]
        self.severity, self.risk_score, self.attributes = rec["severity"], rec["risk_score"], rec["attributes"]
        self._dict = rec["to_dict"]

    def to_dict(self) -> dict:
        return copy.deepcopy(self._dict)


def reference_graph(case: dict):
    """A reference-shaped graph object (what ``load_graph`` hands the route) for ``UnifiedGraph.from_graph``."""
    from agent_bom_b200.graph import AttackPath, UnifiedEdge

    nodes = {n["id"]: RecordNode(n) for n in case["nodes"]}
    edges = [UnifiedEdge(**e) for e in case["edges"]]
    return SimpleNamespace(nodes=nodes, edges=edges, attack_paths=[AttackPath(**p) for p in case["attack_paths"]], interaction_risks=[],
                           scan_id=case["scan_id"], tenant_id=case["tenant_id"], created_at=case["created_at"])


def adopted(case: dict, device: int = 0):
    from agent_bom_b200.graph import UnifiedGraph

    return UnifiedGraph.from_graph(reference_graph(case), device=device)


def focus_kwargs(view_case: dict) -> dict:
    f = view_case["focus"]
    return {"cve": f["cve"], "package": f["package"], "agent": f["agent"], "limit": f["limit"]}


def roundtrip(obj):
    return json.loads(json.dumps(obj, sort_keys=True))
