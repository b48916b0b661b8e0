"""Light records of the legacy agent context graph — only what effective-reach scoring reads.

The reference keeps a second, older graph model next to ``UnifiedGraph``: ``ContextGraph`` with ``NodeKind`` /
``EdgeKind`` (``/root/reference/src/agent_bom/context_graph.py:54-130``).  Effective-reach scoring
(``effective_reach.py``) is defined on that model, so the scorer here accepts any object of this shape — these
records, or the reference's own ``build_context_graph`` output (duck-typed: ``nodes`` dict, ``edges`` list,
``adjacency`` dict of per-node edge lists).  ``context_report.build_context_graph`` builds these records from a scan report.
"""

from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass, field
from enum import Enum


class NodeKind(str, Enum):
    AGENT = "agent"
    SERVER = "server"
    CREDENTIAL = "credential"
    TOOL = "tool"
    VULNERABILITY = "vulnerability"
    IAM_ROLE = "iam_role"


class EdgeKind(str, Enum):
    USES = "uses"
    EXPOSES = "exposes"
    PROVIDES = "provides"
    VULNERABLE_TO = "vulnerable_to"
    SHARES_SERVER = "shares_server"
    SHARES_CREDENTIAL = "shares_credential"
    ATTACHED_TO = "attached_to"


@dataclass
class GraphNode:
    id: str
    kind: NodeKind
    label: str
    metadata: dict = field(default_factory=dict)


@dataclass
class GraphEdge:
    source: str
    target: str
    kind: EdgeKind
    weight: float = 1.0
    metadata: dict = field(default_factory=dict)


def kind_value(kind) -> str:
    return kind.value if isinstance(kind, Enum) else str(kind)


@dataclass
class ContextGraph:
    """Nodes by id, edges in insertion order, and an adjacency that holds every edge at its source AND a mirrored twin
    at its target (context_graph.py:108-127) — the scorer reads ``adjacency`` as the caller left it."""

    nodes: dict[str, GraphNode] = field(default_factory=dict)
    edges: list[GraphEdge] = field(default_factory=list)
    adjacency: dict[str, list[GraphEdge]] = field(default_factory=lambda: defaultdict(list))
    _edge_keys: set = field(default_factory=set)

    def add_node(self, node: GraphNode) -> None:
        self.nodes[node.id] = node

    def add_edge(self, edge: GraphEdge) -> None:
        key = (edge.source, edge.target, kind_value(edge.kind))
        if key in self._edge_keys:
            return
        self._edge_keys.add(key)
        self.edges.append(edge)
        self.adjacency[edge.source].append(edge)
        self.adjacency[edge.target].append(GraphEdge(source=edge.target, target=edge.source, kind=edge.kind, weight=edge.weight, metadata=edge.metadata))
