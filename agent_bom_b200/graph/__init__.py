"""Typed exposure graph — the Python surface of the reference's ``agent_bom.graph`` for the traversal hot path.

    from agent_bom_b200.graph import UnifiedGraph, UnifiedNode, UnifiedEdge, EntityType, RelationshipType, AttackPath
    from agent_bom_b200.graph import compute_dependency_reach, derived_attack_paths

Mirrors ``/root/reference/src/agent_bom/graph/__init__.py:8-100`` for the names the hot path needs.
"""

from .alerts import compute_delta_alerts
from .builder import build_unified_graph_from_report
from .clusters import SEMANTIC_CLUSTER_KINDS, SemanticCluster, SemanticClusterExpansion, semantic_cluster_stats, semantic_clusters, semantic_clusters_view
from .container import UnifiedGraph
from .delta import snapshot_diff
from .dependency_reach import PackageReachability, ReachabilityReport, VulnerabilityReachability, compute_dependency_reach
from .envelope import EdgeIndex, exposure_path_for_attack_path, mcp_exposure_path_payload, serialize_attack_path, serialize_attack_paths
from .fix_first import fix_first_view
from .exposure import derived_attack_paths, exposure_path_rows, materialize_attack_paths, node_risk_100, ranked_attack_paths
from .model import AttackPath, UnifiedEdge, UnifiedNode
from .ocsf import iter_ocsf_events, ocsf_event
from .snapshot import SnapshotGraph, load_snapshot
from .schema import FINDING_ENTITY_TYPES, SEVERITY_RANK, EntityType, NodeStatus, RelationshipType

__all__ = [
    "AttackPath", "EntityType", "FINDING_ENTITY_TYPES", "NodeStatus", "PackageReachability", "ReachabilityReport", "RelationshipType", "SEVERITY_RANK", "SnapshotGraph", "load_snapshot",
    "UnifiedEdge", "UnifiedGraph", "UnifiedNode", "VulnerabilityReachability", "build_unified_graph_from_report", "compute_dependency_reach", "derived_attack_paths", "exposure_path_rows",
    "materialize_attack_paths", "node_risk_100", "ranked_attack_paths", "EdgeIndex", "exposure_path_for_attack_path", "mcp_exposure_path_payload",
    "serialize_attack_path", "serialize_attack_paths", "fix_first_view", "iter_ocsf_events", "ocsf_event",
    "SEMANTIC_CLUSTER_KINDS", "SemanticCluster", "SemanticClusterExpansion", "semantic_cluster_stats", "semantic_clusters", "semantic_clusters_view",
    "snapshot_diff", "compute_delta_alerts",
]
