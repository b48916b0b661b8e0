"""The agent context-graph report: builder, lateral paths, interaction risks and the serialised body (SURVEY §8 f3 / f4).

Reference: ``/root/reference/src/agent_bom/context_graph.py`` — ``build_context_graph`` (:157-388), ``find_lateral_paths``
(:397-597), ``compute_interaction_risks`` (:603-725) and ``to_serializable`` (:731-801).  The REST route
(``api/routes/scan.py:671-708``), the MCP ``context_graph`` tool (``mcp_tools/analysis.py:70-117``) and the CLI's
``--context-graph`` section (``cli/agents/__init__.py:1731-1760``) all run that chain; ``build_context_graph`` +
``context_graph_report`` here is the same chain with its graph work on the device:

* the builder's loops are restated section by section (node order, edge order, adjacency with mirrored twins, weights and
  metadata dicts equal the reference's), then this package's ``effective_reach.annotate_graph`` scores every vulnerability on
  the device (the reference's scorer is O(V·E) and is most of its build time);
* every agent's lateral paths come from one device search and one device enrichment (``lateral.find_lateral_paths_many``);
* ``compute_interaction_risks`` stays on the host: it is one pass over ``graph.edges``, and any device version would need an
  O(E) Python encoding of those same edges first.

Two rules of the reference depend on tables outside its graph code and are injectable, as in ``graph/builder.py``:
``classify_tool(name, description, declared_capabilities) -> list[str]`` (the reference's ``_classify_tool``, :141-151;
default: no capabilities, what the reference answers when its classifier cannot be imported) and
``is_credential_key(name) -> bool`` (default: ``graph.builder``'s fallback rule).

There is no CPU fallback: without the CUDA library the scorer raises ``EngineUnavailable``; scorer errors are not swallowed.
"""

from __future__ import annotations

import re
import time
from collections import defaultdict
from dataclasses import dataclass
from typing import Any, Callable, Iterable, Optional

from .context_graph import ContextGraph, EdgeKind, GraphEdge, GraphNode, NodeKind, kind_value
from .lateral import SEVERITY_RISK_SCORE, LateralPath, find_lateral_paths_many

_CONTROL_CHARS_RE = re.compile(r"[\x00-\x1f\x7f]")
_UNTRUSTED_PREFIX = "[UNTRUSTED MCP METADATA] "

# agent_bom.graph's NODE_KIND_TO_ENTITY / EDGE_KIND_TO_RELATIONSHIP (graph/compat.py), as the values to_serializable emits
NODE_KIND_TO_ENTITY = {"agent": "agent", "server": "server", "credential": "credential", "tool": "tool", "vulnerability": "vulnerability",
                       "iam_role": "service_account"}
EDGE_KIND_TO_RELATIONSHIP = {"uses": "uses", "exposes": "exposes_cred", "provides": "provides_tool", "vulnerable_to": "vulnerable_to",
                             "shares_server": "shares_server", "shares_credential": "shares_cred", "attached_to": "member_of"}


def _untrusted_metadata_text(value: object, *, max_length: int = 1000) -> str:
    """A tool description as the builder stores it: control characters and line separators blanked, prefixed, cut (:43-50)."""
    text = _CONTROL_CHARS_RE.sub(" ", str(value)).replace("\u2028", " ").replace("\u2029", " ")
    return f"{_UNTRUSTED_PREFIX}{text[:max_length]}"


def _no_capabilities(name, description="", declared_capabilities=None) -> list[str]:
    return []


@dataclass
class InteractionRisk:
    """Cross-agent interaction risk pattern (``agent_bom.graph.InteractionRisk``)."""

    pattern: str
    agents: list[str]
    risk_score: float
    description: str
    owasp_agentic_tag: Optional[str] = None


def build_context_graph(agents_data: list[dict], blast_data: list[dict], *, classify_tool: Callable[[Any, Any, Any], Iterable[str]] | None = None,
                        is_credential_key: Callable[[str], bool] | None = None, device: int = 0, timings: dict | None = None) -> ContextGraph:
    """The context graph of a scan report's ``agents`` and ``blast_radius`` lists, effective-reach annotations included
    (:157-388).  ``timings``, when given, receives the seconds of the builder's loops (``build``) and of the scorer (``score``)."""
    from .effective_reach import annotate_graph

    if is_credential_key is None:
        from .graph.builder import _default_is_credential_key as is_credential_key
    classify = classify_tool or _no_capabilities
    t0 = time.perf_counter()
    graph = ContextGraph()
    server_to_agents: dict[Any, list] = defaultdict(list)
    cred_to_agents: dict[Any, list] = defaultdict(list)

    # agents, their IAM roles, servers, credentials and tools (:177-299)
    for agent_dict in agents_data:
        agent_name = agent_dict.get("name", "unknown")
        agent_id = f"agent:{agent_name}"
        graph.add_node(GraphNode(id=agent_id, kind=NodeKind.AGENT, label=agent_name,
                                 metadata={"agent_type": agent_dict.get("type", ""), "status": agent_dict.get("status", ""),
                                           "server_count": len(agent_dict.get("mcp_servers", []))}))
        cloud_principal = (agent_dict.get("metadata") or {}).get("cloud_principal")
        if cloud_principal and isinstance(cloud_principal, dict):
            principal_id = cloud_principal.get("principal_id") or cloud_principal.get("principal_name", "")
            if principal_id:
                role_id = f"iam_role:{principal_id}"
                if role_id not in graph.nodes:
                    graph.add_node(GraphNode(id=role_id, kind=NodeKind.IAM_ROLE, label=principal_id,
                                             metadata={"principal_type": cloud_principal.get("principal_type", ""),
                                                       "provider": cloud_principal.get("provider", ""), "service": cloud_principal.get("service", "")}))
                graph.add_edge(GraphEdge(source=role_id, target=agent_id, kind=EdgeKind.ATTACHED_TO, weight=2.0,
                                         metadata={"principal_type": cloud_principal.get("principal_type", "")}))
        for srv_dict in agent_dict.get("mcp_servers", []):
            srv_name = srv_dict.get("name", "unknown")
            srv_id = f"server:{agent_name}:{srv_name}"
            graph.add_node(GraphNode(id=srv_id, kind=NodeKind.SERVER, label=srv_name,
                                     metadata={"command": srv_dict.get("command", ""), "transport": srv_dict.get("transport", ""),
                                               "package_count": len(srv_dict.get("packages", [])), "agent": agent_name}))
            graph.add_edge(GraphEdge(source=agent_id, target=srv_id, kind=EdgeKind.USES))
            server_to_agents[srv_name].append(agent_name)
            for env_key in srv_dict.get("env", {}):
                if is_credential_key(env_key):
                    cred_id = f"cred:{env_key}"
                    if cred_id not in graph.nodes:
                        graph.add_node(GraphNode(id=cred_id, kind=NodeKind.CREDENTIAL, label=env_key, metadata={"servers": []}))
                    if srv_id not in graph.nodes[cred_id].metadata["servers"]:
                        graph.nodes[cred_id].metadata["servers"].append(srv_id)
                    graph.add_edge(GraphEdge(source=srv_id, target=cred_id, kind=EdgeKind.EXPOSES, weight=2.0))
                    cred_to_agents[env_key].append(agent_name)
            for tool_dict in srv_dict.get("tools", []):
                tool_name = tool_dict.get("name", "unknown")
                tool_desc = tool_dict.get("description", "")
                tool_id = f"tool:{srv_id}:{tool_name}"
                capabilities = list(classify(tool_name, tool_desc, tool_dict.get("capabilities")))
                graph.add_node(GraphNode(id=tool_id, kind=NodeKind.TOOL, label=tool_name,
                                         metadata={"description": _untrusted_metadata_text(tool_desc), "description_trust": "untrusted_external_mcp_metadata",
                                                   "capabilities": capabilities, "server": srv_id, "agent": agent_name}))
                graph.add_edge(GraphEdge(source=srv_id, target=tool_id, kind=EdgeKind.PROVIDES, weight=3.0 if "execute" in capabilities else 1.0))

    # vulnerabilities and the servers they affect (:302-340)
    seen_vulns: set = set()
    for br_dict in blast_data:
        vuln_id = br_dict.get("vulnerability_id", "")
        if not vuln_id:
            continue
        severity = br_dict.get("severity", "").lower()
        if vuln_id not in seen_vulns:
            seen_vulns.add(vuln_id)
            graph.add_node(GraphNode(id=f"vuln:{vuln_id}", kind=NodeKind.VULNERABILITY, label=vuln_id,
                                     metadata={"severity": severity, "cvss_score": br_dict.get("cvss_score"), "epss_score": br_dict.get("epss_score"),
                                               "is_kev": br_dict.get("is_kev", False), "risk_score": br_dict.get("risk_score", 0),
                                               "package": br_dict.get("package", "")}))
        for agent_name in br_dict.get("affected_agents", []):
            for srv_name in br_dict.get("affected_servers", []):
                srv_id = f"server:{agent_name}:{srv_name}"
                if srv_id in graph.nodes:
                    graph.add_edge(GraphEdge(source=srv_id, target=f"vuln:{vuln_id}", kind=EdgeKind.VULNERABLE_TO,
                                             weight=SEVERITY_RISK_SCORE.get(severity, 1.0), metadata={"package": br_dict.get("package", "")}))

    # agent <-> agent cliques per shared server name, then per shared credential name; add_edge keeps the first (:343-373)
    for kind, weight, key, table in ((EdgeKind.SHARES_SERVER, 3.0, "server", server_to_agents), (EdgeKind.SHARES_CREDENTIAL, 4.0, "credential", cred_to_agents)):
        for name, agent_names in table.items():
            unique = sorted(set(agent_names))
            if len(unique) >= 2:
                for i, a1 in enumerate(unique):
                    for a2 in unique[i + 1:]:
                        graph.add_edge(GraphEdge(source=f"agent:{a1}", target=f"agent:{a2}", kind=kind, weight=weight, metadata={key: name}))
    t1 = time.perf_counter()
    annotate_graph(graph, device=device)
    if timings is not None:
        timings.update(build=t1 - t0, score=time.perf_counter() - t1)
    return graph


def compute_interaction_risks(graph) -> list[InteractionRisk]:
    """Shared-credential, shared-server, execute-tool-overlap and multi-hop-vulnerability patterns, sorted by score (:603-725)."""
    risks: list[InteractionRisk] = []
    shared_servers: dict[Any, list[str]] = defaultdict(list)
    shared_creds: dict[Any, list[str]] = defaultdict(list)
    for edge in graph.edges:
        k = kind_value(edge.kind)
        if k == "shares_server":
            shared_servers[edge.metadata.get("server", "")].extend([edge.source.removeprefix("agent:"), edge.target.removeprefix("agent:")])
        elif k == "shares_credential":
            shared_creds[edge.metadata.get("credential", "")].extend([edge.source.removeprefix("agent:"), edge.target.removeprefix("agent:")])

    for cred_name, agent_names in shared_creds.items():
        unique = sorted(set(agent_names))
        if len(unique) >= 2:
            risks.append(InteractionRisk(
                pattern="shared_credential", agents=unique, risk_score=7.0 + min(len(unique) * 0.5, 2.0),
                description=(f"Credential '{cred_name}' is shared across {len(unique)} agents ({', '.join(unique)}). Compromising one agent grants "
                             f"access to the credential used by others."),
                owasp_agentic_tag="ASI07"))
    for srv_name, agent_names in shared_servers.items():
        unique = sorted(set(agent_names))
        if len(unique) >= 2:
            risks.append(InteractionRisk(
                pattern="shared_server", agents=unique, risk_score=5.0 + min(len(unique) * 0.5, 2.0),
                description=f"MCP server '{srv_name}' is shared across {len(unique)} agents ({', '.join(unique)}). A vulnerability in this server affects all."))

    execute_agents: dict[Any, set] = defaultdict(set)
    for node in graph.nodes.values():
        if kind_value(node.kind) == "tool" and "execute" in node.metadata.get("capabilities", []):
            agent_name = node.metadata.get("agent", "")
            if agent_name:
                execute_agents[node.label].add(agent_name)
    for tool_name, agents in execute_agents.items():
        if len(agents) >= 2:
            unique = sorted(agents)
            risks.append(InteractionRisk(
                pattern="tool_overlap_execute", agents=unique, risk_score=6.0 + min(len(unique) * 0.5, 2.0),
                description=(f"EXECUTE-capable tool '{tool_name}' is accessible to {len(unique)} agents ({', '.join(unique)}). Code execution from "
                             f"any of them can pivot laterally."),
                owasp_agentic_tag="ASI07"))

    for edge in graph.edges:
        if kind_value(edge.kind) != "vulnerable_to":
            continue
        srv_node, vuln_node = graph.nodes.get(edge.source), graph.nodes.get(edge.target)
        if not srv_node or not vuln_node:
            continue
        sev = vuln_node.metadata.get("severity", "")
        if sev not in ("critical", "high"):
            continue
        srv_name = srv_node.label
        if srv_name in shared_servers:
            unique = sorted(set(shared_servers[srv_name]))
            risks.append(InteractionRisk(
                pattern="multi_hop_vuln", agents=unique, risk_score=8.0 + (1.0 if sev == "critical" else 0.0),
                description=(f"{sev.upper()} vulnerability {vuln_node.label} in shared server '{srv_name}' affects agents: {', '.join(unique)}. "
                             f"Exploit chains across agents are possible."),
                owasp_agentic_tag="ASI07"))

    # multi-hop findings de-duplicated by (third word of the description, agent set): the first word of a vulnerability label
    seen: set = set()
    deduped: list[InteractionRisk] = []
    for risk in risks:
        if risk.pattern == "multi_hop_vuln":
            key = (risk.description.split(" ")[2], frozenset(risk.agents))
            if key in seen:
                continue
            seen.add(key)
        deduped.append(risk)
    deduped.sort(key=lambda r: r.risk_score, reverse=True)
    return deduped


def lateral_paths_for(graph, *, agent: str | None = None, max_depth: int = 4, device: int = 0, timings: dict | None = None) -> list[LateralPath]:
    """The paths the route collects: from ``agent:{agent}`` only (none when that node is absent), or from every agent node in node
    order, each agent's list sorted by composite risk; one device search and one enrichment for all of them."""
    if agent:
        node_id = f"agent:{agent}"
        sources = [node_id] if node_id in graph.nodes else []
    else:
        sources = [nid for nid, node in graph.nodes.items() if kind_value(node.kind) == "agent"]
    if not sources:
        return []
    return [p for per_source in find_lateral_paths_many(graph, sources, max_depth, device=device, timings=timings) for p in per_source]


def to_serializable(graph, lateral_paths: list[LateralPath] | None = None, interaction_risks: list[InteractionRisk] | None = None) -> dict:
    """The report body: nodes, edges, lateral paths, interaction risks and stats, keys in the reference's order (:731-801)."""
    paths = lateral_paths or []
    risks = interaction_risks or []
    edge_kinds = [kind_value(e.kind) for e in graph.edges]
    return {
        "nodes": [{"id": n.id, "kind": kind_value(n.kind), "entity_type": NODE_KIND_TO_ENTITY.get(kind_value(n.kind), "server"), "label": n.label,
                   "metadata": n.metadata} for n in graph.nodes.values()],
        "edges": [{"source": e.source, "target": e.target, "kind": k, "relationship": EDGE_KIND_TO_RELATIONSHIP.get(k, k), "weight": e.weight,
                   "metadata": e.metadata} for e, k in zip(graph.edges, edge_kinds)],
        "lateral_paths": [{"source": p.source, "target": p.target, "hops": p.hops, "edges": [kind_value(ek) for ek in p.edges],
                           "composite_risk": p.composite_risk, "summary": p.summary, "credential_exposure": p.credential_exposure,
                           "tool_exposure": p.tool_exposure, "vuln_ids": p.vuln_ids} for p in paths],
        "interaction_risks": [{"pattern": r.pattern, "agents": r.agents, "risk_score": r.risk_score, "description": r.description,
                               "owasp_agentic_tag": r.owasp_agentic_tag} for r in risks],
        "stats": {
            "total_nodes": len(graph.nodes),
            "total_edges": len(graph.edges),
            "agent_count": sum(1 for n in graph.nodes.values() if kind_value(n.kind) == "agent"),
            "shared_server_count": edge_kinds.count("shares_server"),
            "shared_credential_count": edge_kinds.count("shares_credential"),
            "lateral_path_count": len(paths),
            "max_lateral_depth": max((len(p.hops) - 1 for p in paths), default=0),
            "highest_path_risk": max((p.composite_risk for p in paths), default=0.0),
            "interaction_risk_count": len(risks),
        },
    }


def context_graph_report(graph, *, agent: str | None = None, max_depth: int = 4, device: int = 0, timings: dict | None = None) -> dict:
    """``to_serializable(graph, paths, compute_interaction_risks(graph))`` as the REST route, the MCP tool and the CLI build it:
    with ``agent`` only that agent's paths, otherwise every agent's.  A search that exceeds its safety valve raises
    ``LateralSearchOverflow``; no partial body is returned.  ``timings``, when given, receives per-stage seconds."""
    paths = lateral_paths_for(graph, agent=agent, max_depth=max_depth, device=device, timings=timings)
    t0 = time.perf_counter()
    risks = compute_interaction_risks(graph)
    t1 = time.perf_counter()
    body = to_serializable(graph, paths, risks)
    if timings is not None:
        timings.update(risks=t1 - t0, serialise=time.perf_counter() - t1)
    return body


__all__ = ["EDGE_KIND_TO_RELATIONSHIP", "NODE_KIND_TO_ENTITY", "InteractionRisk", "build_context_graph", "compute_interaction_risks",
           "context_graph_report", "lateral_paths_for", "to_serializable"]
