#!/usr/bin/env python3
"""Generate tests/golden/context/report.json.xz by running the UNMODIFIED reference context-graph chain.

Runs only where the reference tree exists (imports ``/root/reference/src``).  For each input the reference's
``build_context_graph`` builds the graph (its own ``annotate_graph`` included), and the report body is what the REST route
assembles (``api/routes/scan.py:671-708``): ``find_lateral_paths`` per agent, ``compute_interaction_risks``, ``to_serializable``.

Inputs:
- scenarios built with the reference's own test helpers (``tests/test_context_graph.py``): shared servers and credentials,
  declared and classified capabilities, untrusted descriptions, vulnerabilities, IAM roles, the 20-agent path cap;
- seeded fleets (``oracle/context_report_oracle.py``) of 40 and 120 agents, small enough for the reference's O(V·E) scorer;
- hand-wired graphs on the reference's container: adjacency entries that are not in ``edges``, sharing edges without
  metadata, ghost targets, one server label on many servers, string and dict ``capabilities``, empty and multi-word
  vulnerability labels, two shared names with the same agent set, and one graph whose ``capabilities`` is an int (the
  reference raises ``TypeError``).

Recorded per input: the report lists (built inputs), each tool's capabilities as the reference's classifier answers them and
the env keys its credential rule accepts (so a test can inject both), the built graph (nodes, edges and adjacency with weights
and metadata), and report bodies for ``agent=None`` at depths 1, 2, 4 and 6, for each agent at depth 4 (every sixth on the
120-agent fleet) and for an unknown agent.  Bodies are stored as JSON text per top-level key (nodes / edges / interaction
risks once per graph), so key order is kept; a body that raises is stored as its exception.  The file is xz-compressed: the
all-agent bodies repeat the per-agent path lists, which xz's window finds and gzip's 32 KiB window does not (about 0.2 MiB
against 1.6 MiB).

    python oracle/make_context_report_golden.py
"""

from __future__ import annotations

import copy
import importlib.util
import json
import lzma
import sys
from pathlib import Path

REF = Path("/root/reference")
sys.path.insert(0, str(REF / "src"))
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from agent_bom.constants import is_credential_key  # noqa: E402
from agent_bom.context_graph import (  # noqa: E402
    ContextGraph,
    EdgeKind,
    GraphEdge,
    GraphNode,
    NodeKind,
    _classify_tool,
    build_context_graph,
    compute_interaction_risks,
    find_lateral_paths,
    to_serializable,
)

from oracle.context_report_oracle import fleet  # noqa: E402

OUT = ROOT / "tests" / "golden" / "context" / "report.json.xz"
DEPTHS = (1, 2, 4, 6)


def _entry(e):
    return [e.source, e.target, e.kind.value, e.weight, e.metadata]


def graph_doc(g):
    return {"nodes": [[n.id, n.kind.value, n.label, n.metadata] for n in g.nodes.values()],
            "edges": [_entry(e) for e in g.edges],
            "adjacency": [[nid, [_entry(e) for e in lst]] for nid, lst in g.adjacency.items()]}


def report(g, agent, depth):
    """The REST route's body (agent filter) at a depth the MCP tool allows; an exception is recorded as such."""
    try:
        paths = []
        if agent:
            nid = f"agent:{agent}"
            if nid in g.nodes:
                paths = find_lateral_paths(g, nid, max_depth=depth)
        else:
            for nid, node in g.nodes.items():
                if node.kind == NodeKind.AGENT:
                    paths.extend(find_lateral_paths(g, nid, max_depth=depth))
        risks = compute_interaction_risks(g)
        return to_serializable(g, paths, risks), None
    except Exception as exc:  # noqa: BLE001 - the golden records what the reference raises
        return None, f"{type(exc).__name__}: {exc}"


def reports_doc(g, every=1):
    agents = [n.label for n in g.nodes.values() if n.kind == NodeKind.AGENT][::every]
    cases = [(None, d) for d in DEPTHS] + [(a, 4) for a in agents] + [("no-such-agent", 4), ("", 2)]
    shared, out = None, []
    for agent, depth in cases:
        body, error = report(g, agent, depth)
        if error is not None:
            out.append({"agent": agent, "max_depth": depth, "error": error})
            continue
        parts = {k: json.dumps(v) for k, v in body.items()}
        if shared is None:
            shared = {k: parts[k] for k in ("nodes", "edges", "interaction_risks")}
        assert all(parts[k] == shared[k] for k in shared)
        out.append({"agent": agent, "max_depth": depth, "keys": list(body), "lateral_paths": parts["lateral_paths"], "stats": parts["stats"]})
    return shared, out


def input_doc(name, agents, blast, every=1):
    """Build with the reference and record what a test needs to rebuild it with injected rules."""
    tool_caps, cred_keys = {}, []
    for a in agents:
        for s in a.get("mcp_servers", []):
            for k in s.get("env", {}):
                if is_credential_key(k) and k not in cred_keys:
                    cred_keys.append(k)
            for t in s.get("tools", []):
                name_, desc, declared = t.get("name", "unknown"), t.get("description", ""), t.get("capabilities")
                tool_caps[json.dumps([name_, desc, declared])] = _classify_tool(name_, desc, declared)
    g = build_context_graph(copy.deepcopy(agents), copy.deepcopy(blast))
    shared, reps = reports_doc(g, every)
    doc = {"name": name, "input": {"agents": agents, "blast": blast, "tool_caps": tool_caps, "cred_keys": cred_keys}, "graph": graph_doc(g),
           "body": shared, "reports": reps}
    print(f"{name}: {len(g.nodes)} nodes {len(g.edges)} edges, {len(reps)} reports, "
          f"{sum(json.loads(r['stats'])['lateral_path_count'] for r in reps if 'stats' in r)} paths")
    return doc


def hand_doc(name, g, extra):
    shared, reps = reports_doc(g)
    doc = {"name": name, "input": None, "graph": graph_doc(g), "extra_adjacency": extra, "body": shared, "reports": reps}
    print(f"{name}: {len(g.nodes)} nodes {len(g.edges)} edges, {len(reps)} reports")
    return doc


def hand_wired(bad_caps: bool = False):
    """A graph the builder cannot make: see the module docstring."""
    g = ContextGraph()
    nodes = [("agent:a", NodeKind.AGENT, "a", {}), ("agent:b", NodeKind.AGENT, "b", {}), ("agent:c", NodeKind.AGENT, "c", {}),
             ("agent:d", NodeKind.AGENT, "d", {}), ("agent:e", NodeKind.AGENT, "e", {})]
    for i, owner in enumerate("abcde"):
        nodes.append((f"server:{owner}:s", NodeKind.SERVER, "s", {"agent": owner}))           # one label on five servers
    nodes += [("server:a:t", NodeKind.SERVER, "t", {"agent": "a"}), ("server:b:t", NodeKind.SERVER, "t", {"agent": "b"}),
              ("tool:1", NodeKind.TOOL, "exec-str", {"agent": "a", "capabilities": "can_execute_code"}),
              ("tool:2", NodeKind.TOOL, "read-str", {"agent": "b", "capabilities": "read"}),
              ("tool:3", NodeKind.TOOL, "exec-dict", {"agent": "c", "capabilities": 5 if bad_caps else {"execute": True}}),
              ("tool:4", NodeKind.TOOL, "exec-str", {"agent": "d", "capabilities": []}),
              ("tool:5", NodeKind.TOOL, "plain", {"agent": "e"}),
              ("cred:1", NodeKind.CREDENTIAL, "GITHUB_TOKEN", {"servers": []}), ("cred:2", NodeKind.CREDENTIAL, "DB_PASSWORD", {"agent": "c"}),
              ("vuln:1", NodeKind.VULNERABILITY, "", {"severity": "critical"}),
              ("vuln:2", NodeKind.VULNERABILITY, "CVE-2 and more words", {"severity": "high"}),
              ("vuln:3", NodeKind.VULNERABILITY, "CVE-3", {"severity": "weird"}), ("vuln:4", NodeKind.VULNERABILITY, "CVE-4", {}),
              ("vuln:5", NodeKind.VULNERABILITY, "CVE-2 other", {"severity": "critical"})]
    for nid, kind, label, meta in nodes:
        g.add_node(GraphNode(id=nid, kind=kind, label=label, metadata=meta))
    edges = [("agent:a", "server:a:s", EdgeKind.USES, {}), ("agent:b", "server:b:s", EdgeKind.USES, {}), ("agent:c", "server:c:s", EdgeKind.USES, {}),
             ("agent:d", "server:d:s", EdgeKind.USES, {}), ("agent:e", "server:e:s", EdgeKind.USES, {}),
             ("agent:a", "server:a:t", EdgeKind.USES, {}), ("agent:b", "server:b:t", EdgeKind.USES, {}),
             ("server:a:s", "tool:1", EdgeKind.PROVIDES, {}), ("server:b:s", "tool:2", EdgeKind.PROVIDES, {}), ("server:c:s", "tool:3", EdgeKind.PROVIDES, {}),
             ("server:d:s", "tool:4", EdgeKind.PROVIDES, {}), ("server:e:s", "tool:5", EdgeKind.PROVIDES, {}),
             ("server:a:s", "cred:1", EdgeKind.EXPOSES, {}), ("server:c:s", "cred:2", EdgeKind.EXPOSES, {}), ("server:b:t", "cred:1", EdgeKind.EXPOSES, {}),
             ("server:b:s", "vuln:1", EdgeKind.VULNERABLE_TO, {}), ("server:a:s", "vuln:2", EdgeKind.VULNERABLE_TO, {}),
             ("server:a:t", "vuln:5", EdgeKind.VULNERABLE_TO, {}), ("server:b:t", "vuln:5", EdgeKind.VULNERABLE_TO, {}),
             ("server:d:s", "vuln:3", EdgeKind.VULNERABLE_TO, {}), ("server:e:s", "vuln:4", EdgeKind.VULNERABLE_TO, {}),
             ("server:c:s", "ghost:tool", EdgeKind.PROVIDES, {}), ("server:c:s", "tool:5", EdgeKind.EXPOSES, {}),   # ghost target; kind mismatch
             ("agent:a", "agent:b", EdgeKind.SHARES_SERVER, {"server": "s"}), ("agent:a", "agent:b", EdgeKind.SHARES_CREDENTIAL, {"credential": "GITHUB_TOKEN"}),
             ("agent:a", "agent:c", EdgeKind.SHARES_SERVER, {}),                                                   # no metadata
             ("agent:b", "agent:c", EdgeKind.SHARES_SERVER, {"server": "t"}), ("agent:b", "agent:a", EdgeKind.SHARES_SERVER, {"server": "t"}),
             ("agent:c", "agent:d", EdgeKind.SHARES_CREDENTIAL, {"credential": "ONLY_ON_THE_LINK"}),
             ("agent:d", "agent:e", EdgeKind.SHARES_SERVER, {"server": "nowhere"}), ("agent:c", "agent:e", EdgeKind.SHARES_CREDENTIAL, {})]
    for s, t, k, meta in edges:
        g.add_edge(GraphEdge(source=s, target=t, kind=k, metadata=meta))
    extra = [("agent:d", "agent:d", "agent:a", EdgeKind.SHARES_SERVER, {"server": "s"}),        # adjacency only: the search sees it, risks do not
             ("agent:e", "agent:e", "agent:b", EdgeKind.SHARES_CREDENTIAL, {"credential": "DB_PASSWORD"}),
             ("server:e:s", "server:e:s", "cred:2", EdgeKind.EXPOSES, {}), ("server:e:s", "server:e:s", "ghost:cred", EdgeKind.EXPOSES, {})]
    for owner, s, t, k, meta in extra:
        g.adjacency[owner].append(GraphEdge(source=s, target=t, kind=k, metadata=meta))
    return g, [[owner, s, t, k.value, 1.0, meta] for owner, s, t, k, meta in extra]


def main():
    spec = importlib.util.spec_from_file_location("ref_test_context_graph_report", REF / "tests" / "test_context_graph.py")
    rt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rt)
    docs = []
    principal = {"principal_id": "arn:aws:iam::123:role/Shared", "principal_name": "Shared", "principal_type": "role", "provider": "aws", "service": "lambda"}
    scenarios = {
        "ref_shared_server": ([rt._agent(name="agent-a", servers=[rt._server(name="shared-srv")]), rt._agent(name="agent-b", servers=[rt._server(name="shared-srv")])], []),
        "ref_risk_scoring": ([rt._agent(name="agent-a", servers=[rt._server(name="srv", env={"SECRET_KEY": "x"})]), rt._agent(name="agent-b", servers=[rt._server(name="srv")])],
                             [rt._blast(severity="critical", agents=["agent-a", "agent-b"], servers=["srv"])]),
        "ref_tools": ([rt._agent(name="agent-a", servers=[rt._server(name="srv", tools=[rt._tool("run_shell", "Execute shell commands"),
                                                                                         rt._tool("reader", "Reads", capabilities=["write"]),
                                                                                         rt._tool("odd", "line break\x07bell " + "x" * 1200)])]),
                       rt._agent(name="agent-b", servers=[rt._server(name="srv", tools=[rt._tool("run_shell", "Execute shell commands")])])], []),
        "ref_shared_credential": ([rt._agent(name=f"agent-{i}", servers=[rt._server(name=f"own-{i}", env={"GITHUB_TOKEN": "x", "HOME": "/h"})]) for i in range(4)],
                                  [rt._blast(vuln_id="CVE-2025-0002", severity="high", agents=["agent-0", "agent-1"], servers=["own-0", "own-1"]),
                                   rt._blast(vuln_id="CVE-2025-0002", severity="HIGH", agents=["agent-2"], servers=["own-2"]),
                                   {"vulnerability_id": "", "severity": "low"}, {"vulnerability_id": "CVE-2025-0003"}]),
        "ref_cap_20_agents": ([rt._agent(name=f"agent-{i}", servers=[rt._server(name="shared", env={"KEY": "x"}, tools=[rt._tool("exec", "run code")])])
                               for i in range(20)], [rt._blast(severity="critical", agents=[f"agent-{i}" for i in range(20)], servers=["shared"])]),
        "ref_iam_roles": ([{"name": "fn1", "type": "cloud", "status": "active", "mcp_servers": [rt._server(name="s")], "metadata": {"cloud_principal": dict(principal)}},
                           {"name": "fn2", "type": "cloud", "status": "active", "mcp_servers": [rt._server(name="s")], "metadata": {"cloud_principal": dict(principal)}},
                           {"name": "plain", "mcp_servers": [], "metadata": {"cloud_principal": {"principal_name": "only-name"}}},
                           {"name": "fn1", "type": "again", "mcp_servers": []}], []),
        "ref_empty": ([], []),
    }
    for name, (agents, blast) in scenarios.items():
        docs.append(input_doc(name, agents, blast))
    for n_agents, seed, clique in ((40, 11, 10), (120, 12, 30)):
        agents, blast, _c, _k = fleet(n_agents, seed, clique=clique)
        docs.append(input_doc(f"fleet_{n_agents}", agents, blast, every=1 if n_agents < 100 else 6))
    g, extra = hand_wired()
    docs.append(hand_doc("hand_wired", g, extra))
    g, extra = hand_wired(bad_caps=True)
    docs.append(hand_doc("hand_wired_bad_capabilities", g, extra))
    OUT.parent.mkdir(parents=True, exist_ok=True)
    with lzma.open(OUT, "wb", preset=9 | lzma.PRESET_EXTREME) as fh:
        fh.write(json.dumps(docs, separators=(",", ":")).encode())
    print(f"-> {OUT} {OUT.stat().st_size / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
