"""CPU oracle for the context-graph report — plain Python.  TEST INFRASTRUCTURE ONLY.

* ``fleet``: a seeded scan report (``agents`` and ``blast_radius`` lists) shaped like an agent fleet: per agent one private
  and ``shared`` shared MCP servers drawn from a pool sized so each shared name is used by about ``clique`` agents, two tools
  per server (one execute-capable), a credential env key on some servers (``cred_share`` of them a key shared fleet-wide,
  the rest from a pool sized like the server pool) and ``agents / 2`` critical / high / medium vulnerabilities.  It also
  returns the tool classifier and credential-key rule the golden generator records from the reference for such reports.
* ``describe``: what ``_build_lateral_path`` (``/root/reference/src/agent_bom/context_graph.py:480-597``) folds into one
  path — credential / tool / vulnerability lists, execute count, severity — restated with a label -> servers index, so a
  ``shares_server`` hop does not scan every node and large seeded fleets can be checked path by path.  The first-add rules
  are restated literally (lists and ``in``), independent of the device's sort-based de-duplication.
"""

from __future__ import annotations

import random

SEV = {"critical": 8.0, "high": 6.0, "medium": 4.0, "low": 2.0, "info": 0.5, "informational": 0.5, "none": 0.0, "unknown": 0.0}
TOOLS = [("run_shell", "Execute arbitrary shell commands", ["execute"]), ("exec_sql", "Execute SQL", ["execute"]),
         ("list_files", "List files in a directory", ["read"]), ("http_get", "Fetch a URL", ["network"]), ("write_file", "Write a file", ["write"])]


def fleet(agents: int, seed: int, *, clique: int = 50, shared: int = 2, cred_share: float = 0.3, tool_names: int = 40):
    """(agents_data, blast_data, classify_tool, is_credential_key) of a seeded fleet."""
    rng = random.Random(seed)
    pool = max(1, (agents * shared) // max(clique, 1))
    cred_pool = [f"SVC_{i:04d}_TOKEN" for i in range(pool)]
    agents_data = []
    for a in range(agents):
        names = [f"own-{a:05d}"] + [f"shared-{i:04d}" for i in rng.sample(range(pool), min(shared, pool))]
        servers = []
        for name in names:
            env = {"HOME": "/h"}
            if rng.random() < 0.3:
                env["GITHUB_TOKEN" if rng.random() < cred_share else rng.choice(cred_pool)] = "x"
            tools = []
            for t in (rng.choice(TOOLS[:2]), rng.choice(TOOLS[2:])):
                tools.append({"name": f"{t[0]}_{rng.randrange(tool_names)}", "description": t[1], "capabilities": list(t[2])})
            servers.append({"name": name, "command": "npx srv", "transport": "stdio", "env": env, "tools": tools, "packages": [{"name": "p"}]})
        agents_data.append({"name": f"agent-{a:05d}", "type": "custom", "status": "configured", "mcp_servers": servers})
    blast = []
    for v in range(agents // 2):
        a = rng.randrange(agents)
        srv = rng.choice(agents_data[a]["mcp_servers"])["name"]
        blast.append({"vulnerability_id": f"CVE-2040-{v:05d}", "package": "p", "severity": rng.choice(["critical", "high", "medium"]),
                      "cvss_score": rng.choice([None, 5.5, 7.8, 9.8]), "epss_score": rng.choice([None, 0.02, 0.4]), "is_kev": rng.random() < 0.1,
                      "affected_agents": [f"agent-{a:05d}"] + [f"agent-{rng.randrange(agents):05d}" for _ in range(2)], "affected_servers": [srv]})

    def classify_tool(name, description="", declared=None):
        return [str(c) for c in declared] if isinstance(declared, list) else []

    def is_credential_key(key):
        return key != "HOME"

    return agents_data, blast, classify_tool, is_credential_key


def _k(kind) -> str:
    return getattr(kind, "value", kind)


def servers_by_label(graph) -> dict:
    """Server node ids per label, in node order."""
    out: dict = {}
    for nid, n in graph.nodes.items():
        if _k(n.kind) == "server":
            out.setdefault(n.label, []).append(nid)
    return out


def describe(graph, hops, kinds, index=None):
    """(credentials, tools, vulnerabilities, execute count, severity) of one path."""
    index = servers_by_label(graph) if index is None else index
    creds, tools, vulns = [], [], []
    box = [0.0, 0]

    def note(o):
        k = _k(o.kind)
        if k == "credential":
            if o.label not in creds:
                creds.append(o.label)
        elif k == "tool":
            if o.label not in tools:
                tools.append(o.label)
                if "execute" in o.metadata.get("capabilities", []):
                    box[1] += 1
        elif k == "vulnerability":
            if o.label not in vulns:
                vulns.append(o.label)
                box[0] = max(box[0], SEV.get(o.metadata.get("severity", ""), 0))

    def surface(sid):
        for e in graph.adjacency.get(sid, []):
            o = graph.nodes.get(e.target)
            if o and (_k(e.kind), _k(o.kind)) in (("exposes", "credential"), ("provides", "tool"), ("vulnerable_to", "vulnerability")):
                note(o)

    for h in hops:
        n = graph.nodes.get(h)
        if n:
            surface(h) if _k(n.kind) == "server" else note(n) if _k(n.kind) in ("credential", "tool", "vulnerability") else None
    for i, kind in enumerate(kinds):
        if i >= len(hops) - 1 or _k(kind) not in ("shares_server", "shares_credential"):
            continue
        link = next((e for e in graph.adjacency.get(hops[i], []) if e.target == hops[i + 1] and _k(e.kind) == _k(kind)), None)
        if link is None:
            continue
        if _k(kind) == "shares_server":
            name = link.metadata.get("server", "")
            if name:
                for sid in index.get(name, ()):
                    surface(sid)
        else:
            name = link.metadata.get("credential", "")
            if name and name not in creds:
                creds.append(name)
    return creds, tools, vulns, box[1], box[0]
