"""Generate tests/golden/hops/ with the UNMODIFIED reference's expand_blast_radius_hops (scanners/blast_radius.py:16-97).

Every case is plain data (see tests/hops_golden.py).  Here it is built into the reference's own Agent, MCPServer and
BlastRadius objects, the reference expands it, and the five fields it wrote are stored (credentials sorted: the reference
returns them in set order).  The cases: the scenarios of the reference's tests/test_multi_hop_blast_radius.py, seeded fleets of
200 agents at depths 0-5 and 10, and hand-built edge cases.

    python oracle/make_hops_golden.py            # writes tests/golden/hops/cases.json.xz
    python oracle/make_hops_golden.py --time     # instead times the reference on the profile's fleets (profiles/)
"""

from __future__ import annotations

import json
import lzma
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, "/root/reference/src")

from oracle import hops_oracle  # noqa: E402

SENTINEL = -12345


def _ref_objects(data: dict):
    from agent_bom.models import Agent, AgentStatus, AgentType, BlastRadius, MCPServer, Package, Severity, TransportType, Vulnerability

    agents = []
    for a in data["agents"]:
        servers = []
        for s in a["servers"]:
            srv = MCPServer(name=s["name"], command="node", args=[], transport=TransportType.STDIO)
            srv.env = {k: "***" for k in s.get("env", s["creds"])}
            servers.append(srv)
        agents.append(Agent(name=a["name"], agent_type=AgentType(a["type"]), config_path="/tmp/x", source="golden", status=AgentStatus.CONFIGURED,
                            mcp_servers=servers))
    by_name = {}
    for ag in agents:
        by_name.setdefault(ag.name, ag)
    radii = []
    for k, b in enumerate(data["blast_radii"]):
        affected = [by_name.get(n) or Agent(name=n, agent_type=AgentType.CUSTOM, config_path="/tmp/x", source="golden", status=AgentStatus.CONFIGURED,
                                             mcp_servers=[]) for n in b["agents"]]
        br = BlastRadius(vulnerability=Vulnerability(id=f"CVE-2025-{k:04d}", summary="", severity=Severity.HIGH),
                         package=Package(name=f"pkg-{k}", version="1.0.0", ecosystem="npm"),
                         affected_servers=[MCPServer(name=n, command="node", args=[], transport=TransportType.STDIO) for n in b["servers"]],
                         affected_agents=affected, exposed_credentials=[], exposed_tools=[])
        br.risk_score = b["risk"]
        br.hop_depth = SENTINEL
        radii.append(br)
    return agents, radii


def run_reference(data: dict, depth: int) -> dict:
    """The case with the credential names the reference reads and its expected fields."""
    from agent_bom.scanners.blast_radius import expand_blast_radius_hops

    agents, radii = _ref_objects(data)
    plain_agents = [{"name": a.name, "type": a.agent_type.value, "servers": [{"name": s.name, "creds": list(s.credential_names)} for s in a.mcp_servers]}
                    for a in agents]
    expand_blast_radius_hops(radii, agents, max_depth=depth)
    expected = []
    for br in radii:
        if br.hop_depth == SENTINEL:
            expected.append(None)
            continue
        expected.append({"hop_depth": br.hop_depth, "delegation_chain": br.delegation_chain, "transitive_agents": br.transitive_agents,
                         "transitive_credentials": sorted(br.transitive_credentials), "transitive_risk_score": br.transitive_risk_score})
    return {"depth": depth, "agents": plain_agents, "blast_radii": data["blast_radii"], "expected": expected}


def _a(name, type_, *servers):
    return {"name": name, "type": type_, "servers": [{"name": s[0], "creds": list(s[1:])} if isinstance(s, tuple) else {"name": s, "creds": []} for s in servers]}


def _case(name, agents, radii, depths):
    return [(f"{name}@{d}", {"agents": agents, "blast_radii": [{"agents": r[0], "servers": r[1], "risk": r[2] if len(r) > 2 else 6.0} for r in radii]}, d)
            for d in depths]


def reference_test_scenarios():
    c = "custom"
    out = []
    out += _case("test_no_op_at_depth_1", [_a("agent1", c, "srv1")], [(["agent1"], ["srv1"])], [1, 0])
    out += _case("test_finds_transitive_agent", [_a("agent1", c, "shared-server", "other-server"), _a("agent2", c, "other-server")],
                 [(["agent1"], ["shared-server"])], [2])
    out += _case("test_transitive_credentials_collected", [_a("agent1", c, "shared-server", ("secret-server", "AWS_SECRET_KEY")),
                                                          _a("agent2", c, ("secret-server", "AWS_SECRET_KEY"))], [(["agent1"], ["shared-server"])], [2])
    out += _case("test_no_infinite_loop", [_a("agent1", c, "srv-a", "srv-b"), _a("agent2", c, "srv-b", "srv-a")], [(["agent1"], ["srv-a"])], [3])
    out += _case("test_hop2_factor", [_a("agent1", c, "srv1", "srv2"), _a("agent2", c, "srv2")], [(["agent1"], ["srv1"], 8.0)], [2])
    out += _case("test_hop3_factor", [_a("agent1", c, "srv1", "srv2"), _a("agent2", c, "srv2", "srv3"), _a("agent3", c, "srv3")],
                 [(["agent1"], ["srv1"], 10.0)], [3])
    out += _case("test_depth_clamped_to_5", [_a("agent1", c, "srv1", "srv2"), _a("agent2", c, "srv2")], [(["agent1"], ["srv1"])], [10])
    out += _case("test_no_transitive_at_depth_1", [_a("a1", c, "shared"), _a("a2", c, "shared")], [(["a1"], ["shared"])], [1])
    out += _case("test_multiple_brs_expanded", [_a("agent1", c, "srv1", "srv2"), _a("agent2", c, "srv2")],
                 [(["agent1"], ["srv1"]), (["agent1"], ["srv1"])], [2])
    return out


def hand_cases():
    out = []
    # A and B share the vulnerable server V: B is reachable only through V, which is never expanded
    out += _case("shared_direct_server", [_a("A", "cursor", "V", "W"), _a("B", "cline", "V"), _a("C", "windsurf", "W", "X"), _a("E", "custom", "X")],
                 [(["A"], ["V"]), (["A", "B"], ["V"]), (["B"], ["V"])], [2, 3, 5])
    # two agents named D: found through X, D takes the first object's type and credentials and expands through the last's Z
    out += _case("duplicate_names", [_a("A", "custom", "V", "X"), _a("D", "cursor", ("X", "X_TOKEN"), ("Y", "Y_SECRET")), _a("F", "cline", "Y"),
                                     _a("D", "windsurf", ("Z", "Z_PASSWORD")), _a("G", "claude-desktop", "Z"), _a("H", "cursor", "X", "Z")],
                 [(["A"], ["V"]), (["D"], ["Y"]), (["G"], ["Z"])], [2, 3, 4, 5])
    out += _case("server_listed_twice", [_a("A", "custom", "V", "S", "S"), _a("B", "cursor", "S", "T", "S"), _a("C", "cline", "T", "T"), _a("D", "cline", "T")],
                 [(["A"], ["V"]), (["B"], ["T"])], [2, 3, 5])
    out += _case("affected_missing", [_a("A", "custom", "V", "S"), _a("B", "cursor", "S")],
                 [(["ghost", "A"], ["V"]), (["ghost"], ["V"]), (["ghost", "ghost2"], ["nowhere"])], [2, 3])
    out += _case("affected_share_server", [_a("A", "custom", "V", "S", "T"), _a("B", "cursor", "V", "S", "U"), _a("C", "cline", "S"), _a("D", "cline", "U", "T"),
                                           _a("E", "windsurf", "T")], [(["A", "B"], ["V"]), (["B", "A"], ["V"]), (["A", "B"], ["V", "S"])], [2, 3, 5])
    out += _case("no_agents", [_a("A", "custom", "V", "S"), _a("B", "cursor", "S")], [([], ["V"]), ([], []), (["A"], ["V"])], [2, 5])
    out += _case("non_ascii", [_a("agënt→1", "custom", "sërver→α", "共有"), _a("エージェント", "cursor", ("共有", "КЛЮЧ_TOKEN")), _a("a→b", "cline", "共有", "→"),
                               _a("😀", "windsurf", "→")], [(["agënt→1"], ["sërver→α"]), (["😀"], ["→"])], [2, 3, 5])
    out += _case("rounding_ties", [_a("A", "custom", "V", "S"), _a("B", "cursor", "S", "T"), _a("C", "cline", "T", "U"), _a("D", "cline", "U", "W"),
                                   _a("E", "windsurf", "W")],
                 [(["A"], ["V"], r) for r in (1.05, 2.15, 0.25, 3.35, 0.45, 0.05, 1.25, 2.5, 7.3, 0.1, 0.15, 9.99)], [2, 3, 4, 5])
    out += _case("repeated_credentials", [_a("A", "custom", "V", "S"), _a("B", "cursor", ("S", "AWS_API_KEY", "GITHUB_TOKEN", "PATH"), ("T", "AWS_API_KEY")),
                                          _a("C", "cline", ("T", "AWS_API_KEY", "DB_PASSWORD"), ("S", "GITHUB_TOKEN"))], [(["A"], ["V"])], [2, 3])
    return out


def main():
    cases = []
    for name, data, depth in reference_test_scenarios() + hand_cases():
        cases.append({"name": name} | run_reference(data, depth))
    for seed, depths in ((11, [0, 1, 2, 3, 4, 5, 10]),):
        data = hops_oracle.fleet(200, seed)
        for d in depths:
            cases.append({"name": f"fleet200_s{seed}@{d}"} | run_reference(data, d))
    data = hops_oracle.clique_fleet(200, 5, clique=20)
    for d in (3, 5):
        cases.append({"name": f"clique200@{d}"} | run_reference(data, d))
    out = ROOT / "tests" / "golden" / "hops"
    out.mkdir(parents=True, exist_ok=True)
    # xz, not gzip: the four blast radii of a signature repeat the same lists far beyond gzip's 32 KiB window (0.34 MB against 8.7 MB)
    with lzma.open(out / "cases.json.xz", "wt", encoding="utf-8", preset=9 | lzma.PRESET_EXTREME) as f:
        json.dump({"source": "unmodified reference expand_blast_radius_hops (scanners/blast_radius.py:16-97)", "cases": cases}, f, ensure_ascii=False)
    print(f"{len(cases)} cases -> {out / 'cases.json.xz'} ({(out / 'cases.json.xz').stat().st_size} bytes)")


def time_reference():
    """The reference on the profile's clique fleets, one process, one core."""
    from agent_bom.scanners.blast_radius import expand_blast_radius_hops

    rows = []
    for n in (1000, 4000):
        data = hops_oracle.clique_fleet(n, 7)
        for d in (2, 3, 5):
            agents, radii = _ref_objects(data)
            t0 = time.perf_counter()
            expand_blast_radius_hops(radii, agents, max_depth=d)
            dt = time.perf_counter() - t0
            ent = sum(len(br.transitive_agents) for br in radii)
            rows.append({"agents": n, "blast_radii": len(radii), "depth": d, "seconds": round(dt, 3), "transitive_entries": ent})
            print(rows[-1], flush=True)
    rec = {"what": "unmodified reference expand_blast_radius_hops on profiles/blast_radius_hops_profile.py's clique fleets (clique_fleet(n, seed=7))",
           "host": "CPU-only build host, one core, CPython 3.12; no GPU involved — not comparable like-for-like with the H100 profile", "rows": rows}
    (ROOT / "profiles" / "blast_radius_hops_reference.json").write_text(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    if "--time" in sys.argv:
        time_reference()
    else:
        main()
