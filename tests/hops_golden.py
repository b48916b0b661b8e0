"""Shared helpers of the multi-hop blast-radius tests: the goldens and small duck-typed agents and blast radii built from them.

A case stores plain data: agents (name, type value, servers with the credential names the reference read), blast radii
(affected agent names, affected server names, risk score), the depth, and per blast radius the five fields the reference
wrote, or ``None`` where it left them untouched.
"""

from __future__ import annotations

import json
import lzma
from pathlib import Path

GOLDEN = Path(__file__).resolve().parent / "golden" / "hops" / "cases.json.xz"
FIELDS = ("hop_depth", "delegation_chain", "transitive_agents", "transitive_credentials", "transitive_risk_score")


class AgentType:
    def __init__(self, value: str):
        self.value = value


class Server:
    def __init__(self, name: str, creds: list[str]):
        self.name = name
        self.credential_names = list(creds)


class Agent:
    def __init__(self, name: str, type_value: str, servers: list[Server]):
        self.name = name
        self.agent_type = AgentType(type_value)
        self.mcp_servers = servers


class Named:
    def __init__(self, name: str):
        self.name = name


class Radius:
    def __init__(self, agents: list[str], servers: list[str], risk: float):
        self.affected_agents = [Named(n) for n in agents]
        self.affected_servers = [Named(n) for n in servers]
        self.risk_score = risk
        self.hop_depth = 1
        self.delegation_chain: list = []
        self.transitive_agents: list = []
        self.transitive_credentials: list = []
        self.transitive_risk_score = 0.0


def objects(data: dict) -> tuple[list[Agent], list[Radius]]:
    agents = [Agent(a["name"], a["type"], [Server(s["name"], s["creds"]) for s in a["servers"]]) for a in data["agents"]]
    radii = [Radius(b["agents"], b["servers"], b["risk"]) for b in data["blast_radii"]]
    return agents, radii


def fields(br) -> dict:
    out = {f: getattr(br, f) for f in FIELDS}
    out["transitive_credentials"] = sorted(out["transitive_credentials"])
    return out


def untouched(br) -> bool:
    return (br.hop_depth, br.delegation_chain, br.transitive_agents, br.transitive_credentials, br.transitive_risk_score) == (1, [], [], [], 0.0)


def load_cases() -> list[dict]:
    with lzma.open(GOLDEN, "rt", encoding="utf-8") as f:
        return json.load(f)["cases"]
