"""Plain-Python statement of the multi-hop blast-radius expansion (reference: scanners/blast_radius.py:16-97).

``expand`` answers from the objects themselves: per blast radius ``None`` (left untouched) or its five fields, with the
credentials sorted.  ``device_arrays`` answers from an ``agent_bom_b200.blast_radius.Encoding`` in the device's result shape
(``HopArrays``), so the host materialisation can be checked without a device.
"""

from __future__ import annotations

from collections import deque

import numpy as np

FACTORS = {1: 1.0, 2: 0.7, 3: 0.5, 4: 0.35, 5: 0.25}


def expand(blast_radii, agents, max_depth: int) -> list[dict | None]:
    depth = max(1, min(max_depth, 5))
    if depth <= 1:
        return [None] * len(blast_radii)
    servers_of: dict[str, list[str]] = {}
    users: dict[str, list] = {}
    for agent in agents:
        servers_of[agent.name] = [s.name for s in agent.mcp_servers]
        for s in agent.mcp_servers:
            users.setdefault(s.name, []).append(agent)
    out: list[dict | None] = []
    for br in blast_radii:
        seen_agents = {a.name for a in br.affected_agents}
        direct = {s.name for s in br.affected_servers}
        seen_servers = set(direct)
        queue: deque = deque()
        for a in br.affected_agents:
            for s in servers_of.get(a.name, ()):
                if s not in direct:
                    queue.append((1, [a.name, s]))
                    seen_servers.add(s)
        found: list[dict] = []
        creds: set[str] = set()
        while queue:
            hop, path = queue.popleft()
            for agent in users.get(path[-1], ()):
                if agent.name in seen_agents:
                    continue
                seen_agents.add(agent.name)
                longer = path + [agent.name]
                found.append({"name": agent.name, "type": agent.agent_type.value, "hop": hop + 1, "chain": "→".join(longer)})
                for s in agent.mcp_servers:
                    creds.update(s.credential_names)
                if hop + 1 < depth:
                    for s in servers_of.get(agent.name, ()):
                        if s not in seen_servers:
                            seen_servers.add(s)
                            queue.append((hop + 1, longer + [s]))
        if not found:
            out.append(None)
            continue
        deepest = max(f["hop"] for f in found)
        out.append({"hop_depth": deepest, "delegation_chain": [f["chain"] for f in found], "transitive_agents": found,
                    "transitive_credentials": sorted(creds), "transitive_risk_score": round(br.risk_score * FACTORS[deepest], 2)})
    return out


def device_arrays(enc, max_depth: int, sigs=None):
    """The device's answer for every signature of ``enc`` (or for ``sigs``, in that order), by a FIFO search over its interned ids."""
    from agent_bom_b200.blast_radius import HopArrays

    ns_off, ns = enc.name_srv_off.tolist(), enc.name_srv.tolist()
    so_off, occ_name = enc.srv_occ_off.tolist(), enc.occ_name.tolist()
    cs_off, cs = enc.cset_off.tolist(), enc.cset_cred.tolist()
    occ_obj = enc.occ_obj.tolist()
    n_first = len(enc.first_srv)
    first_off, first_srv = enc.first_off.tolist(), enc.first_srv.tolist()
    ma_off, ma = enc.mark_agent_off.tolist(), enc.mark_agent.tolist()
    ms_off, ms = enc.mark_srv_off.tolist(), enc.mark_srv.tolist()
    sig_off, d_occ, d_hop, d_par, e_srv, e_par, cred_off, cred = [0], [], [], [], [], [], [0], []
    for s in range(len(enc.sig_members)) if sigs is None else sigs:
        seen_a = set(ma[ma_off[s]:ma_off[s + 1]])
        seen_s = set(ms[ms_off[s]:ms_off[s + 1]])
        queue = deque((1, k, first_srv[k]) for k in range(first_off[s], first_off[s + 1]))
        creds: set[int] = set()
        while queue:
            hop, entry, srv = queue.popleft()
            for o in range(so_off[srv], so_off[srv + 1]):
                n = occ_name[o]
                if n in seen_a:
                    continue
                seen_a.add(n)
                d = len(d_occ)
                d_occ.append(o)
                d_hop.append(hop + 1)
                d_par.append(entry)
                c = occ_obj[o]
                creds.update(cs[cs_off[c]:cs_off[c + 1]])
                if hop + 1 < max_depth:
                    for q in range(ns_off[n], ns_off[n + 1]):
                        if ns[q] not in seen_s:
                            seen_s.add(ns[q])
                            queue.append((hop + 1, n_first + len(e_srv), ns[q]))
                            e_srv.append(ns[q])
                            e_par.append(d)
        sig_off.append(len(d_occ))
        cred.extend(sorted(creds))
        cred_off.append(len(cred))
    return HopArrays(np.asarray(sig_off, np.int64), np.asarray(d_occ, np.int32), np.asarray(d_hop, np.int8), np.asarray(d_par, np.int64), n_first,
                     np.asarray(e_srv, np.int32), np.asarray(e_par, np.int64), np.asarray(cred_off, np.int64), np.asarray(cred, np.int32))


TYPES = ("claude-desktop", "cursor", "windsurf", "cline", "custom")
CRED_POOL = tuple(f"{p}_{k}" for p in ("AWS", "GITHUB", "SLACK", "DB", "OPENAI", "STRIPE") for k in ("API_KEY", "TOKEN", "SECRET", "PASSWORD", "AUTH"))


def _server_data(rng, name: str, creds_of: dict) -> dict:
    if name not in creds_of:
        k = int(rng.integers(0, 3))
        creds_of[name] = [CRED_POOL[int(i)] for i in rng.choice(len(CRED_POOL), size=k, replace=False)]
    return {"name": name, "creds": list(creds_of[name])}


def _radii(rng, agents: list[dict], server_names: list[str]) -> list[dict]:
    """Every server name carries 2 packages x 2 CVEs: four blast radii whose affected agents are the name's users."""
    users: dict[str, list[str]] = {}
    for a in agents:
        for s in a["servers"]:
            users.setdefault(s["name"], []).append(a["name"])
    out = []
    for s in server_names:
        for _ in range(4):
            out.append({"agents": list(users.get(s, ())), "servers": [s], "risk": round(float(rng.uniform(0.5, 10.0)), 1)})
    return out


def fleet(n_agents: int, seed: int) -> dict:
    """Seeded fleet as plain data: every agent has one private server and 3 drawn from a pool of n_agents / 5 shared names."""
    rng = np.random.default_rng(seed)
    pool = [f"shared-{k}" for k in range(max(1, n_agents // 5))]
    creds_of: dict = {}
    agents = []
    for i in range(n_agents):
        names = [f"private-{i}"] + [pool[int(k)] for k in rng.choice(len(pool), size=min(3, len(pool)), replace=False)]
        agents.append({"name": f"agent-{i}", "type": TYPES[int(rng.integers(len(TYPES)))], "servers": [_server_data(rng, n, creds_of) for n in names]})
    return {"agents": agents, "blast_radii": _radii(rng, agents, [f"private-{i}" for i in range(n_agents)] + pool)}


def clique_fleet(n_agents: int, seed: int, clique: int = 50) -> dict:
    """Seeded fleet of cliques: every agent has a private server and its clique's server; the first agent of each clique also
    uses the previous clique's server, so a search from a private server walks back clique by clique (hops 4 and 5 at depth 5)."""
    rng = np.random.default_rng(seed)
    creds_of: dict = {}
    agents = []
    for i in range(n_agents):
        c = i // clique
        names = [f"private-{i}", f"clique-{c}"] + ([f"clique-{c - 1}"] if i % clique == 0 and c else [])
        agents.append({"name": f"agent-{i}", "type": TYPES[int(rng.integers(len(TYPES)))], "servers": [_server_data(rng, n, creds_of) for n in names]})
    n_cliques = (n_agents + clique - 1) // clique
    return {"agents": agents, "blast_radii": _radii(rng, agents, [f"private-{i}" for i in range(n_agents)] + [f"clique-{c}" for c in range(n_cliques)])}
