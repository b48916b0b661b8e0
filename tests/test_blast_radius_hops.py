"""Multi-hop blast-radius expansion on the host (no device): the oracle against the reference's goldens, the encoding and
signature grouping, materialisation from device-shaped arrays, and the paths that never reach the device."""

from __future__ import annotations

import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from agent_bom_b200 import blast_radius as hops  # noqa: E402
from hops_golden import Agent, Radius, Server, fields, load_cases, objects, untouched  # noqa: E402
from oracle import hops_oracle  # noqa: E402

CASES = load_cases()
IDS = [c["name"] for c in CASES]


def _expected(case):
    return [None if e is None else e | {"transitive_credentials": sorted(e["transitive_credentials"])} for e in case["expected"]]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_matches_reference(case):
    agents, radii = objects(case)
    assert hops_oracle.expand(radii, agents, case["depth"]) == _expected(case)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_materialise_from_oracle_arrays(case):
    """The host half of the drop-in, fed the oracle's device-shaped arrays, writes exactly the reference's fields."""
    agents, radii = objects(case)
    depth = hops.clamp_depth(case["depth"])
    if depth > 1:
        enc = hops.encode(radii, agents)
        hops.apply(radii, enc, hops.materialise(enc, hops_oracle.device_arrays(enc, depth)))
    for br, want in zip(radii, _expected(case)):
        if want is None:
            assert untouched(br)
        else:
            assert fields(br) == want


def _dup_fleet():
    agents = [Agent("A", "custom", [Server("V", []), Server("X", [])]),
              Agent("D", "cursor", [Server("X", ["X_TOKEN"]), Server("Y", ["Y_SECRET"])]),
              Agent("D", "windsurf", [Server("Z", ["Z_PASSWORD"]), Server("Z", [])])]
    return agents


def test_encoding_duplicate_name_rules():
    agents = _dup_fleet()
    enc = hops.encode([Radius(["A"], ["V"], 1.0)], agents)
    assert enc.names == ["A", "D"] and enc.servers == ["V", "X", "Y", "Z"]
    # name -> servers: the last object named D wins, duplicates kept
    assert enc.name_srv_off.tolist() == [0, 2, 4] and enc.name_srv.tolist() == [0, 1, 3, 3]
    # server -> occurrences: every (object, server) pair in agents order; X is used by A and the first D
    assert enc.srv_occ_off.tolist() == [0, 1, 3, 4, 6]
    assert enc.occ_name.tolist() == [0, 0, 1, 1, 1, 1] and enc.occ_obj.tolist() == [0, 0, 1, 1, 2, 2]
    assert enc.obj_type == ["custom", "cursor", "windsurf"]
    assert enc.creds == ["X_TOKEN", "Y_SECRET", "Z_PASSWORD"]
    assert enc.cset_off.tolist() == [0, 0, 2, 3] and enc.cset_cred.tolist() == [0, 1, 2]


def test_signature_grouping():
    agents = _dup_fleet()
    radii = [Radius(["A"], ["V"], 1.0), Radius(["A"], ["V", "V"], 2.0), Radius(["A", "ghost"], ["V"], 3.0), Radius(["A"], ["X", "V"], 4.0),
             Radius(["A"], ["V", "X"], 5.0), Radius(["ghost", "A"], ["V"], 6.0), Radius([], [], 7.0)]
    enc = hops.encode(radii, agents)
    # the direct servers are a set, the affected names an ordered tuple
    assert enc.sig_members == [[0, 1], [2], [3, 4], [5], [6]]
    # visited marks: affected names present in agents; direct servers plus the first queue level
    assert enc.mark_agent.tolist() == [0, 0, 0, 0] and enc.mark_agent_off.tolist() == [0, 1, 2, 3, 4, 4]
    assert enc.first_srv.tolist() == [1, 1, 1] and enc.first_root == ["A", "A", "A"]
    assert enc.first_off.tolist() == [0, 1, 2, 2, 3, 3]
    assert enc.mark_srv_off.tolist() == [0, 2, 4, 6, 8, 8] and enc.mark_srv.tolist() == [0, 1, 0, 1, 0, 1, 0, 1]


def test_first_level_deduplicated_in_queue_order():
    agents = [Agent("A", "custom", [Server("V", []), Server("S", []), Server("S", []), Server("T", [])]), Agent("B", "custom", [Server("T", []), Server("U", [])])]
    enc = hops.encode([Radius(["B", "A"], ["V"], 1.0)], agents)
    assert [enc.servers[s] for s in enc.first_srv.tolist()] == ["T", "U", "S"]
    assert enc.first_root == ["B", "B", "A"]


@pytest.mark.parametrize("depth", [1, 0, -3])
def test_depth_at_most_one_touches_nothing_and_needs_no_device(depth, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("the device was reached")

    monkeypatch.setattr(hops, "search", no_device)
    monkeypatch.setattr(hops._lib, "load", no_device)
    agents = [Agent("A", "custom", [Server("V", []), Server("S", [])]), Agent("B", "cursor", [Server("S", ["K_TOKEN"])])]
    br = Radius(["A"], ["V"], 5.0)
    hops.expand_blast_radius_hops([br], agents, max_depth=depth)
    assert untouched(br)


def test_nothing_discovered_leaves_fields_untouched():
    agents = [Agent("A", "custom", [Server("V", []), Server("S", [])]), Agent("B", "cursor", [Server("V", [])])]
    radii = [Radius(["A"], ["V"], 5.0), Radius([], ["V"], 1.0)]
    for br in radii:
        br.hop_depth, br.delegation_chain = 7, ["kept"]
    enc = hops.encode(radii, agents)
    per_sig = hops.materialise(enc, hops_oracle.device_arrays(enc, 3))
    assert per_sig == [None, None]
    hops.apply(radii, enc, per_sig)
    assert all(br.hop_depth == 7 and br.delegation_chain == ["kept"] and br.transitive_agents == [] for br in radii)


def test_each_blast_radius_gets_fresh_containers():
    agents = [Agent("A", "custom", [Server("V", []), Server("S", [])]), Agent("B", "cursor", [Server("S", ["K_TOKEN"])])]
    radii = [Radius(["A"], ["V"], 5.0), Radius(["A"], ["V"], 3.0)]
    enc = hops.encode(radii, agents)
    hops.apply(radii, enc, hops.materialise(enc, hops_oracle.device_arrays(enc, 2)))
    a, b = radii
    assert a.transitive_agents == b.transitive_agents and a.transitive_agents is not b.transitive_agents
    assert a.transitive_agents[0] is not b.transitive_agents[0]
    assert a.delegation_chain is not b.delegation_chain and a.transitive_credentials is not b.transitive_credentials
    assert (a.transitive_risk_score, b.transitive_risk_score) == (3.5, 2.1)


def test_hop_risk_factors():
    assert hops.HOP_RISK_FACTORS == {1: 1.0, 2: 0.7, 3: 0.5, 4: 0.35, 5: 0.25}


@pytest.mark.parametrize("n,seed,depth", [(150, 3, 2), (150, 3, 4), (120, 9, 5)])
def test_oracle_arrays_agree_with_oracle_on_fleets(n, seed, depth):
    data = hops_oracle.fleet(n, seed)
    agents, radii = objects(data)
    want = hops_oracle.expand(radii, agents, depth)
    enc = hops.encode(radii, agents)
    hops.apply(radii, enc, hops.materialise(enc, hops_oracle.device_arrays(enc, depth)))
    for br, w in zip(radii, want):
        assert (untouched(br) if w is None else fields(br) == w)
