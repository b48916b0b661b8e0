"""Multi-hop blast-radius expansion on the H100: every reference golden field by field, seeded fleets against the oracle (300
agents at depths 2-5, 1 000 agents at depths 2 and 3), a 4 000-agent fleet at depth 5 (a seeded sample of 256 signatures in
full, and every signature's discovery count against a sparse reachability count), forced tiny batches, and device memory
returned after the call."""

from __future__ import annotations

import gc
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sp

sys.path.insert(0, str(Path(__file__).resolve().parent))

from agent_bom_b200 import blast_radius as hops  # noqa: E402
from hops_golden import fields, load_cases, objects, untouched  # noqa: E402
from oracle import hops_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = load_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden(case):
    agents, radii = objects(case)
    hops.expand_blast_radius_hops(radii, agents, max_depth=case["depth"])
    for br, want in zip(radii, case["expected"]):
        if want is None:
            assert untouched(br)
        else:
            assert fields(br) == want | {"transitive_credentials": sorted(want["transitive_credentials"])}


def _check_fleet(data, depth, **kw):
    agents, radii = objects(data)
    enc = hops.encode(radii, agents)
    # the oracle answers one blast radius per signature; the others of a signature differ only in their own risk score
    reps = [radii[m[0]] for m in enc.sig_members]
    want = hops_oracle.expand(reps, agents, depth)
    hops.expand_blast_radius_hops(radii, agents, max_depth=depth, **kw)
    n_found = 0
    for members, w in zip(enc.sig_members, want):
        for b in members:
            br = radii[b]
            if w is None:
                assert untouched(br)
                continue
            n_found += 1
            assert fields(br) == w | {"transitive_risk_score": round(br.risk_score * hops.HOP_RISK_FACTORS[w["hop_depth"]], 2)}
    return n_found


@pytest.mark.parametrize("depth", [2, 3, 4, 5])
def test_fleet_300_equals_oracle(depth):
    assert _check_fleet(hops_oracle.fleet(300, 41), depth) > 0


@pytest.mark.parametrize("depth", [2, 3])
def test_fleet_1000_equals_oracle(depth):
    assert _check_fleet(hops_oracle.fleet(1000, 43), depth) > 0


@pytest.mark.parametrize("depth", [3, 5])
def test_clique_fleet_equals_oracle(depth):
    assert _check_fleet(hops_oracle.clique_fleet(400, 44, clique=25), depth) > 0


def _normal(arr, row: int) -> tuple:
    """A signature's discoveries as (occurrence, hop, parent) with the parent named by content: a first-level entry id, or the
    entry's server and the signature-local index of its parent discovery."""
    a, b = int(arr.sig_off[row]), int(arr.sig_off[row + 1])
    out = []
    for i in range(a, b):
        p = int(arr.parent[i])
        if p < arr.n_first:
            key = ("first", p)
        else:
            k = p - arr.n_first
            key = ("entry", int(arr.entry_srv[k]), int(arr.entry_parent[k]) - a)
        out.append((int(arr.occ[i]), int(arr.hop[i]), key))
    return tuple(out), tuple(arr.cred[arr.cred_off[row]:arr.cred_off[row + 1]].tolist())


def _reach_counts(enc, depth: int) -> np.ndarray:
    """Per signature, how many agent names a search to `depth` discovers: level by level over sparse name/server incidence."""
    n_sig, n_names, n_srv = len(enc.sig_members), len(enc.names), len(enc.servers)
    ns = sp.csr_matrix((np.ones(len(enc.name_srv), np.float32), enc.name_srv, enc.name_srv_off), shape=(n_names, n_srv))
    occ_srv = np.repeat(np.arange(n_srv), np.diff(enc.srv_occ_off))
    sn = sp.csr_matrix((np.ones(len(occ_srv), np.float32), (occ_srv, enc.occ_name)), shape=(n_srv, n_names))

    def rows(off, vals, width):
        m = np.zeros((n_sig, width), bool)
        m[np.repeat(np.arange(n_sig), np.diff(off)), vals] = True
        return m

    seen_a = rows(enc.mark_agent_off, enc.mark_agent, n_names)
    seen_s = rows(enc.mark_srv_off, enc.mark_srv, n_srv)
    front = rows(enc.first_off, enc.first_srv, n_srv)
    count = np.zeros(n_sig, np.int64)
    for hop in range(1, depth):
        new = (np.asarray((sn.T @ front.T.astype(np.float32))).T > 0) & ~seen_a
        count += new.sum(1)
        seen_a |= new
        if hop + 1 < depth:
            front = (np.asarray((ns.T @ new.T.astype(np.float32))).T > 0) & ~seen_s
            seen_s |= front
    return count


def test_fleet_4000_depth_5_sampled():
    data = hops_oracle.fleet(4000, 47)
    agents, radii = objects(data)
    enc = hops.encode(radii, agents)
    arr = hops.search(enc, 5)
    n_sig = len(enc.sig_members)
    assert arr.stats["discoveries"] == int(arr.sig_off[-1]) > 1_000_000
    assert np.array_equal(np.diff(arr.sig_off), _reach_counts(enc, 5))
    sample = np.random.default_rng(47).choice(n_sig, size=256, replace=False).tolist()
    want = hops_oracle.device_arrays(enc, 5, sigs=sample)
    for row, s in enumerate(sample):
        assert _normal(arr, s) == _normal(want, row), f"signature {s}"


def test_tiny_batches_identical():
    data = hops_oracle.fleet(300, 53)
    agents, radii = objects(data)
    enc = hops.encode(radii, agents)
    whole = hops.search(enc, 4)
    tiny = hops.search(enc, 4, batch=3)
    assert whole.stats["batches"] == 1 and tiny.stats["batches"] == -(-len(enc.sig_members) // 3)
    per_whole, per_tiny = hops.materialise(enc, whole), hops.materialise(enc, tiny)
    assert per_whole == per_tiny
    assert sum(r is not None for r in per_whole) > 0
    for s in range(len(enc.sig_members)):
        assert _normal(whole, s) == _normal(tiny, s)
    # the drop-in with tiny batches writes the same fields
    a_agents, a_radii = objects(data)
    b_agents, b_radii = objects(data)
    hops.expand_blast_radius_hops(a_radii, a_agents, max_depth=4)
    hops.expand_blast_radius_hops(b_radii, b_agents, max_depth=4, batch=1)
    assert [fields(x) for x in a_radii] == [fields(x) for x in b_radii]


def test_device_memory_returned():
    import torch

    data = hops_oracle.fleet(1000, 59)
    agents, radii = objects(data)
    enc = hops.encode(radii, agents)
    hops.search(enc, 3)                                   # context, module load
    gc.collect()
    free0, _ = torch.cuda.mem_get_info()
    arr = hops.search(enc, 5)
    assert arr.stats["discoveries"] > 0
    del arr
    gc.collect()
    free1, _ = torch.cuda.mem_get_info()
    assert abs(free0 - free1) < (4 << 20)
