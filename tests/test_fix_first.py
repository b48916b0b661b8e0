"""CPU-only checks of the fix-first view (graph/fix_first.py) against the unmodified reference's route.

* the focus bytes: on every fixture graph and focus, the device's row predicate evaluated on the bytes ``node_focus`` builds
  (restated here in numpy) gives the reference ``_path_matches_focus`` verdict on every derived path;
* the host predicate gives the reference verdict on every path, persisted ones included;
* the persisted-path branch end to end (it never touches the device): ``fix_first_view`` equals the reference's response;
* card assembly: every golden card is rebuilt from its own attack path.
"""

from __future__ import annotations

import numpy as np
import pytest

from agent_bom_b200 import _lib
from agent_bom_b200.graph import AttackPath, fix_first_view
from agent_bom_b200.graph.fix_first import edge_lookup, fix_first_card, node_focus, path_matches_focus
from fix_first_golden import adopted, cases, focus_kwargs, roundtrip

GRAPH_CASES = cases()


def device_predicate(focus: np.ndarray, need: int, idx: list[int]) -> bool:
    """What rank_keys_kernel decides for a row (agent, server, vulnerable source or the server, finding) — csrc/paths.cuh."""
    a, s, vs, f = idx
    on_hops = (int(focus[a]) | int(focus[s]) | int(focus[vs])) & ~_lib.FOCUS_CVE_FINDING
    on_f = int(focus[f])
    got = on_hops | on_f | (_lib.FOCUS_CVE if on_f & _lib.FOCUS_CVE_FINDING else 0)
    return (got & need) == need


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_focus_bytes_and_host_predicate_match_the_reference_verdicts(case):
    g = adopted(case)
    paths = [AttackPath(**p) for p in case["paths"]]
    assert case["verdicts"]
    for v in case["verdicts"]:
        want = [c == "1" for c in v["match"]]
        assert [path_matches_focus(g, p, **v["focus"]) for p in paths] == want, v["focus"]
        if case["persisted"]:
            continue
        focus, need = node_focus(g, **v["focus"])
        if focus is None:
            assert all(want)
            continue
        assert focus.shape == (g.csr.n_nodes,) and not focus[g.csr.n_real:].any()      # ghosts carry no bits
        for p, w in zip(paths, want):
            h = [g.csr.idx(x) for x in p.hops]
            row = [h[0], h[1], h[2] if len(h) == 4 else h[1], h[-1]]
            assert device_predicate(focus, need, row) == w, (v["focus"], p.hops)


def test_persisted_paths_branch_end_to_end():
    case = next(c for c in GRAPH_CASES if c["name"] == "kat_probe")
    assert case["persisted"]
    g = adopted(case)
    for vc in case["views"]:
        assert roundtrip(fix_first_view(g, **focus_kwargs(vc))) == roundtrip(vc["view"]), vc["focus"]


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["name"] for c in GRAPH_CASES])
def test_card_assembly_for_the_golden_paths(case):
    g = adopted(case)
    index = edge_lookup(g)
    n = 0
    for vc in case["views"]:
        for card in vc["view"]["cards"]:
            p = AttackPath(**card["attack_path"])
            assert roundtrip(fix_first_card(g, p, card["rank"], index)) == roundtrip(card)
            n += 1
    assert n > 0


def test_limit_bounds():
    g = adopted(GRAPH_CASES[0])
    for bad in (0, 26, -1):
        with pytest.raises(ValueError):
            fix_first_view(g, limit=bad)
