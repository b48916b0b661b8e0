"""The kernels that consume the walk's result slices, with root-frontier de-duplication pinned on and off.

Two device kernels write one value per slice entry: ``reach_invert_kernel`` (pass 2a of the dependency reach,
csrc/reach.cuh) and ``subtree_rollup_kernel`` (the sampled bottleneck score, csrc/centrality.cuh).  Under de-duplication
(csrc/dedup.cuh) the members of a frontier group point (q_start, q_count) at the group's one slice, so slices ALIAS and
an output indexed by q_start is shared by every member.  The "shared-frontier fleet" below makes that happen on purpose:
hundreds of agents in groups that USE the same ordered server list.

Every GPU test sets de-duplication (and any tier option) explicitly and puts back what was there before, so the cached
device graphs leave each test as they entered it.
"""

from __future__ import annotations

import contextlib
from collections import deque
from dataclasses import dataclass

import numpy as np
import pytest

from oracle import oracle as orc
from test_gpu_parity import REACH4, SEEDED, VULN_PKG, graphs_for
from test_gpu_tiers import CONFIGS

AGENT, SERVER, PACKAGE, TOOL, VULN, CRED, GHOST = 0, 1, 2, 3, 8, 10, 255
USES, DEPENDS_ON, PROVIDES_TOOL, EXPOSES_CRED, CONTAINS, AFFECTS, VULNERABLE_TO, OWNS = 1, 2, 3, 4, 7, 8, 9, 17
TRAV, BIDIR = 1, 2
L1_CAP = 8          # dedup.cuh: longest frontier a source may have and still share its walk
DEDUP = [pytest.param(True, id="dedup_on"), pytest.param(False, id="dedup_off")]
REACH_KEYS = ("pkg_ids", "pkg_off", "pkg_agents", "pkg_minhop", "vuln_ids", "vuln_poff", "vuln_pkgs", "vuln_aoff", "vuln_agents", "vuln_minhop")


# ── the shared-frontier fleet (plain numpy, no GPU) ─────────────────────────────────────────────────────────────────────
@dataclass
class Fleet:
    src: np.ndarray
    dst: np.ndarray
    rel: np.ndarray
    flags: np.ndarray
    node_type: np.ndarray     # ghosts last
    rank: np.ndarray          # random permutation; ids are spelled so that their string order is exactly this rank
    ids: list
    n_real: int
    agents: np.ndarray        # every agent, in node order
    wide: np.ndarray          # agents with more than L1_CAP passing frontier entries (never share a walk)
    bare: np.ndarray          # agents without a passing edge (empty frontier)
    looped: np.ndarray        # group members that a package of their own shared server CONTAINS (reached back)
    reordered: list           # (server list, same servers in another order) pairs that both got agents

    def doc(self) -> dict:
        """The fleet in the golden-fixture layout, for ``golden_util.graph_from_fixture``."""
        n = self.n_real
        return dict(node_ids=self.ids, n_real=n, node_types=self.node_type[:n].tolist(), node_labels=[""] * n, node_risk=[0.0] * n,
                    node_severity=["none"] * n,
                    edges=np.stack([self.src, self.dst, self.rel, self.flags], axis=1).astype(np.int64).tolist())


def shared_frontier_fleet(seed: int = 5) -> Fleet:
    rng = np.random.default_rng(seed)
    n_srv, layers, per_layer, n_tool, n_cred, n_vuln = 240, 6, 400, 300, 100, 500

    # agents first (the reference's bottleneck sample is the first 50 nodes): plan every agent's ordered server list
    plans: list[list[int]] = []      # per agent: server slots in USES order (-1 = the ghost)
    kinds: list[str] = []
    reordered_lists = []
    for gi in range(44):
        k = int(rng.integers(1, 4))
        servers = [int(s) for s in rng.choice(n_srv, size=k, replace=False)]
        if gi == 7:
            servers = servers[:1] + [-1]                              # a frontier holding an id without a node record
        lists = [servers]
        if k >= 2 and gi % 3 == 0:
            lists.append(servers[::-1])                               # same set, other order: must be a different group
            reordered_lists.append((tuple(servers), tuple(servers[::-1])))
        for lst in lists:
            size = int(rng.integers(2, 41))
            plans.extend([list(lst)] * size)
            kinds.extend(["group"] * size)
    for _ in range(24):                                               # 9..14 distinct servers: ineligible for sharing
        plans.append([int(s) for s in rng.choice(n_srv, size=int(rng.integers(L1_CAP + 1, 15)), replace=False)])
        kinds.append("wide")
    for _ in range(30):                                               # no passing edge at all (some own a credential)
        plans.append([])
        kinds.append("bare")
    order = rng.permutation(len(plans))                               # interleave groups in node order
    plans = [plans[i] for i in order]
    kinds = [kinds[i] for i in order]

    n_agent = len(plans)
    base_srv = n_agent
    base_pkg = base_srv + n_srv
    base_tool = base_pkg + layers * per_layer
    base_cred = base_tool + n_tool
    base_vuln = base_cred + n_cred
    n_real = base_vuln + n_vuln
    ghost = n_real                                                    # two ids without node records, last
    node_type = np.concatenate([np.full(n_agent, AGENT), np.full(n_srv, SERVER), np.full(layers * per_layer, PACKAGE), np.full(n_tool, TOOL),
                                np.full(n_cred, CRED), np.full(n_vuln, VULN), np.full(2, GHOST)]).astype(np.uint8)
    n = len(node_type)

    edges: list[tuple[int, int, int, int]] = []

    def edge(s, d, r, fl=TRAV):
        edges.append((int(s), int(d), int(r), int(fl)))

    def srv(slot):
        return ghost if slot < 0 else base_srv + slot

    def pkg(layer, i):
        return base_pkg + layer * per_layer + i

    # agents: USES in list order; some rows carry filtered entries or repeated neighbours that do not change the frontier
    bare_ids = []
    for a, (lst, kind) in enumerate(zip(plans, kinds)):
        if kind == "bare":
            bare_ids.append(a)
            if a % 2:
                edge(a, base_cred + a % n_cred, OWNS)
            continue
        for j, s in enumerate(lst):
            r = rng.random()
            edge(a, srv(s), USES, TRAV if r > 0.1 else 0)             # non-traversable edges still pass (no traversable filter)
            if kind == "group" and r > 0.85:
                edge(a, base_cred + j, OWNS)                          # not in the reach mask: filtered out of the frontier
            if kind == "group" and r < 0.05:
                edge(a, srv(s), DEPENDS_ON)                           # same neighbour again: de-duplicated in the frontier
    # servers: tools, credentials, and 1..3 packages at a random layer (so package chains below a server are 1..6 deep)
    server_root_pkg = {}
    for s in range(n_srv):
        for _ in range(int(rng.integers(1, 3))):
            edge(base_srv + s, base_tool + int(rng.integers(n_tool)), PROVIDES_TOOL)
        if rng.random() < 0.5:
            edge(base_srv + s, base_cred + int(rng.integers(n_cred)), EXPOSES_CRED)
        for j in range(int(rng.integers(1, 4))):
            p = pkg(int(rng.integers(layers)), int(rng.integers(per_layer)))
            if j == 0:
                server_root_pkg[s] = p
            edge(base_srv + s, p, DEPENDS_ON if rng.random() < 0.7 else CONTAINS, BIDIR | TRAV if rng.random() < 0.05 else TRAV)
    # packages: each layer depends on / contains the next; some edges non-traversable, some bidirectional
    for layer in range(layers - 1):
        for i in range(per_layer):
            for _ in range(int(rng.integers(1, 3))):
                fl = (TRAV if rng.random() > 0.1 else 0) | (BIDIR if rng.random() < 0.05 else 0)
                edge(pkg(layer, i), pkg(layer + 1, int(rng.integers(per_layer))), DEPENDS_ON if rng.random() < 0.7 else CONTAINS, fl)
    edge(pkg(layers - 1, 0), ghost + 1, DEPENDS_ON)
    # a few group members are reached back: a package below their own first server CONTAINS them
    group_agents = [a for a, k in enumerate(kinds) if k == "group" and plans[a][0] >= 0]
    looped = sorted(int(a) for a in rng.choice(group_agents, size=12, replace=False))
    for a in looped:
        edge(server_root_pkg[plans[a][0]], a, CONTAINS)
    # vulnerabilities: AFFECTS (vuln -> package), VULNERABLE_TO (package -> vuln), both, attached to non-packages, or to nothing
    for v in range(n_vuln):
        vid, r = base_vuln + v, rng.random()
        pk = [pkg(int(rng.integers(layers)), int(rng.integers(per_layer))) for _ in range(int(rng.integers(1, 4)))]
        if r < 0.35:
            for p in pk:
                edge(vid, p, AFFECTS, TRAV | (BIDIR if rng.random() < 0.1 else 0))
        elif r < 0.6:
            for p in pk:
                edge(p, vid, VULNERABLE_TO)
        elif r < 0.75:
            edge(vid, pk[0], AFFECTS)
            edge(pk[0], vid, VULNERABLE_TO)
            if len(pk) > 1:
                edge(vid, pk[1], AFFECTS)
        elif r < 0.85:
            edge(vid, base_srv + int(rng.integers(n_srv)), AFFECTS)
            edge(base_tool + int(rng.integers(n_tool)), vid, VULNERABLE_TO)
    # one edge per (source, target, relationship), as UnifiedGraph.add_edge keeps it (the first one's flags win)
    e = np.asarray(edges, dtype=np.int64)
    _, first = np.unique(e[:, :3], axis=0, return_index=True)
    e = e[np.sort(first)]
    rank = rng.permutation(n).astype(np.int32)
    ids = [f"n{int(rank[i]):05d}-{int(node_type[i])}" for i in range(n)]
    agents = np.arange(n_agent, dtype=np.int32)
    reordered = [pair for pair in reordered_lists if list(pair[0]) in plans and list(pair[1]) in plans]
    return Fleet(src=e[:, 0].astype(np.int32), dst=e[:, 1].astype(np.int32), rel=e[:, 2].astype(np.uint8), flags=e[:, 3].astype(np.uint8),
                 node_type=node_type, rank=rank, ids=ids, n_real=n_real, agents=agents,
                 wide=np.asarray([a for a, k in enumerate(kinds) if k == "wide"], dtype=np.int32), bare=np.asarray(bare_ids, dtype=np.int32),
                 looped=np.asarray(looped, dtype=np.int32), reordered=reordered)


def level1_list(og: orc.OracleGraph, f: int, mask: int, real_roots: bool = False):
    """dedup.cuh ``level1_list`` for a forward walk: the ordered, de-duplicated passing neighbours of ``f`` other than ``f``,
    or None when ``f`` cannot share a walk (invalid id, more than 4 * L1_CAP row entries, more than L1_CAP neighbours)."""
    if f < 0 or f >= og.n_nodes or (real_roots and og.node_type[f] == GHOST):
        return None
    a, b = int(og.fwd_off[f]), int(og.fwd_off[f + 1])
    if b - a > 4 * L1_CAP:
        return None
    out: list[int] = []
    for p in range(a, b):
        if not (mask >> (int(og.fwd_meta[p]) & 0x1F)) & 1:
            continue
        v = int(og.fwd_nbr[p])
        if v == f or v in out:
            continue
        if len(out) == L1_CAP:
            return None
        out.append(v)
    return tuple(out)


def frontier_groups(og: orc.OracleGraph, sources, mask: int) -> dict:
    """frontier -> (members, members the group's own walk does NOT reach back); the dependency-reach walk sets no
    REAL_ROOTS flag, so only the id range and the row length decide eligibility."""
    groups: dict = {}
    for f in sources:
        lst = level1_list(og, int(f), mask)
        if lst is not None:
            groups.setdefault(lst, []).append(int(f))
    fronts = list(groups)
    seeds = np.asarray([v for lst in fronts for v in lst], dtype=np.int32)
    w = orc.distances_many(og, seeds, mask)
    out, k = {}, 0
    for lst in fronts:
        reached = set(lst)
        for _ in lst:
            reached.update(w.nodes[int(w.off[k]): int(w.off[k + 1])].tolist())
            k += 1
        out[lst] = (groups[lst], [a for a in groups[lst] if a not in reached])
    return out


_fleet: dict = {}


def fleet() -> Fleet:
    if "fleet" not in _fleet:
        _fleet["fleet"] = shared_frontier_fleet()
    return _fleet["fleet"]


def fleet_oracle_graph() -> orc.OracleGraph:
    if "og" not in _fleet:
        f = fleet()
        _fleet["og"] = orc.build_csr(len(f.node_type), f.src, f.dst, f.rel, f.flags, f.node_type)
    return _fleet["og"]


def test_fleet_frontiers_alias():
    """The fleet really makes the dependency-reach walk share slices: >= 10 frontier groups with two or more members that
    their group's walk does not reach back, next to the other cases the de-duplication has to tell apart."""
    f, og = fleet(), fleet_oracle_graph()
    assert len(f.agents) >= 600
    groups = frontier_groups(og, f.agents, REACH4)
    shared = [lst for lst, (_, kept) in groups.items() if len(kept) >= 2]
    assert len(shared) >= 10, len(shared)
    assert sum(len(groups[lst][1]) for lst in shared) >= 256          # enough sharing agents that every >= 256-agent shard can share too
    assert any(len(lst) == 0 for lst in shared)                       # agents without a passing edge form one empty-frontier group
    assert any(len(lst) >= 2 for lst in shared)
    # the same servers in another order are another frontier
    assert f.reordered
    for a, b in f.reordered:
        fa = tuple(int(x) for x in np.asarray(a) + len(f.agents))
        fb = tuple(int(x) for x in np.asarray(b) + len(f.agents))
        assert fa in groups and fb in groups and set(groups[fa][0]).isdisjoint(groups[fb][0])
    # agents with more than L1_CAP passing neighbours walk alone
    assert len(f.wide) and all(level1_list(og, int(a), REACH4) is None for a in f.wide)
    # members reached back from their own shared server take the individual walk, the rest of their group still shares
    looped = set(f.looped.tolist())
    back = {a for lst, (members, kept) in groups.items() for a in members if a not in kept}
    assert looped <= back
    assert any(len(kept) >= 2 and set(members) & looped for members, kept in groups.values())
    # attachment kinds of the vulnerabilities
    vul = set(np.flatnonzero(f.node_type == VULN).tolist())
    aff = {(int(s), int(d)) for s, d, r in zip(f.src, f.dst, f.rel) if r == AFFECTS and s in vul}
    vto = {(int(d), int(s)) for s, d, r in zip(f.src, f.dst, f.rel) if r == VULNERABLE_TO and d in vul}
    assert aff & vto and aff - vto and vto - aff
    assert any(f.node_type[p] != PACKAGE for _, p in aff | vto)
    assert vul - {v for v, _ in aff | vto}
    assert (f.flags & BIDIR).any() and not (f.flags & TRAV).all() and (f.node_type == GHOST).sum() == 2


def test_fleet_adopts_edge_for_edge():
    """The fleet rebuilt through the package's own model (UnifiedGraph) has the same edge stream, node order and id-string
    ranks, so the oracle's answer on the fleet's arrays is the host API's expected answer."""
    from golden_util import graph_from_fixture

    f = fleet()
    c = graph_from_fixture(f.doc()).csr
    assert c.node_ids == f.ids and c.n_real == f.n_real
    for name in ("src", "dst", "rel", "flags", "node_type", "node_rank"):
        np.testing.assert_array_equal(getattr(c, name), getattr(f, {"node_rank": "rank"}.get(name, name)), err_msg=name)


# ── bottleneck references (no GPU) ───────────────────────────────────────────────────────────────────────────────────────
def reference_bottleneck_counts(og: orc.OracleGraph, sources) -> np.ndarray:
    """graph/container.py:548-567 transcribed: a BFS over the forward adjacency lists in list order, ``visited`` holding
    each reached node's path through its first discoverer; +1 for every node strictly inside a path.  Sources that are
    not recorded nodes (out of range, ghost ids) are skipped: the reference samples its recorded nodes only."""
    off, nbr = og.fwd_off.tolist(), og.fwd_nbr.tolist()
    n = og.n_nodes
    scores = [0] * n
    for src in (int(s) for s in sources):
        if not 0 <= src < n or og.node_type[src] == GHOST:
            continue
        visited = {src: [src]}
        queue = deque([src])
        while queue:
            current = queue.popleft()
            for p in range(off[current], off[current + 1]):
                t = nbr[p]
                if t not in visited:
                    visited[t] = visited[current] + [t]
                    queue.append(t)
        for path in visited.values():
            for node in path[1:-1]:
                scores[node] += 1
    return np.asarray(scores, dtype=np.uint64)


def reference_ranking(counts: np.ndarray, ids: list, n_real: int, top_n: int) -> list:
    """The reference's normalisation and ordering of the transcription's counts (a ghost strictly inside a path is its KeyError)."""
    inside = np.flatnonzero(counts[n_real:])
    if inside.size:
        raise KeyError(ids[n_real + int(inside[0])])
    scores = {ids[i]: float(counts[i]) for i in range(n_real)}
    total = sum(scores.values()) or 1.0
    normalised = {nid: score / total for nid, score in scores.items()}
    return sorted(normalised.items(), key=lambda x: x[1], reverse=True)[:top_n]


def subtree_counts(og: orc.OracleGraph, sources) -> np.ndarray:
    """The same counts at scale: the oracle's unbounded BFS trees (first-discoverer parents), every entry's number of proper
    descendants rolled up with one ``np.add.at`` per depth level from the deepest up, then summed per node."""
    w = orc.bfs_many(og, np.asarray(sources, dtype=np.int32), 2**31 - 1, False)
    T = int(w.off[-1])
    scores = np.zeros(og.n_nodes, dtype=np.uint64)
    if T == 0:
        return scores
    q_of = np.repeat(np.arange(len(w.off) - 1), np.diff(w.off))
    gpar = np.where(w.aux >= 0, w.off[q_of] + w.aux, -1)
    depth = np.where(gpar < 0, 1, 0)
    todo = np.flatnonzero(depth == 0)
    while todo.size:                                  # parents precede their children: one level per round
        pd = depth[gpar[todo]]
        ready = pd > 0
        depth[todo[ready]] = pd[ready] + 1
        todo = todo[~ready]
    desc = np.zeros(T, dtype=np.int64)
    for level in range(int(depth.max()), 1, -1):
        at = np.flatnonzero(depth == level)
        np.add.at(desc, gpar[at], desc[at] + 1)
    np.add.at(scores, w.nodes, desc.astype(np.uint64))
    return scores


def wide_level_graph():
    """A source whose BFS levels 1 and 2 hold 6 000 nodes each (wider than a 1024-thread block); mid i also points at leaf
    i + 1, so leaf i + 1's first discoverer is mid i, not mid i + 1."""
    w = 6000
    root, mid, leaf, tail = 0, np.arange(1, w + 1), np.arange(w + 1, 2 * w + 1), np.arange(2 * w + 1, 2 * w + 51)
    src = np.concatenate([np.full(w, root), mid, mid, leaf])          # mid i lists leaf i before leaf i + 1
    dst = np.concatenate([mid, leaf, np.roll(leaf, -1), tail[np.arange(w) % 50]])
    n = 2 * w + 51
    nt = np.random.default_rng(3).integers(0, 24, size=n).astype(np.uint8)
    return src.astype(np.int32), dst.astype(np.int32), np.full(4 * w, USES, np.uint8), np.full(4 * w, TRAV, np.uint8), nt


def chain_graph(n: int = 3000):
    """A 3 000-node chain (3 000 serial BFS levels), with a few back edges that are scanned but never discover anything."""
    src = np.concatenate([np.arange(n - 1), np.arange(10, n, 97)])
    dst = np.concatenate([np.arange(1, n), np.arange(10, n, 97) - 7])
    ne = len(src)
    nt = np.random.default_rng(4).integers(0, 24, size=n).astype(np.uint8)
    return src.astype(np.int32), dst.astype(np.int32), np.full(ne, DEPENDS_ON, np.uint8), np.full(ne, TRAV, np.uint8), nt


def test_bottleneck_references_agree():
    """The two references are the same function: the reference's path transcription and the per-level subtree roll-up."""
    f, og = fleet(), fleet_oracle_graph()
    rng = np.random.default_rng(8)
    sample = np.concatenate([np.arange(50), rng.integers(0, og.n_nodes, size=30), [-1, og.n_nodes + 5, f.n_real, 3, 3]])
    np.testing.assert_array_equal(subtree_counts(og, sample), reference_bottleneck_counts(og, sample))
    for make, sources in ((chain_graph, [0, 1000, 2999]), (wide_level_graph, [0, 0, 17, 6001])):
        src, dst, rel, fl, nt = make()
        g = orc.build_csr(len(nt), src, dst, rel, fl, nt)
        np.testing.assert_array_equal(subtree_counts(g, sources), reference_bottleneck_counts(g, sources))
    # wide graph: mid 1 discovers leaves 1 and 2, every later mid the next leaf, the last mid none; the first 50 leaves
    # discover the tails
    want = reference_bottleneck_counts(g, [0])
    assert (want[1], want[2], want[5999], want[6000]) == (4, 2, 1, 0)
    assert (want[6001], want[6050], want[6051]) == (1, 1, 0)
    assert subtree_counts(og, np.zeros(0, np.int32)).sum() == 0


# ── device side ──────────────────────────────────────────────────────────────────────────────────────────────────────────
@contextlib.contextmanager
def pinned(dg, dedup: bool, tiers: str | None = None):
    """De-duplication on or off and, optionally, one tier configuration of test_gpu_tiers.CONFIGS; the previous values of
    every option touched are restored on exit."""
    names = ("dedup",) + tuple(CONFIGS["default"])
    before = {k: dg.get_option(k) for k in names}
    try:
        if tiers is not None:
            for k, v in CONFIGS[tiers].items():
                dg.set_option(k, v)
        dg.set_dedup(dedup)
        yield dg
    finally:
        for k, v in before.items():
            dg.set_option(k, v)


_dev: dict = {}


def fleet_device():
    """(oracle graph, device graph, host CSR with the fleet's id strings)."""
    if "fleet" not in _dev:
        from agent_bom_b200.engine import DeviceGraph
        from agent_bom_b200.graph import csr as csrmod

        f = fleet()
        h = csrmod.from_arrays(f.ids, f.node_type, f.src, f.dst, f.rel, f.flags, n_real=f.n_real, node_rank=f.rank)
        _dev["fleet"] = (fleet_oracle_graph(), DeviceGraph.upload(h), h)
    return _dev["fleet"]


def reach_graph(key):
    """(oracle graph, device graph, agents, node rank) for the fleet or a seeded graph of test_gpu_parity."""
    if key == "fleet":
        og, dg, _ = fleet_device()
        return og, dg, fleet().agents, fleet().rank
    og, dg, nt, rank, _ = graphs_for(key)
    return og, dg, np.flatnonzero(nt == AGENT).astype(np.int32), rank


_want: dict = {}


def reach_oracle(key):
    if key not in _want:
        if key == "fleet":
            og, agents, rank = fleet_oracle_graph(), fleet().agents, fleet().rank
        else:
            og, _, agents, rank = reach_graph(key)
        _want[key] = orc.dependency_reach(og, agents, REACH4, VULN_PKG, rank)
    return _want[key]


def assert_reach_equal(got, want, what=""):
    for k in REACH_KEYS:
        np.testing.assert_array_equal(np.asarray(got[k]), np.asarray(want[k]), err_msg=f"{k} {what}")


REACH_GRAPHS = [pytest.param("fleet", id="fleet"), pytest.param(SEEDED[1], id="seeded_2000"), pytest.param(SEEDED[2], id="seeded_6000")]


@pytest.mark.gpu
@pytest.mark.parametrize("tiers", [None, "shrunk", "warp-tiers-only"], ids=["library_tiers", "shrunk", "warp_tiers_only"])
@pytest.mark.parametrize("dedup", DEDUP)
@pytest.mark.parametrize("key", REACH_GRAPHS)
def test_dependency_reach_matches_oracle(key, dedup, tiers):
    """All ten arrays of the dependency reach == the oracle, with the walk sharing slices between agents or not."""
    og, dg, agents, _ = reach_graph(key)
    want = reach_oracle(key)
    with pinned(dg, dedup, tiers):
        got = dg.dependency_reach(agents, REACH4, VULN_PKG)
        stats = dg.last_walk_stats()
    assert stats["queries"] == len(agents)
    if dedup:
        assert 0 < stats["groups"] < stats["eligible"], stats          # agents really shared slices
    else:
        assert stats["groups"] == 0, stats
    assert_reach_equal(got, want)
    assert int(want["pkg_off"][-1]) > 0 and int(want["vuln_aoff"][-1]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("dedup", DEDUP)
def test_dependency_reach_merge_of_shared_frontier_shards(dedup):
    """Agent shards of >= 256 (each de-duplicates on its own) and uneven cuts, merged on the device and on the host by
    dist.merge_dependency_reach == the oracle's unsplit answer."""
    from agent_bom_b200.dist import merge_dependency_reach

    og, dg, agents, rank = reach_graph("fleet")
    want = reach_oracle("fleet")
    n = len(agents)
    assert n >= 3 * 256
    with pinned(dg, dedup):
        for cuts in ([0, 256, 512, n], [0, 1, n // 3, n // 3, n - 300, n]):
            parts = []
            for a, b in zip(cuts, cuts[1:]):
                parts.append(dg.dependency_reach(agents[a:b], REACH4, VULN_PKG))
                stats = dg.last_walk_stats()
                if dedup and b - a >= 256:
                    assert 0 < stats["groups"] < stats["eligible"], (a, b, stats)
            assert_reach_equal(merge_dependency_reach(parts, rank, "cuda:0"), want, f"device merge {cuts}")
            assert_reach_equal(merge_dependency_reach(parts, rank), want, f"host merge {cuts}")


@pytest.mark.gpu
@pytest.mark.parametrize("dedup", DEDUP)
def test_compute_dependency_reach_on_adopted_fleet(dedup):
    """graph.dependency_reach.compute_dependency_reach on a UnifiedGraph built from the fleet through the package's own
    model: every PackageReachability / VulnerabilityReachability equals the oracle's arrays spelled as id strings."""
    from agent_bom_b200.graph import compute_dependency_reach
    from agent_bom_b200.graph.dependency_reach import PackageReachability, VulnerabilityReachability
    from golden_util import graph_from_fixture

    f = fleet()
    want = reach_oracle("fleet")                  # the fleet's ids sort in node-rank order, so the oracle's orders are the reference's
    if "graph" not in _dev:
        _dev["graph"] = graph_from_fixture(f.doc())
    g = _dev["graph"]
    np.testing.assert_array_equal(g.csr.node_rank[: f.n_real], f.rank[: f.n_real])
    ids = f.ids
    with pinned(g.device_graph, dedup):
        rep = compute_dependency_reach(g)
    po, pa, pm = want["pkg_off"], want["pkg_agents"], want["pkg_minhop"]
    packages = {ids[p]: PackageReachability(ids[p], tuple(ids[a] for a in pa[po[i]: po[i + 1]]), int(pm[i]))
                for i, p in enumerate(want["pkg_ids"])}
    vpo, vp, vao, va, vm = want["vuln_poff"], want["vuln_pkgs"], want["vuln_aoff"], want["vuln_agents"], want["vuln_minhop"]
    vulns = {ids[v]: VulnerabilityReachability(ids[v], tuple(ids[p] for p in vp[vpo[i]: vpo[i + 1]]), tuple(ids[a] for a in va[vao[i]: vao[i + 1]]),
                                               int(vm[i]))
             for i, v in enumerate(want["vuln_ids"])}
    assert list(rep.packages.items()) == list(packages.items())
    assert list(rep.vulnerabilities.items()) == list(vulns.items())
    assert [p.min_hop_distance for p in rep.packages.values()] == pm.tolist()
    assert [v.min_hop_distance for v in rep.vulnerabilities.values()] == vm.tolist()
    assert sum(p.reachable for p in rep.packages.values()) > 100 and 0 < len(rep.reachable_vulnerability_ids) < len(vulns)


_bn: dict = {}


def bottleneck_case(case):
    """(oracle graph, device graph, sources, expected raw counts)."""
    if case in _bn:
        return _bn[case]
    if case in ("fleet_700", "empty"):
        og, dg, _ = fleet_device()
        f = fleet()
        rng = np.random.default_rng(31)
        n = og.n_nodes
        ghosts = np.flatnonzero(f.node_type == GHOST)
        sources = np.concatenate([f.agents[:520], rng.integers(0, n, size=150), f.agents[:20], [-1, n + 5], ghosts, np.arange(f.n_real - 8, f.n_real)])
        if case == "empty":
            sources = sources[:0]
        assert case == "empty" or len(sources) > 2 * 132
    elif case == "whole_graph_12":
        og, dg, _, _, _ = graphs_for(SEEDED[3])
        sources = np.random.default_rng(29).integers(0, og.n_nodes, size=12)
    else:
        from agent_bom_b200.engine import DeviceGraph
        from agent_bom_b200.graph import csr as csrmod

        src, dst, rel, fl, nt = wide_level_graph() if case == "wide_level" else chain_graph()
        og = orc.build_csr(len(nt), src, dst, rel, fl, nt)
        dg = DeviceGraph.upload(csrmod.from_arrays(None, nt, src, dst, rel, fl))
        sources = [0, 0, 17, 6001, 12005] if case == "wide_level" else [0, 1000, 2999, 1500, 1]
    sources = np.asarray(sources, dtype=np.int32)
    want = subtree_counts(og, sources)
    if case == "whole_graph_12":
        w = orc.bfs_many(og, sources, 2**31 - 1, False)
        assert int(np.diff(w.off).max()) > 20000                     # whole-graph walks: through G1 to GX
    if case == "wide_level":
        w = orc.bfs_many(og, sources[:1], 2**31 - 1, False)
        assert (w.aux >= 0).sum() > 5000                              # one BFS level wider than the block
    _bn[case] = (og, dg, sources, want)
    return _bn[case]


@pytest.mark.gpu
@pytest.mark.parametrize("tiers", ["default", "warp-tiers-only", "shrunk"])
@pytest.mark.parametrize("case", ["fleet_700", "wide_level", "chain_3000", "whole_graph_12", "empty"])
def test_bottleneck_scores_match_subtree_sizes(case, tiers):
    """Raw bottleneck scores == the per-level subtree roll-up of the oracle's BFS trees, bit-identical with de-duplication on
    and off: a change that lets these PARENTS walks share slices (whose roll-up scratch would then be shared too) fails here."""
    og, dg, sources, want = bottleneck_case(case)
    got = {}
    for dedup in (True, False):
        with pinned(dg, dedup, tiers):
            got[dedup] = dg.bottleneck_scores(sources)
    np.testing.assert_array_equal(got[True], got[False])
    np.testing.assert_array_equal(got[True], want)
    assert got[True].dtype == np.uint64 and (case == "empty") == (int(want.sum()) == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("dedup", DEDUP)
@pytest.mark.parametrize("case", ["fleet_sample", "wide_level", "chain_3000"])
def test_bottleneck_scores_match_reference_semantics(case, dedup):
    """Raw scores == the transcription of the reference's path loop, and ``rank_bottlenecks`` == its normalised, sorted list."""
    from agent_bom_b200.backend import rank_bottlenecks

    if case == "fleet_sample":
        og, dg, h = fleet_device()
        sources = np.arange(50, dtype=np.int32)                       # the reference's own sample: the first 50 nodes
        ids, n_real = fleet().ids, fleet().n_real
    else:
        from agent_bom_b200.graph import csr as csrmod

        og, dg, _, _ = bottleneck_case(case)
        sources = np.asarray([0, 0, 17] if case == "wide_level" else [0, 1000], dtype=np.int32)
        ids, n_real = [f"v{i:05d}" for i in range(og.n_nodes)], og.n_nodes
        h = csrmod.from_arrays(ids, og.node_type, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    want = reference_bottleneck_counts(og, sources)
    with pinned(dg, dedup):
        got = dg.bottleneck_scores(sources)
    np.testing.assert_array_equal(got, want)
    for top in (5, 20, n_real):
        assert rank_bottlenecks(h, got, top) == reference_ranking(want, ids, n_real, top)
