"""The device-buffer launches bench.py times, run on bench.py's own schedule and compared exactly with the CPU oracle.

bench.py's ``value`` comes from ``one_step``: per batch ``my[s:e]`` (a slice of one device tensor) the impact walk
(``DeviceWalk.launch`` -> ``abb_walk_launch``) runs on the current stream and the exposure-path count + fill (``DevicePaths``) on a
second stream, into caller-owned arenas sized once by a fitted pass; ``--mode enumerate`` adds a bfs walk and four masked
traverse_subgraph walks after them.  Its parity gate goes through the host API instead (library-owned arenas and stream, re-run
on overflow), so these tests replay that schedule and read every output through ``q_start`` / ``q_count`` (``q_estart`` /
``q_ecount``); they also pin the caller-arena contract of ``DeviceWalk`` and the frontier signatures multi-GPU runs shard by.
Needs a GPU.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import pytest
import torch

from agent_bom_b200 import estate
from agent_bom_b200.engine import DeviceGraph, WalkResult
from agent_bom_b200.graph.schema import N_ENTITY_TYPES
from agent_bom_b200.torch_api import DevicePaths, DeviceWalk, frontier_signatures, shard_by_signature
from bench import DYN, MASKS, MAX_DEPTH, WORKLOADS, device_csr, oracle_graph_from
from golden_util import seeded_graph
from oracle import oracle as orc
from test_gpu_device_paths import assert_rows_equal, hub_graph
from test_gpu_graph_shapes import assert_traverse_equal, assert_walk_equal

pytestmark = pytest.mark.gpu

GRAPHS = ("S", "M1", "seeded", "hub")
EXTRA = ("bfs",) + tuple(f"traverse[{name}]" for name, _, _ in MASKS)       # bench.py's enumerate-mode walks, in its order
L1_CAP = 8                      # dedup.cuh: longest depth-1 frontier a de-duplicated source may have
SIG_INELIGIBLE = 1 << 47        # dedup.cuh: marks a source that is walked on its own; its low bits are its query index
DEDUP_MIN = 256                 # abb200.cu dedup_applies: smallest batch that is de-duplicated
SENTINEL = -0x5A5A5A5B
GUARD = 4096                    # entries past an arena's stated capacity that a launch must leave alone
Q_FIELDS = ("q_start", "q_count", "q_maxd", "q_flags", "q_hist", "q_estart", "q_ecount")
ARENAS = ("nodes", "parent", "depth", "edges")

_graphs: dict = {}
_want: dict = {}


def graph(key):
    """bench.py's S / M1 estate (sources: every finding) or a seeded / hub graph (sources: every node, ghosts included,
    shuffled), built through bench.py's ``device_csr`` and ``oracle_graph_from``."""
    if key not in _graphs:
        if key in WORKLOADS:
            g = estate.generate(WORKLOADS[key][0], 2145, estate.BENCH_KNOBS, exact_rank=False)
            sources = g.findings
        else:
            if key == "hub":
                src, dst, rel, flags, nt, rank = hub_graph()
            else:
                src, dst, rel, flags, nt = seeded_graph(3000, 20000, 7)
                rank = np.random.default_rng(8).permutation(len(nt)).astype(np.int32)
            g = SimpleNamespace(node_type=nt, src=src, dst=dst, rel=rel, flags=flags, node_rank=rank)
            sources = np.random.default_rng(9).permutation(len(nt))
        host = device_csr(g)
        sources = np.ascontiguousarray(sources, dtype=np.int32)
        _graphs[key] = SimpleNamespace(og=oracle_graph_from(host), dg=DeviceGraph.upload(host), rank=g.node_rank, sources=sources,
                                       my=torch.from_numpy(sources).cuda())
    return _graphs[key]


def spec(kind):
    if kind == "impact":
        return DeviceGraph.spec_impact_of(MAX_DEPTH)
    if kind == "bfs":
        return DeviceGraph.spec_bfs(MAX_DEPTH, True)
    _, mask, static = next(m for m in MASKS if kind == f"traverse[{m[0]}]")
    return DeviceGraph.spec_traverse(1, MAX_DEPTH, -1, -1, False, mask, static, False, True)


def want(key, kind, s, e):
    """The oracle's answer for sources[s:e] of graph `key` (exposure-path rows for kind "paths"), as parity_gate computes it."""
    k = (key, kind, s, e)
    if k not in _want:
        g = graph(key)
        f = g.sources[s:e]
        if kind == "impact":
            _want[k] = orc.impact_many(g.og, f, MAX_DEPTH)
        elif kind == "paths":
            _want[k] = orc.derived_paths(g.og, f, g.rank)
        elif kind == "bfs":
            _want[k] = orc.bfs_many(g.og, f, MAX_DEPTH, True)
        else:
            _, mask, static = next(m for m in MASKS if kind == f"traverse[{m[0]}]")
            m = (mask or 0xFFFFFFFF) & (~DYN if static else 0xFFFFFFFF)
            _want[k] = orc.traverse_many(g.og, f, np.arange(e - s + 1, dtype=np.int64), direction=1, max_depth=MAX_DEPTH, rel_mask=m)
    return _want[k]


def oracle_need(w):
    """(node slots, edge slots) the oracle's result takes: a plain launch needs exactly that (traverse slices hold their roots)."""
    return int(w.off[-1]), int(w.eoff[-1]) if w.eoff is not None else 0


def snapshot(w: DeviceWalk, nq: int) -> dict:
    """Copies, ordered on the current stream, of what a caller reads after a launch of `nq` queries."""
    out = {k: getattr(w, k)[: nq * (N_ENTITY_TYPES if k == "q_hist" else 1)].clone() for k in Q_FIELDS if getattr(w, k) is not None}
    out.update({k: getattr(w, k).clone() for k in ARENAS if getattr(w, k) is not None})
    return out


def as_result(snap: dict, nq: int) -> WalkResult:
    h = {k: v.cpu().numpy() for k, v in snap.items()}
    r = WalkResult(start=h["q_start"], count=h["q_count"], maxd=h["q_maxd"], flags=h["q_flags"], nodes=h["nodes"], parent=h.get("parent"),
                   depth=h.get("depth"), estart=h.get("q_estart"), ecount=h.get("q_ecount"), edges=h.get("edges"))
    if "q_hist" in h:
        r.hist = h["q_hist"].reshape(nq, N_ENTITY_TYPES)
    return r


def assert_matches(kind, got: WalkResult, w, what):
    """What parity_gate compares for each walk kind, plus the per-query flags (no root / truncated)."""
    if kind.startswith("traverse"):
        assert_traverse_equal(got, w, what)
        return
    assert_walk_equal(got, w, aux="parent" if kind == "bfs" else None, shift=-1, what=what)
    np.testing.assert_array_equal(got.flags, w.flags, err_msg=f"flags {what}")
    if kind == "impact":
        np.testing.assert_array_equal(got.hist, w.hist, err_msg=f"histograms {what}")


def paths_snapshot(p: DevicePaths, nq: int) -> dict:
    return {"f_off": p.f_off[: nq + 1].clone(), **{k: getattr(p, k).clone() for k in ("hops", "rels", "ncred", "ntool")}}


def paths_rows(snap: dict):
    f_off = snap["f_off"].cpu().numpy()
    r = int(f_off[-1])
    return (f_off, snap["hops"][: 4 * r].view(r, 4).cpu().numpy(), snap["rels"][: 4 * r].view(r, 4).cpu().numpy(),
            snap["ncred"][:r].cpu().numpy(), snap["ntool"][:r].cpu().numpy())


def ragged_batch(n: int) -> int:
    """An odd batch size (so most slices ``my[s:e]`` start off a 16-byte boundary) of at least DEDUP_MIN + 1 queries, such that
    every batch but the last is de-duplicated and the last, ragged one is shorter than DEDUP_MIN and takes the plain tiers."""
    for b in range(max(DEDUP_MIN + 1, n // 5) | 1, n, 2):
        if 32 <= n % b < DEDUP_MIN:
            return b
    raise AssertionError(f"no ragged batch size for {n} sources")


# ── 1 + 2. bench.py's loop: fitted pass, reserve, steps (walk on main, paths on a second stream, enumerate walks after) ────────
def one_step(my, batches, walk, paths, extra, side):
    """bench.py's ``one_step`` (``side`` None: its sequential form), each batch's outputs copied on the main stream before the
    next batch reuses the buffers: the copies are stream-ordered, so the launches are enqueued with no host wait between batches."""
    main = torch.cuda.current_stream()
    out = []
    for s, e in batches:
        if side is not None:
            side.wait_stream(main)
            walk.launch(my[s:e])
            paths.count(my[s:e], stream=side)
            paths.fill(my[s:e], stream=side)
            main.wait_stream(side)
        else:
            walk.launch(my[s:e])
            paths.count(my[s:e])
            paths.fill(my[s:e])
        for _kind, w in extra:
            w.launch(my[s:e])
        out.append((snapshot(walk, e - s), paths_snapshot(paths, e - s), [snapshot(w, e - s) for _kind, w in extra]))
    return out


@pytest.mark.parametrize("dedup,overlap", [pytest.param(True, True, id="dedup-overlap"), pytest.param(False, True, id="plain-overlap"),
                                           pytest.param(True, False, id="dedup-one-stream")])
@pytest.mark.parametrize("key", GRAPHS)
def test_bench_step_matches_oracle(key, dedup, overlap):
    """Every batch of one step, impact walk + exposure-path rows + the five enumerate-mode walks launched back to back on the
    same graph scratch.  The ragged last batch runs on walk and path buffers sized for the larger ones."""
    g = graph(key)
    g.dg.set_dedup(dedup)
    n = len(g.sources)
    batch = ragged_batch(n)
    batches = [(s, min(s + batch, n)) for s in range(0, n, batch)]
    # the arenas start small, so the fitted pass grows each of them at least once
    walk = DeviceWalk(g.dg, spec("impact"), batch, node_cap=1 << 10)
    paths = DevicePaths(g.dg, batch)
    extra = [(kind, DeviceWalk(g.dg, spec(kind), batch, node_cap=1 << 10, edge_cap=1 << 10)) for kind in EXTRA]
    need_nodes = need_rows = 0
    for s, e in batches:
        n_need, _ = walk.launch_fitted(g.my[s:e])
        rows = paths.run_fitted(g.my[s:e])
        need_nodes, need_rows = max(need_nodes, n_need), max(need_rows, rows)
        if not dedup or e - s < DEDUP_MIN:
            assert n_need == oracle_need(want(key, "impact", s, e))[0]
        assert rows == want(key, "paths", s, e).hops.shape[0]
        for kind, w in extra:
            assert w.launch_fitted(g.my[s:e]) == oracle_need(want(key, kind, s, e)), kind
    walk.reserve(need_nodes)
    paths.reserve(need_rows)
    torch.cuda.synchronize()
    got = one_step(g.my, batches, walk, paths, extra, torch.cuda.Stream() if overlap else None)
    torch.cuda.synchronize()
    for (s, e), (w_snap, p_snap, x_snaps) in zip(batches, got):
        what = f"{key} batch [{s}, {e})"
        assert_matches("impact", as_result(w_snap, e - s), want(key, "impact", s, e), f"impact {what}")
        assert_rows_equal(paths_rows(p_snap), want(key, "paths", s, e), g.sources[s:e])
        for kind, snap in zip(EXTRA, x_snaps):
            assert_matches(kind, as_result(snap, e - s), want(key, kind, s, e), f"{kind} {what}")


# ── 3. caller-owned arenas ──────────────────────────────────────────────────────────────────────────────────────────────────
ARENA_CASES = [pytest.param("impact", True, id="impact-dedup"), pytest.param("impact", False, id="impact-plain"),
               pytest.param("bfs", True, id="bfs"), pytest.param("traverse[all]", True, id="traverse-all")]
BIG = 1001                      # a de-duplicated batch for the impact walk when de-duplication is on


def exact_need(kind, dedup, nq):
    """A de-duplicated launch stores each shared slice once, so it needs fewer node slots than the oracle's total."""
    return not (kind == "impact" and dedup and nq >= DEDUP_MIN)


def guard(w: DeviceWalk, node_cap: int, edge_cap: int = 0):
    """Give `w` arenas of `node_cap` / `edge_cap` entries followed by GUARD entries it is not told about, all SENTINEL."""
    def arena(cap):
        return torch.full((cap + GUARD,), SENTINEL, dtype=torch.int32, device=w.q_start.device)

    w.node_cap = node_cap
    w.nodes = arena(node_cap)
    w.parent = arena(node_cap) if w.parent is not None else None
    w.depth = arena(node_cap) if w.depth is not None else None
    if w.q_estart is not None:
        w.edge_cap, w.edges = edge_cap, arena(edge_cap)
    return [(t, cap) for t, cap in ((w.nodes, node_cap), (w.parent, node_cap), (w.depth, node_cap), (w.edges, edge_cap)) if t is not None]


def assert_untouched(guards, what):
    for t, cap in guards:
        bad = int((t[cap:] != SENTINEL).sum())
        assert bad == 0, f"{what}: {bad} entries written past the arena's capacity of {cap}"


@pytest.mark.parametrize("kind,dedup", ARENA_CASES)
def test_short_arena_reports_need_and_stays_in_bounds(kind, dedup):
    """A launch into arenas too small for the batch writes nothing past their capacity and reports the exact need in
    ``needed()``; per-query counts (and histograms) are right even so, and ``launch_fitted`` then gives the oracle's answer."""
    g = graph("S")
    g.dg.set_dedup(dedup)
    roots = g.my[:BIG]
    w_all = want("S", kind, 0, BIG)
    w = DeviceWalk(g.dg, spec(kind), BIG, node_cap=1, edge_cap=1)
    guards = guard(w, 0, 0)
    w.launch(roots)
    need = w.needed()
    assert_untouched(guards, "empty arena")
    if exact_need(kind, dedup, BIG):
        assert need == oracle_need(w_all)
    else:
        assert 0 < need[0] <= oracle_need(w_all)[0] and need[1] == 0
    np.testing.assert_array_equal(w.q_count[:BIG].cpu().numpy(), np.diff(w_all.off))
    if kind == "impact":
        np.testing.assert_array_equal(w.q_hist[: BIG * N_ENTITY_TYPES].view(BIG, -1).cpu().numpy(), w_all.hist)
    # one slot short (the last slice reserved does not fit by one entry), and half the need
    for node_cap, edge_cap in ((need[0] - 1, max(need[1] - 1, 0)), (need[0] // 2, need[1] // 2)):
        what = f"{kind} with arenas of {node_cap} / {edge_cap}"
        guards = guard(w, node_cap, edge_cap)
        w.launch(roots)
        assert w.needed() == need, what
        assert_untouched(guards, what)
        assert w.launch_fitted(roots) == need, what
        assert_untouched(guards, what)
        assert w.node_cap >= need[0] and w.edge_cap >= need[1]
        assert_matches(kind, as_result(snapshot(w, BIG), BIG), w_all, what)


@pytest.mark.parametrize("kind,dedup", ARENA_CASES)
def test_launch_walks_only_the_first_n_queries(kind, dedup):
    """``launch(roots, n_queries=n)`` with a longer roots tensor walks the first n roots only: no per-query output past n and
    no arena entry past the reported need is written, though the buffers have room for every root."""
    g = graph("S")
    g.dg.set_dedup(dedup)
    for n in (BIG, 97):
        roots = g.my[: n + 40]
        w = DeviceWalk(g.dg, spec(kind), n + 40, node_cap=1, edge_cap=1)
        room = oracle_need(want("S", kind, 0, n + 40))
        w.reserve(room[0] + 1, room[1] + 1)
        for k in Q_FIELDS + ARENAS:
            if getattr(w, k) is not None:
                getattr(w, k).fill_(SENTINEL)
        w.launch(roots, n_queries=n)
        need = w.needed()
        w_n = want("S", kind, 0, n)
        if exact_need(kind, dedup, n):
            assert need == oracle_need(w_n)
        for k in Q_FIELDS:
            t = getattr(w, k)
            if t is not None:
                tail = t[n * (N_ENTITY_TYPES if k == "q_hist" else 1):]
                assert bool((tail == SENTINEL).all()), f"{kind}: {k} written past query {n}"
        for k in ARENAS:
            t = getattr(w, k)
            if t is not None:
                assert bool((t[need[1] if k == "edges" else need[0]:] == SENTINEL).all()), f"{kind}: {k} written past the need"
        assert_matches(kind, as_result(snapshot(w, n), n), w_n, f"{kind} n_queries={n} of {n + 40} roots")


@pytest.mark.parametrize("kind,dedup", ARENA_CASES)
def test_walk_reused_for_smaller_batches(kind, dedup):
    """A walk sized by a large batch, reused for smaller ones (one still de-duplicated, one not): every per-query field is the
    smaller batch's own and ``needed()`` counts that launch only."""
    g = graph("S")
    g.dg.set_dedup(dedup)
    w = DeviceWalk(g.dg, spec(kind), BIG, node_cap=1, edge_cap=1)
    w.launch_fitted(g.my[:BIG])
    for s, e in ((2000, 2301), (4000, 4097)):
        w.launch(g.my[s:e])
        w_se = want("S", kind, s, e)
        need = w.needed()
        assert need[0] <= w.node_cap and need[1] <= w.edge_cap
        if exact_need(kind, dedup, e - s):
            assert need == oracle_need(w_se)
        else:
            assert need[0] <= oracle_need(w_se)[0]
        assert_matches(kind, as_result(snapshot(w, e - s), e - s), w_se, f"{kind} [{s}, {e}) after a batch of {BIG}")


# ── 4. frontier signatures and the shards bench.py builds from them ─────────────────────────────────────────────────────────
def restated_frontiers(og, roots):
    """``level1_list`` (dedup.cuh) for the impact spec: per root its ordered, distinct reverse neighbours other than itself, or
    None when the root is walked on its own (an invalid id or a ghost, a reverse row of more than 4 * L1_CAP entries, or more than
    L1_CAP distinct neighbours).  Also returns how many roots are None for the last reason."""
    out, over = [], 0
    for f in roots.tolist():
        if f < 0 or f >= og.n_nodes or og.node_type[f] == orc.GHOST or og.rev_off[f + 1] - og.rev_off[f] > 4 * L1_CAP:
            out.append(None)
            continue
        lst = []
        for v in og.rev_nbr[og.rev_off[f]: og.rev_off[f + 1]].tolist():
            if v != f and v not in lst:
                lst.append(v)
        if len(lst) > L1_CAP:
            lst = None
            over += 1
        out.append(None if lst is None else tuple(lst))
    return out, over


@pytest.mark.parametrize("key", GRAPHS)
def test_frontier_signatures_and_shards(key):
    """Signatures computed on a second stream: equal signatures exactly when the restated frontiers are equal, the individual
    marker with the query index for every other source, and shards that partition the sources without splitting a group."""
    g = graph(key)
    n = len(g.sources)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    sig_dev = frontier_signatures(g.dg, spec("impact"), g.my, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    sig = sig_dev.cpu().numpy()
    fronts, over = restated_frontiers(g.og, g.sources)
    alone = np.array([fr is None for fr in fronts])
    if key in ("seeded", "hub"):
        assert over > 0                     # sources with more than L1_CAP distinct depth-1 neighbours are in the fixture
    q = np.arange(n, dtype=np.int64)
    np.testing.assert_array_equal(sig[alone], SIG_INELIGIBLE | q[alone])
    assert (sig[~alone] >> 47 == 0).all()
    # group id: one per distinct restated frontier; a source walked on its own is a group of one
    ids: dict = {}
    group = np.array([ids.setdefault(fr, len(ids)) if fr is not None else -1 - i for i, fr in enumerate(fronts)], dtype=np.int64)
    pairs = np.unique(np.stack([sig[~alone], group[~alone]]), axis=1).shape[1]
    assert pairs == len(np.unique(sig[~alone])) == len(ids)
    for world in (1, 2, 3, 8):
        owner = np.stack([shard_by_signature(sig_dev, world, r).cpu().numpy() for r in range(world)])
        assert (owner.sum(axis=0) == 1).all(), f"world {world}: not a partition"
        rank = owner.argmax(axis=0)
        assert np.unique(np.stack([group, rank]), axis=1).shape[1] == len(np.unique(group)), f"world {world}: a group is split"
