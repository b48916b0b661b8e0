"""Root-frontier de-duplication's fallbacks (dedup.cuh, ``enqueue_dedup_walk``), forced on purpose and compared with the oracle.

A single-source walk batch of 256 or more queries is grouped by a 47-bit signature of each source's level-1 frontier S'; one
canonical walk per group is seeded with S' and its members share its slice.  Three fallbacks send a source to an individual walk
instead, and each must be right for the shared answers to be right:

1. a member whose S' differs from its group head's (a signature collision: state 1 in ``dedup_members_kernel``);
2. a member whose own source the canonical walk reaches (state 2, marked inside the walk tiers, only for state-0 members);
3. an ineligible source: an invalid id, a ghost (specs with real roots), a row of more than 4 * L1_CAP entries, or more than
   L1_CAP distinct neighbours.

The fixture is a small index-space graph whose sources sit on the colliding frontier pairs of test_dedup_signatures.py: several
sources per frontier, interleaved so that in some groups the head has the pair's first frontier and in others its second, sources
that their own group's walk reaches through a cycle, sources of one frontier that the other frontier's walk reaches (a state-1
member that would also qualify for state 2), a heavy pair whose canonical walk S1 hands to the big block tier, and the
eligibility edges (rows of 32 and 33 entries, 8 and 9 distinct neighbours, a self-loop, parallel edges, empty frontiers, ghosts,
ids -1 and n, a repeated root).  Every walk kind that de-duplicates runs through the host walk (copies and zero-copy), the chunked
host walk and the caller-arena launch bench.py times, with de-duplication on and off and the big block tier on and off.  Results
must equal the oracle's individual walks, and ``last_walk_stats`` and the caller arena's need are pinned exactly to a
restatement of the grouping.  Needs a GPU.
"""

from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from agent_bom_b200.engine import DeviceGraph, WalkResult
from agent_bom_b200.graph import csr as gcsr
from agent_bom_b200.graph.schema import N_ENTITY_TYPES
from agent_bom_b200.torch_api import DeviceWalk, frontier_signatures, shard_by_signature
from oracle import oracle as orc
from test_dedup_signatures import COLLISIONS, SIG_INELIGIBLE, frontier_signature
from test_gpu_graph_shapes import assert_walk_equal

pytestmark = pytest.mark.gpu

L1_CAP = 8                      # dedup.cuh: longest frontier a grouped source may have; its raw row may hold 4 * L1_CAP entries
DEDUP_MIN = 256                 # abb200.cu dedup_applies: smallest batch that is de-duplicated
GHOST = 255
FWD, REV = 1, 2                 # walk directions (ABB_DIR_*)
N = 12288
SRC0, SRC_END = 8192, 9216      # designed sources take ids from SRC0; every other id is background
REL_KEEP, REL_DROP = 1, 5       # REL_DROP edges are also non-traversable: both filtered specs skip them
DIST_MASK = 0xFFFFFFFF & ~(1 << REL_DROP)
HEAVY = 300                     # neighbours of one frontier node: more candidates than S1's 256-entry queue
REV_PAIRS, FWD_PAIRS = COLLISIONS[:4], COLLISIONS[4:]
RAW_FWD = 2                     # FWD_PAIRS[:2] collide under every forward spec; the rest only once REL_DROP edges are filtered out


@dataclass(frozen=True)
class Case:
    direction: int
    depth: int                  # -1: unbounded
    trav: bool = False
    rel_mask: int = 0xFFFFFFFF
    real_roots: bool = True
    kind: str = "impact"

    @property
    def mode(self) -> str:
        """Which designed frontier the case's sources should have: reverse rows, raw forward rows or filtered forward rows."""
        if self.direction == REV:
            return "rev"
        return "filt" if self.trav or self.rel_mask != 0xFFFFFFFF else "raw"

    def spec(self):
        if self.kind == "impact":
            return DeviceGraph.spec_impact_of(self.depth)
        if self.kind == "reachable":
            return DeviceGraph.spec_reachable_from(self.depth, self.trav)
        return DeviceGraph.spec_distances(self.rel_mask)

    def oracle(self, og, roots):
        if self.kind == "impact":
            return orc.impact_many(og, roots, self.depth)
        if self.kind == "reachable":
            return orc.reachable_many(og, roots, self.depth, self.trav)
        return orc.distances_many(og, roots, self.rel_mask)


CASES = {
    "impact-d1": Case(REV, 1),             # the canonical walks have depth 0: nothing can reach a member's source
    "impact-d2": Case(REV, 2),
    "impact-d4": Case(REV, 4),
    "reachable": Case(FWD, 4, kind="reachable"),
    "reachable-trav": Case(FWD, 4, trav=True, kind="reachable"),
    "distances-mask": Case(FWD, -1, rel_mask=DIST_MASK, real_roots=False, kind="distances"),
}


# ── fixture ─────────────────────────────────────────────────────────────────────────────────────────────────────────────────
class Builder:
    """Edge stream of the fixture.  A source's row for a direction lists its neighbours in edge order, so rows are written by
    adding their edges in the order wanted; background edges never touch a designed source."""

    def __init__(self, rng):
        self.rng = rng
        self.src, self.dst, self.rel, self.flags = [], [], [], []
        self.next_source = SRC0
        frontier = {v for f1, f2 in COLLISIONS for v in f1 + f2}
        self.pool = np.array([v for v in list(range(SRC0)) + list(range(SRC_END, N)) if v not in frontier], dtype=np.int64)
        self.free = iter(rng.permutation(self.pool).tolist())
        self.intended: dict = {}            # (mode, source) -> its S' (None: ineligible)
        self.roles: dict = {}               # source -> (pair tag, side, kind) for collision sources

    def source(self) -> int:
        s = self.next_source
        self.next_source += 1
        assert s < SRC_END
        return s

    def fresh(self, k: int = 1) -> list[int]:
        return [next(self.free) for _ in range(k)]

    def edge(self, u, v, keep=True):
        self.src.append(u)
        self.dst.append(v)
        self.rel.append(REL_KEEP if keep else REL_DROP)
        self.flags.append(gcsr.EDGE_TRAVERSABLE if keep else 0)

    def row(self, s, nbrs, direction, keep=None):
        for i, v in enumerate(nbrs):
            k = True if keep is None else keep[i]
            if direction == REV:
                self.edge(v, s, k)
            else:
                self.edge(s, v, k)

    def reach(self, u, s, direction):
        """Make source s one hop from u for a walk in `direction` (s's own row in that direction is unchanged)."""
        if direction == REV:
            self.edge(s, u)
        else:
            self.edge(u, s)

    def intend(self, direction, s, raw, filtered=None):
        if direction == REV:
            self.intended[("rev", s)] = raw
        else:
            self.intended[("raw", s)] = raw
            self.intended[("filt", s)] = raw if filtered is None else filtered


def background(b: Builder):
    """A sparse random graph over the background ids (collision frontier nodes included) with mixed relationships and
    traversability, and the heavy frontier nodes' HEAVY in- (reverse pairs) or out-neighbours (forward pairs)."""
    rng = b.rng
    pool = np.concatenate([b.pool, np.array([v for f1, f2 in COLLISIONS for v in f1 + f2])])
    for u in rng.permutation(pool).tolist():
        for v in rng.choice(pool, size=rng.choice(4, p=[0.3, 0.35, 0.25, 0.1])).tolist():
            b.src.append(u)
            b.dst.append(v)
            b.rel.append(int(rng.choice([1, 2, 3, REL_DROP])))
            b.flags.append(gcsr.EDGE_TRAVERSABLE if rng.random() < 0.7 else 0)
    for v in rng.choice(b.pool, size=HEAVY, replace=False).tolist():
        b.edge(v, REV_PAIRS[0][0][0])
    for v in rng.choice(b.pool, size=HEAVY, replace=False).tolist():
        b.edge(FWD_PAIRS[0][0][0], v)


def collision_sources(b: Builder, direction, pairs, filtered_from: int) -> list[list[int]]:
    """Per pair, five sources on each frontier: three plain, one its own frontier's walk reaches in one hop ("own"), one the
    other frontier's walk reaches ("cross").  Pairs from `filtered_from` on give each source a leading REL_DROP edge to a node of
    its own, so their raw rows differ and only the filtered frontiers collide.  Even pairs list a first-frontier source first."""
    out = []
    for i, (f1, f2) in enumerate(pairs):
        filt = i >= filtered_from
        sides = ([], [])
        for side, (fr, other) in enumerate(((f1, f2), (f2, f1))):
            for kind in ("plain", "own", "plain", "cross", "plain"):
                s = b.source()
                if filt:
                    x = b.fresh()[0]
                    b.row(s, (x,) + fr, direction, keep=(False, True, True))
                    b.intend(direction, s, (x,) + fr, fr)
                else:
                    b.row(s, fr, direction)
                    b.intend(direction, s, fr)
                if kind == "own":
                    b.reach(fr[1], s, direction)
                elif kind == "cross":
                    b.reach(other[0], s, direction)
                b.roles[s] = ((direction, i), side, kind)
                sides[side].append(s)
        first, second = sides if i % 2 == 0 else sides[::-1]
        out.append([v for ab in zip(first, second) for v in ab])
    return out


def eligibility_sources(b: Builder, direction) -> list[int]:
    out = []

    def add(nbrs, intended, **kw):
        s = b.source()
        b.row(s, [s if v == "self" else v for v in nbrs], direction, **kw)
        b.intend(direction, s, intended)
        out.append(s)
        return s

    p = b.fresh(9)
    add(p[:4] * 8, tuple(p[:4]))                        # 32 entries, 4 distinct: eligible
    add(p[:8] * 4, tuple(p[:8]))                        # 32 entries, exactly L1_CAP distinct
    add(p[:8], tuple(p[:8]))                            # the same frontier from an 8-entry row: a legitimate group of two
    q = b.fresh(9)
    add(q + q[:1] * 23, None)                           # 32 entries, L1_CAP + 1 distinct
    add(q[:2] * 16 + q[:1], None)                       # 33 entries, 2 distinct: the row is too long
    add(q, None)                                        # 9 entries, L1_CAP + 1 distinct
    r = b.fresh(2)
    add([r[0], "self", r[1]], tuple(r))                 # a self-loop is not part of S'
    add([r[0], r[0], r[1]], tuple(r))                   # parallel edges: listed once; same S' as the self-loop source
    for _ in range(3):
        add([], ())                                     # empty frontier: a valid source that reaches nothing
    return out


def ghost_source(b: Builder, direction, nt) -> int:
    s = b.source()
    nbrs = b.fresh(2)
    b.row(s, nbrs, direction)
    nt[s] = GHOST
    return s


def filtered_twins(b: Builder) -> list[int]:
    """Two forward sources with different raw rows and the same filtered frontier: they share a group under the filtered specs."""
    c, d, y1, y2 = b.fresh(4)
    s1, s2 = b.source(), b.source()
    b.row(s1, (y1, c, d), FWD, keep=(False, True, True))
    b.row(s2, (c, y2, d), FWD, keep=(True, False, True))
    b.intend(FWD, s1, (y1, c, d), (c, d))
    b.intend(FWD, s2, (c, y2, d), (c, d))
    return [s1, s2]


def merge(lists):
    """Round-robin merge that keeps each list's order."""
    out, k = [], 0
    while any(k < len(x) for x in lists):
        out += [x[k] for x in lists if k < len(x)]
        k += 1
    return out


_fx: dict = {}


def fixture():
    if "fx" not in _fx:
        rng = np.random.default_rng(20260)
        b = Builder(rng)
        nt = rng.integers(0, N_ENTITY_TYPES, size=N).astype(np.uint8)
        background(b)
        rev = collision_sources(b, REV, REV_PAIRS, len(REV_PAIRS))
        fwd = collision_sources(b, FWD, FWD_PAIRS, RAW_FWD)
        designed = merge(rev + fwd)
        designed += merge([eligibility_sources(b, REV), eligibility_sources(b, FWD)]) + filtered_twins(b)
        ghosts = [ghost_source(b, REV, nt), ghost_source(b, FWD, nt)]
        designed += [-1, ghosts[0], N, ghosts[1], designed[0], designed[3], designed[0]]          # invalid ids, ghosts, repeats
        bg = rng.choice(b.pool, size=760 - len(designed), replace=False).tolist()
        batch = np.array(designed + bg, dtype=np.int32)
        host = gcsr.from_arrays(None, nt, b.src, b.dst, b.rel, b.flags)
        og = orc.build_csr(N, np.array(b.src), np.array(b.dst), np.array(b.rel), np.array(b.flags), nt)
        _fx["fx"] = SimpleNamespace(host=host, og=og, dg=DeviceGraph.upload(host), nt=nt, batch=batch, intended=b.intended, roles=b.roles,
                                    ghosts=ghosts, n_designed=len(designed), cache={})
    return _fx["fx"]


# ── restatement of the grouping ─────────────────────────────────────────────────────────────────────────────────────────────
def level1(host, case: Case, f: int):
    """``level1_list`` (dedup.cuh): f's ordered, distinct passing neighbours other than itself, or None when f is walked alone."""
    if f < 0 or f >= host.n_nodes or (case.real_roots and host.node_type[f] == GHOST):
        return None
    off, nbr, meta = (host.fwd_off, host.fwd_nbr, host.fwd_meta) if case.direction == FWD else (host.rev_off, host.rev_nbr, host.rev_meta)
    a, b = int(off[f]), int(off[f + 1])
    if b - a > 4 * L1_CAP:
        return None
    out: list[int] = []
    for m, v in zip(meta[a:b].tolist(), nbr[a:b].tolist()):
        if not (case.rel_mask >> (m & 0x1F)) & 1 or (case.trav and not m & 0x20) or v == f or v in out:
            continue
        if len(out) == L1_CAP:
            return None
        out.append(v)
    return tuple(out)


def passing_adjacency(host, case: Case):
    off, nbr, meta = (host.fwd_off, host.fwd_nbr, host.fwd_meta) if case.direction == FWD else (host.rev_off, host.rev_nbr, host.rev_meta)
    row = np.repeat(np.arange(host.n_nodes), np.diff(off.astype(np.int64)))
    m = meta.astype(np.int64)
    keep = ((case.rel_mask >> (m & 0x1F)) & 1).astype(bool)
    if case.trav:
        keep &= (m & 0x20) != 0
    return sp.csr_matrix((np.ones(int(keep.sum()), dtype=np.int8), (row[keep], nbr[keep].astype(np.int64))), shape=(host.n_nodes, host.n_nodes))


def ball(adj, seeds, limit: int) -> np.ndarray:
    """Visited set of a walk seeded with `seeds` that expands nodes shallower than `limit` (-1: no limit)."""
    vis = np.zeros(adj.shape[0], dtype=bool)
    front = np.unique(np.asarray(seeds, dtype=np.int64))
    vis[front] = True
    depth = 0
    while front.size and (limit < 0 or depth < limit):
        nxt = np.unique(adj[front].indices)
        front = nxt[~vis[nxt]]
        vis[front] = True
        depth += 1
    return vis


def restate(fx, name: str, nq: int):
    """What the de-duplicated launch of batch[:nq] must do: signatures, statistics, node slots, and what the fixture covers."""
    key = (name, nq)
    if key in fx.cache:
        return fx.cache[key]
    case = CASES[name]
    roots = fx.batch[:nq]
    want = case.oracle(fx.og, roots)
    fr = [level1(fx.host, case, int(f)) for f in roots]
    sig = np.array([SIG_INELIGIBLE | q if fr[q] is None else frontier_signature(fr[q]) for q in range(nq)], dtype=np.int64)
    adj = passing_adjacency(fx.host, case)
    limit = case.depth - 1 if case.depth > 0 else -1
    eligible = [q for q in range(nq) if fr[q] is not None]
    head: dict = {}
    vis: dict = {}
    state = np.full(nq, -1)
    need = 0
    for q in sorted(eligible, key=lambda q: (int(sig[q]), q)):          # the stable radix sort: ties keep query order
        h = head.setdefault(int(sig[q]), q)
        if h == q:
            vis[h] = ball(adj, fr[q], limit)
            need += int(vis[h].sum())                                   # the canonical slice holds S' and all it reaches
        if fr[q] != fr[h]:
            state[q] = 1
        else:
            state[q] = 2 if vis[h][roots[q]] else 0
    individual = np.flatnonzero(state != 0)                             # ineligible (-1), collision (1), reached (2)
    need += int(np.diff(want.off)[individual].sum())
    in_ball = [q for q in np.flatnonzero(state == 1) if vis[head[int(sig[q])]][roots[q]]]
    r = SimpleNamespace(
        want=want, fr=fr, sig=sig, state=state, head=head, need=need, in_ball=in_ball,
        stats={"queries": nq, "groups": len(head), "individual": len(individual), "eligible": len(eligible)},
    )
    fx.cache[key] = r
    return r


# ── comparisons ─────────────────────────────────────────────────────────────────────────────────────────────────────────────
def assert_equal(case: Case, got: WalkResult, want, what: str):
    assert_walk_equal(got, want, aux="depth" if case.kind == "distances" else None, what=what)
    np.testing.assert_array_equal(got.flags, want.flags, err_msg=f"flags {what}")
    if case.kind == "impact":
        np.testing.assert_array_equal(got.hist, want.hist, err_msg=f"histograms {what}")


def device_result(w: DeviceWalk, nq: int) -> WalkResult:
    r = WalkResult(start=w.q_start[:nq].cpu().numpy(), count=w.q_count[:nq].cpu().numpy(), maxd=w.q_maxd[:nq].cpu().numpy(),
                   flags=w.q_flags[:nq].cpu().numpy(), nodes=w.nodes.cpu().numpy(), depth=None if w.depth is None else w.depth.cpu().numpy())
    if w.q_hist is not None:
        r.hist = w.q_hist[: nq * N_ENTITY_TYPES].view(nq, N_ENTITY_TYPES).cpu().numpy()
    return r


def expected_stats(r, nq: int, dedup: bool) -> dict:
    if dedup and nq >= DEDUP_MIN:
        return r.stats
    return {"queries": nq, "groups": 0, "individual": 0, "eligible": 0}


# ── 1. the fixture holds what it is meant to ────────────────────────────────────────────────────────────────────────────────
@pytest.mark.parametrize("name", CASES)
def test_fixture_frontiers_are_the_intended_ones(name):
    """Rows read back as the frontiers they were built to be, and the grouping restated for the full batch contains every
    fallback: collisions with either frontier at the head, own sources reached, collision members the head's walk reaches."""
    fx = fixture()
    case = CASES[name]
    r = restate(fx, name, len(fx.batch))
    checked = set()
    for q, f in enumerate(fx.batch[: fx.n_designed].tolist()):
        if (case.mode, f) in fx.intended:
            assert r.fr[q] == fx.intended[(case.mode, f)], f"source {f}: S' {r.fr[q]} is not the intended {fx.intended[(case.mode, f)]}"
            checked.add(f)
    assert checked == {f for mode, f in fx.intended if mode == case.mode}
    assert r.fr[fx.batch.tolist().index(-1)] is None and r.fr[fx.batch.tolist().index(N)] is None
    for g in fx.ghosts:
        assert (r.fr[fx.batch.tolist().index(g)] is None) == case.real_roots
    # both orders of every colliding pair that collides under this spec, and the fallbacks the pair's sources are built for
    heads = set()
    for q in np.flatnonzero(r.state == 1).tolist():
        h = r.head[int(r.sig[q])]
        role_h, role_q = fx.roles[int(fx.batch[h])], fx.roles[int(fx.batch[q])]
        assert role_h[0] == role_q[0] and role_h[1] != role_q[1], "only the designed pairs collide"
        heads.add((role_h[0], role_h[1]))
    colliding = {(case.direction, i) for i in range(len(REV_PAIRS) if case.mode == "rev" else (RAW_FWD if case.mode == "raw" else len(FWD_PAIRS)))}
    assert {p for p, _ in heads} == colliding
    assert {side for _, side in heads} == {0, 1}
    assert sum(f is None for f in r.fr) >= 5 + 2 * case.real_roots          # ids -1 and n, three over-long rows (+ the ghosts)
    if case.depth == 1:
        assert not (r.state == 2).any() and not r.in_ball
    else:
        assert (r.state == 2).sum() >= len(colliding) and len(r.in_ball) >= len(colliding)
    assert () in r.fr


# ── 2. device signatures and shards ─────────────────────────────────────────────────────────────────────────────────────────
@pytest.mark.parametrize("name", CASES)
def test_device_signatures_equal_the_restated_hash(name):
    fx = fixture()
    case = CASES[name]
    r = restate(fx, name, len(fx.batch))
    roots = torch.from_numpy(fx.batch).cuda()
    sig_dev = frontier_signatures(fx.dg, case.spec(), roots)
    sig = sig_dev.cpu().numpy()
    bad = np.flatnonzero(sig != r.sig)
    assert bad.size == 0, (f"{name}: the device's frontier signature differs from the restated hash for {bad.size} sources (first: query "
                           f"{bad[0]}, device {sig[bad[0]]:#x}, restated {r.sig[bad[0]]:#x}); if dedup.cuh's hash changed on purpose, "
                           f"regenerate the collision constants with oracle/make_signature_collisions.py")
    for world in (2, 3, 8):
        owner = np.stack([shard_by_signature(sig_dev, world, k).cpu().numpy() for k in range(world)])
        assert (owner.sum(axis=0) == 1).all(), f"world {world}: not a partition"
        rank = owner.argmax(axis=0)
        for q in np.flatnonzero(r.state == 1).tolist():
            h = r.head[int(r.sig[q])]
            assert rank[q] == rank[h], f"world {world}: a colliding group is split across ranks"


# ── 3. every entry point against the oracle, statistics pinned ──────────────────────────────────────────────────────────────
@pytest.mark.parametrize("tiers", [2, 0], ids=["big-tier", "warp-tiers"])
@pytest.mark.parametrize("name", CASES)
def test_fallbacks_equal_the_oracle(name, tiers):
    """Host walk (copies, and zero-copy into pinned memory), chunked host walk and caller-arena launch, de-duplication on and off,
    batches of the fixture's full size, 256 and 255: the oracle's answer every time, exact sharing statistics, and (caller arena)
    exactly the node slots the canonical and individual slices take."""
    fx = fixture()
    case = CASES[name]
    dg = fx.dg
    spec = case.spec()
    try:
        dg.set_option("block_tiers", tiers)
        for nq in (len(fx.batch), DEDUP_MIN, DEDUP_MIN - 1):
            r = restate(fx, name, nq)
            roots = fx.batch[:nq]
            roots_dev = torch.from_numpy(np.ascontiguousarray(roots)).cuda()
            for dedup in (True, False):
                dg.set_dedup(dedup)
                what = f"{name} block_tiers={tiers} nq={nq} dedup={dedup}"
                for zc in (False, True, True):             # the second zero-copy call writes into a pinned arena sized by the first
                    dg.set_option("zero_copy", int(zc))
                    got = dg.walk(spec, roots, zero_copy=zc)
                    assert_equal(case, got, r.want, f"{what} host walk zero_copy={zc}")
                    assert dg.last_walk_stats() == expected_stats(r, nq, dedup), f"{what} host walk zero_copy={zc}"
                    del got
                w = DeviceWalk(dg, spec, nq, node_cap=1)
                need = w.launch_fitted(roots_dev)
                assert need[0] == (r.need if dedup and nq >= DEDUP_MIN else int(r.want.off[-1])), f"{what}: caller-arena node need"
                assert w.node_cap == need[0]
                assert_equal(case, device_result(w, nq), r.want, f"{what} caller arena")
                assert dg.last_walk_stats() == expected_stats(r, nq, dedup), f"{what} caller arena"
                if dedup and nq >= DEDUP_MIN and case.depth != 1:        # at depth 1 the canonical walks expand nothing
                    t = dg.last_walk_tier_counts()["first"]
                    assert t["s1_heavy"] >= 1, f"{what}: the heavy group's canonical walk was not handed on as heavy ({t})"
        if case.kind != "distances":                          # depths keep a walk in one piece
            roots = fx.batch
            r = restate(fx, name, len(roots))
            for dedup in (True, False):
                dg.set_dedup(dedup)
                dg.set_option("chunk_min", 64)
                dg.set_option("chunks", 2)
                for call in range(3):                      # a first call at this batch size sizes the pieces
                    got = dg.walk(spec, roots, zero_copy=bool(call & 1))
                    if call:
                        assert dg.get_option("last_host_chunks") == 2
                    assert_equal(case, got, r.want, f"{name} block_tiers={tiers} dedup={dedup} chunked call {call}")
                    del got
                dg.set_option("chunk_min", 2 << 20)
    finally:
        dg.set_option("chunks", 8)
        dg.set_option("chunk_min", 2 << 20)
        dg.set_option("zero_copy", 1)
        dg.set_option("block_tiers", 2)
        dg.set_dedup(True)
