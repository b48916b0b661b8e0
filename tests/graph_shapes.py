"""Graph shapes that push the walk through every storage tier: deep chains, 100 000-entry rows, repeated neighbours, tiny graphs.

``seeded_graph`` (golden_util.py) makes random multigraphs of small diameter, short rows and unique (src, dst, rel) triples.  The
builders here make the shapes it never does, with answers known by construction:

* ``deep()``: directed chains of 254..258, 300, 4 100 and 70 000 nodes (around S1's and the mid block tier's 255-level depth limit,
  the mid tier's 4 096-entry queue, and G1's 65 536-entry queue), a bidirectional chain, a comb, and a dependency chain of
  packages below 300 agents with findings at package depths 10, 254, 255, 256 and 300.
* ``wide()``: a hub with a 100 000-entry forward row and one with a 100 000-entry reverse row (longer than the big block tier's
  36 864-entry queue and G1's 65 536), rows that repeat one neighbour across 32-entry chunk boundaries, self-loops, a 300-node
  clique and a complete bipartite 200 x 200 block.
* ``tiny()``: n = 1, n = 2 with a self-loop, n = 31 / 32 / 33 (one bitmap word and its edges), and a graph whose roots are ghosts.

Each builder returns a ``Shape``: the edge arrays in ``seeded_graph``'s form plus a dict of named node ids.  Node ids are shuffled
with a fixed seed after the graph is laid out, so consecutive queue entries do not share bitmap words or hash buckets by
construction; the edge order (hence every row's order) is the order the builder added the edges in.
"""

from __future__ import annotations

from typing import NamedTuple

import numpy as np

AGENT, SERVER, PACKAGE, TOOL, VULN, CRED, GHOST = 0, 1, 2, 3, 8, 10, 255
USES, DEPENDS_ON, PROVIDES_TOOL, EXPOSES_CRED, CONTAINS, AFFECTS, VULNERABLE_TO, OWNS = 1, 2, 3, 4, 7, 8, 9, 17
TRAV, BIDIR = 1, 2
CHAIN_LENGTHS = (254, 255, 256, 257, 258, 300, 4100)
LONG_CHAIN = 70_000
HUB_ROW = 100_000
FINDING_DEPTHS = (10, 254, 255, 256, 300)        # package-chain depth of the package each finding hangs off
REPEAT_AT = (0, 31, 32, 63, 64, 95, 96, 127, 128)  # row positions of the repeated neighbour: both sides of each 32-entry boundary
REPEAT_RELS = (DEPENDS_ON, EXPOSES_CRED, USES, 13, CONTAINS, 14, PROVIDES_TOOL, OWNS, 26)   # alternately inside / outside REACH4


class Shape(NamedTuple):
    src: np.ndarray
    dst: np.ndarray
    rel: np.ndarray
    flags: np.ndarray
    node_type: np.ndarray
    names: dict


class _Builder:
    """Nodes and edges in logical ids; ``shape`` renames the nodes by a seeded permutation."""

    def __init__(self, seed: int):
        self.rng = np.random.default_rng(seed)
        self.types: list[np.ndarray] = []
        self.n = 0
        self.edges: list[np.ndarray] = []      # [k, 4] blocks of (src, dst, rel, flags), in insertion order
        self.names: dict = {}

    def nodes(self, k: int, types) -> np.ndarray:
        ids = np.arange(self.n, self.n + k, dtype=np.int64)
        self.types.append(np.broadcast_to(np.asarray(types, dtype=np.uint8), (k,)).copy())
        self.n += k
        return ids

    def add(self, src, dst, rel, flags=TRAV):
        src = np.atleast_1d(np.asarray(src, dtype=np.int64))
        dst = np.atleast_1d(np.asarray(dst, dtype=np.int64))
        k = max(len(src), len(dst))
        e = np.empty((k, 4), dtype=np.int64)
        e[:, 0], e[:, 1], e[:, 2], e[:, 3] = src, dst, rel, flags
        self.edges.append(e)

    def chain(self, k: int, types, rel=DEPENDS_ON, flags=TRAV) -> np.ndarray:
        ids = self.nodes(k, types)
        self.add(ids[:-1], ids[1:], rel, flags)
        return ids

    def shape(self, perm_seed: int) -> Shape:
        perm = np.random.default_rng(perm_seed).permutation(self.n)        # logical id i -> node id perm[i]
        node_type = np.empty(self.n, dtype=np.uint8)
        node_type[perm] = np.concatenate(self.types)
        e = np.concatenate(self.edges) if self.edges else np.zeros((0, 4), dtype=np.int64)

        def rename(v):
            if isinstance(v, dict):
                return {k: rename(x) for k, x in v.items()}
            a = np.asarray(v, dtype=np.int64)
            return int(perm[a]) if a.ndim == 0 else perm[a].astype(np.int32)

        return Shape(perm[e[:, 0]].astype(np.int32), perm[e[:, 1]].astype(np.int32), e[:, 2].astype(np.uint8), e[:, 3].astype(np.uint8),
                     node_type, {k: rename(v) for k, v in self.names.items()})


def _mixed_types(rng, k: int) -> np.ndarray:
    """Node types for chain members: no agents (the dependency-reach walk starts at every agent) and no findings."""
    return rng.choice(np.array([PACKAGE, SERVER, TOOL, CRED, 5, 13, 21], dtype=np.uint8), size=k, p=[0.4, 0.1, 0.15, 0.1, 0.1, 0.1, 0.05])


def deep(seed: int = 70) -> Shape:
    """>= 70 000 nodes (G1's queue is then 65 536 entries) in disjoint components; see the module docstring."""
    b = _Builder(seed)
    rng = b.rng
    for k in CHAIN_LENGTHS + (LONG_CHAIN,):
        b.names[f"chain_{k}"] = b.chain(k, _mixed_types(rng, k))
    # bidirectional chain: every edge also walks backwards (reversed copies in both rows)
    b.names["bichain"] = b.chain(300, _mixed_types(rng, 300), rel=CONTAINS, flags=TRAV | BIDIR)
    # comb: spine i -> i + 1 and spine i -> leaf i, so every level holds two entries; every third leaf edge is not traversable
    # and carries a relationship outside the dependency-reach mask
    spine = b.nodes(300, _mixed_types(rng, 300))
    leaf = b.nodes(300, _mixed_types(rng, 300))
    for i in range(300):
        if i + 1 < 300:
            b.add(spine[i], spine[i + 1], DEPENDS_ON)
        b.add(spine[i], leaf[i], EXPOSES_CRED if i % 3 == 0 else PROVIDES_TOOL, 0 if i % 3 == 0 else TRAV)
    b.names["comb_spine"], b.names["comb_leaf"] = spine, leaf
    # 300 agents -USES-> one server -DEPENDS_ON-> pkg 0 -> ... -> pkg 300; every seventh package edge is not traversable
    agents = b.nodes(300, AGENT)
    server = b.nodes(1, SERVER)
    pkgs = b.nodes(301, PACKAGE)
    b.add(agents, np.full(300, server[0]), USES)
    b.add(server, pkgs[:1], DEPENDS_ON)
    b.add(pkgs[:-1], pkgs[1:], DEPENDS_ON, np.where(np.arange(300) % 7 == 3, 0, TRAV))
    vulns = b.nodes(len(FINDING_DEPTHS), VULN)
    b.add(pkgs[list(FINDING_DEPTHS)], vulns, VULNERABLE_TO)
    b.add(agents[:2], pkgs[:1], OWNS)                 # outside the dependency-reach mask: must not shorten any distance
    # two ids without a node record: they point into the comb (a ghost root starts nothing), and the last package points at one
    ghosts = b.nodes(2, GHOST)
    b.add(ghosts, spine[[5, 6]], USES)
    b.add(pkgs[-1], ghosts[1], USES)
    b.names.update(agents=agents, server=server[0], pkgs=pkgs, vulns=vulns, ghosts=ghosts)
    return b.shape(seed + 1)


def wide(seed: int = 100) -> Shape:
    b = _Builder(seed)
    rng = b.rng
    # 100 000 leaves: fhub -> every leaf (forward row of 100 000), every leaf -> rhub (reverse row of 100 000)
    leaves = b.nodes(HUB_ROW, rng.integers(0, 24, size=HUB_ROW).astype(np.uint8))
    fhub, rhub = b.nodes(2, [SERVER, PACKAGE])
    lrel = rng.choice(np.array([USES, DEPENDS_ON, EXPOSES_CRED, CONTAINS, 13], dtype=np.uint8), size=HUB_ROW)
    b.add(np.full(HUB_ROW, fhub), leaves, lrel, np.where(rng.random(HUB_ROW) < 0.1, 0, TRAV))
    b.add(leaves, np.full(HUB_ROW, rhub), DEPENDS_ON, np.where(rng.random(HUB_ROW) < 0.1, 0, TRAV))
    # a row that repeats neighbour x at both sides of every 32-entry boundary up to 128 (distinct relationships, alternately
    # traversable), fillers in between, then a self-loop and a bidirectional self-loop; x leads on to a short tail
    rep, x = b.nodes(2, [AGENT, SERVER])
    fill = b.nodes(160, rng.integers(0, 24, size=160).astype(np.uint8))
    tail = b.chain(40, _mixed_types(rng, 40))
    b.add(x, tail[0], USES)
    k = 0
    for pos in range(140):
        if pos in REPEAT_AT:
            j = REPEAT_AT.index(pos)
            b.add(rep, x, REPEAT_RELS[j], TRAV if j % 2 == 0 else 0)
        else:
            b.add(rep, fill[k], DEPENDS_ON)
            k += 1
    b.add(rep, rep, USES)
    b.add(rep, rep, CONTAINS, TRAV | BIDIR)
    # the same pattern in a reverse row: y is an in-neighbour of rrep at the repeat positions
    rrep, y = b.nodes(2, [VULN, PACKAGE])
    fill2 = b.nodes(160, rng.integers(0, 24, size=160).astype(np.uint8))
    k = 0
    for pos in range(140):
        if pos in REPEAT_AT:
            j = REPEAT_AT.index(pos)
            b.add(y, rrep, REPEAT_RELS[j], TRAV if j % 2 == 0 else 0)
        else:
            b.add(fill2[k], rrep, DEPENDS_ON)
            k += 1
    b.add(tail[-1], y, USES)
    # 300-node clique (every ordered pair, row order shuffled): revisit-dominated levels
    cl = b.nodes(300, _mixed_types(rng, 300))
    ii, jj = np.meshgrid(np.arange(300), np.arange(300), indexing="ij")
    off = ii != jj
    order = rng.permutation(int(off.sum()))
    b.add(cl[ii[off][order]], cl[jj[off][order]], DEPENDS_ON, np.where(rng.random(int(off.sum())) < 0.1, 0, TRAV))
    # complete bipartite 200 x 200, both ways
    left = b.nodes(200, _mixed_types(rng, 200))
    right = b.nodes(200, _mixed_types(rng, 200))
    ii, jj = np.meshgrid(np.arange(200), np.arange(200), indexing="ij")
    b.add(left[ii.ravel()], right[jj.ravel()], USES)
    b.add(right[jj.ravel()], left[ii.ravel()], CONTAINS)
    b.names.update(leaves=leaves, fhub=fhub, rhub=rhub, rep=rep, x=x, fill=fill, rep_tail=tail, rrep=rrep, y=y, clique=cl, left=left, right=right)
    return b.shape(seed + 1)


def tiny() -> dict:
    """name -> Shape: one-node and two-node graphs, the bitmap-word boundary (31, 32, 33 nodes), ghost roots."""
    out = {}
    b = _Builder(1)
    b.names["only"] = b.nodes(1, PACKAGE)
    out["n1"] = b.shape(2)
    b = _Builder(3)
    u = b.nodes(2, [AGENT, SERVER])
    b.add(u[1], u[1], USES)
    b.names["loop"], b.names["other"] = u[1], u[0]
    out["n2_self_loop"] = b.shape(4)
    for n in (31, 32, 33):
        b = _Builder(n)
        ring = b.chain(n, _mixed_types(b.rng, n))      # a ring with one chord, so every node is reached and revisited
        b.add(ring[-1], ring[0], DEPENDS_ON)
        b.add(ring[n // 2], ring[1], USES, 0)
        b.names["ring"] = ring
        out[f"n{n}_ring"] = b.shape(n + 1)
    b = _Builder(5)
    real = b.nodes(6, PACKAGE)
    gh = b.nodes(3, GHOST)
    b.add(gh, real[:3], DEPENDS_ON)
    b.add(real[:-1], real[1:], DEPENDS_ON)
    b.add(real[-1], gh[2], USES)
    b.names["real"], b.names["ghosts"] = real, gh
    out["ghost_roots"] = b.shape(6)
    return out
