"""The NetworkX backend's CPU oracle and path restatements at the edges of the estate golden: non-finite and degenerate weights,
every row length around numpy's pairwise-sum blocks, path counts that overflow, long paths, and graphs of 300 000 nodes.

``tests/golden/context/networkx_edges.json.gz`` (``oracle/make_networkx_edges_golden.py``) holds networkx 3.6.1's answers; the
graphs are rebuilt from the generator parameters it stores.  The GPU side is ``test_gpu_networkx_edges.py``.
"""

from __future__ import annotations

import gzip
import hashlib
import json
from functools import lru_cache
from pathlib import Path

import numpy as np
import pytest

from oracle import nx_oracle
from oracle.make_networkx_edges_golden import case_ops, digraph
from test_networkx_backend import CASES as BACKEND_CASES
from test_networkx_backend import replay

GOLD = json.loads(gzip.decompress((Path(__file__).parent / "golden" / "context" / "networkx_edges.json.gz").read_bytes()))
CASES = GOLD["cases"]
LABELS = [c["label"] for c in CASES]
PAGERANK_LABELS = [c["label"] for c in CASES if "iterations" in c]
CASE = dict(zip(LABELS, CASES))


@lru_cache(maxsize=None)
def ops_of(label: str) -> list:
    """The case's op sequence, rebuilt from its generator parameters (shared: callers do not modify it)."""
    return case_ops(CASE[label]["params"])


def assert_bitwise(got, want, what: str = "") -> None:
    """Equal bit for bit where ``want`` is finite or infinite; NaN exactly where ``want`` is NaN (NaN payloads differ by platform)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    bad = np.flatnonzero(got[~nan].view(np.uint64) != want[~nan].view(np.uint64))
    assert bad.size == 0, f"{what}: {bad.size} scores differ, first at {np.flatnonzero(~nan)[bad[0]]}"


def check_pagerank(case: dict, scores: np.ndarray, iterations: int) -> None:
    """``scores`` / ``iterations`` as the oracle or the device returned them, against networkx's answer for the case."""
    assert iterations == case["iterations"], case["label"]
    if not iterations:
        return
    if "pagerank_sha256" in case:
        for i, want in case["pagerank_at"]:
            assert_bitwise(scores[i:i + 1], [want], f"{case['label']} node {i}")
        assert hashlib.sha256(np.ascontiguousarray(scores, dtype="<f8").tobytes()).hexdigest() == case["pagerank_sha256"]
    else:
        assert_bitwise(scores, case["pagerank"], case["label"])


# ---------------------------------------------------------------- the oracle against the fixture
@pytest.mark.parametrize("label", PAGERANK_LABELS)
def test_oracle_pagerank_matches_networkx(label):
    """Scores and iterations; ``iterations == 0`` is networkx's PowerIterationFailedConvergence (subnormal, tiny-sum, NaN and
    inf - inf rows)."""
    case = CASE[label]
    g = nx_oracle.replay(ops_of(label))
    assert g.n == case["nodes"]
    pr, it = nx_oracle.pagerank(g)
    check_pagerank(case, pr, it)


def test_oracle_betweenness_keeps_networkx_nans():
    """Path counts pass 2^1024 on the chain: networkx's betweenness is NaN past the first layers and 0.0 on the two sources of
    layer 0, which have no predecessors (a back-propagation that visited the source would turn them NaN too)."""
    case = CASE["chain"]
    want = np.asarray(case["betweenness"])
    g = nx_oracle.replay(ops_of("chain"))
    sources = [g.ids.index("L0000_0"), g.ids.index("L0000_1")]
    assert np.isnan(want).sum() > 2000 and want[sources].tolist() == [0.0, 0.0]
    assert_bitwise(nx_oracle.betweenness(g)[0], want, "chain")
    assert_bitwise(nx_oracle.betweenness(g, threads=1)[0], want, "chain, one thread")


def test_fixture_cases_reach_the_edges():
    """What each case is for: the weight cases converge and fail where networkx does, the sweep has its row lengths, the long-path
    answers outgrow the device's first path arena (max(8 per pair, 65 536) nodes)."""
    failing = {c["label"] for c in CASES if c.get("iterations") == 0}
    assert failing == {"weights:subnormal-weights", "weights:tiny-row-sum", "weights:nan-weight", "weights:inf-minus-inf"}
    assert CASE["weights:overflow-row-sum"]["iterations"] > 0 and CASE["weights:inf-weight"]["iterations"] > 0
    g = nx_oracle.replay(ops_of("rows"))
    lengths = set(np.diff(g.foff).tolist())
    assert {1, 8, 16, 127, 128, 129, 130, 255, 256, 257, 1023, 1024, 1025, 8191, 8192, 8193, 65537} <= lengths
    assert np.bincount(g.fnbr, minlength=g.n).max() == 20_000
    case = CASE["long-path"]
    total = sum(len(p) for _, _, p in case["shortest"] if p)
    assert total > max(65_536, 8 * len(case["shortest"]))
    assert any(p is None for _, _, p in case["shortest"])


# ---------------------------------------------------------------- each new case can fail
def scipy_pagerank(g: nx_oracle.DiGraphArrays, *, dangling_by_sum: bool = False, keep_zero_rows: bool = False):
    """networkx's _pagerank_scipy restated on scipy with two rules switchable: ``dangling_by_sum`` flags a row by ``S == 0`` before
    the inversion (so an overflowed sum is not dangling), ``keep_zero_rows`` scales every entry by its row's inverse (so a row
    with inverse 0 keeps 0 * inf = NaN entries).  Both off, it is networkx's rule.  Returns (scores, iterations), (None, 0)."""
    sp = pytest.importorskip("scipy.sparse")
    n = g.n
    row = np.repeat(np.arange(n), np.diff(g.foff))
    A = sp.coo_array((g.w, (row, g.fnbr)), shape=(n, n)).tocsr()
    with np.errstate(all="ignore"):
        S = A.sum(axis=1)
        flagged = np.where(S == 0)[0]
        S[S != 0] = 1.0 / S[S != 0]
        if keep_zero_rows:
            A = sp.csr_array((A.data * np.repeat(S, np.diff(A.indptr)), A.indices, A.indptr), shape=A.shape)
        else:
            A = sp.dia_array((S.T, 0), shape=A.shape).tocsr() @ A
        x = p = np.repeat(1.0 / n, n)
        dangling = flagged if dangling_by_sum else np.where(S == 0)[0]
        for it in range(100):
            xlast = x
            x = 0.85 * (x @ A + sum(x[dangling]) * p) + (1 - 0.85) * p
            if np.absolute(x - xlast).sum() < n * 1e-6:
                return x, it + 1
    return None, 0


def test_restated_scipy_rules_tell_the_weight_cases_apart():
    """networkx's rules reproduce every weight case; flagging dangling rows by their sum misses the overflowing rows, and keeping
    the entries of a row with inverse 0 turns an inf weight into a failure to converge."""
    for label in PAGERANK_LABELS:
        if not label.startswith("weights:"):
            continue
        case = CASE[label]
        pr, it = scipy_pagerank(nx_oracle.replay(ops_of(label)))
        assert it == case["iterations"], label
        if it:
            assert_bitwise(pr, case["pagerank"], label)
    for label in ("weights:overflow-row-sum", "weights:negative-overflow-row-sum", "weights:inf-weight"):
        pr, it = scipy_pagerank(nx_oracle.replay(ops_of(label)), dangling_by_sum=True)
        assert it != CASE[label]["iterations"] or pr.tolist() != CASE[label]["pagerank"], label
    pr, it = scipy_pagerank(nx_oracle.replay(ops_of("weights:inf-weight")), keep_zero_rows=True)
    assert it == 0 and CASE["weights:inf-weight"]["iterations"] > 0


def test_fringe_tie_rule_changes_long_path_answers():
    """networkx expands the forward fringe while it is no longer than the reverse one; the diamonds make the other rule pick
    different middle nodes on most far-apart pairs."""
    case = CASE["long-path"]
    rows = nx_oracle.Rows.of(replay(ops_of("long-path")).csr)
    differ = sum(nx_oracle.shortest_path(rows, s, t, ties_forward=False) != want for s, t, want in case["shortest"])
    assert differ >= 50


# ---------------------------------------------------------------- the path restatements against both fixtures
def test_path_restatements_match_the_long_path_answers():
    case = CASE["long-path"]
    rows = nx_oracle.Rows.of(replay(ops_of("long-path")).csr)
    for s, t, want in case["shortest"]:
        assert nx_oracle.shortest_path(rows, s, t) == want, (s, t)
    for s, d, want in case["bfs"]:
        assert nx_oracle.bfs(rows, s, d) == want, (s, d)


@pytest.mark.parametrize("case", BACKEND_CASES, ids=[c["label"] for c in BACKEND_CASES])
def test_path_restatements_match_the_backend_golden(case):
    """Every ``shortest_path`` and ``bfs`` answer of the reference NetworkXBackend between nodes of the graph."""
    b = replay(case["ops"])
    c = b.csr
    rows, ids = nx_oracle.Rows.of(c), c.node_ids
    named = lambda p: None if p is None else [ids[i] for i in p]    # noqa: E731
    checked = 0
    for s, t, want in case["shortest"]:
        if s in c.index and t in c.index:
            assert named(nx_oracle.shortest_path(rows, c.index[s], c.index[t])) == want, (s, t)
            checked += 1
    for s, d, want in case["bfs"]:
        if s in c.index:
            assert [named(p) for p in nx_oracle.bfs(rows, c.index[s], d)] == want, (s, d)
    assert checked or not ids


# ---------------------------------------------------------------- estates and scale
def estate_ops(agents: int, knobs, *, both_ways: bool = False) -> list:
    """A generator estate as backend ops: bidirectional relationships as undirected edges, weights varied by relationship;
    ``both_ways`` adds every edge in both directions, which gives many equally short paths."""
    from agent_bom_b200 import estate

    est = estate.generate(agents, 2145, knobs, exact_rank=False)
    ids = [f"v{i}" for i in range(len(est.node_type))]
    ops = [["n", v, "node", v, {}] for v in ids]
    weights = (1.0, 0.5, 0.25, 1.5, 2.0, 1 / 3)
    for s, d, r, f in zip(est.src.tolist(), est.dst.tolist(), est.rel.tolist(), est.flags.tolist()):
        ops.append(["e", ids[s], ids[d], "rel", weights[r % len(weights)], not both_ways and not (f & 2), {}])
    return ops


def _walk(rows_of: list[list[int]], v: int, steps: int, rng) -> int:
    for _ in range(steps):
        row = rows_of[v]
        if not row:
            break
        v = row[int(rng.integers(0, len(row)))]
    return v


def estate_pairs(rows: nx_oracle.Rows, seed: int, count: int = 2000) -> list[tuple[int, int]]:
    """Seeded (source, target) pairs: half uniform (mostly without a path on a directed estate), half from a node with successors
    to the end of a random walk of 1-12 steps (with a path).  Then the farthest nodes of 50 sources' BFS trees (the longest
    answers), pairs with no path (a source without successors, a target without predecessors), s == t, and pairs from and to the
    node of largest degree."""
    rng = np.random.default_rng(seed)
    n = len(rows.succ)
    with_succ = np.flatnonzero([bool(r) for r in rows.succ])
    pairs = []
    for i in range(count):
        if i % 2:
            pairs.append((int(rng.integers(0, n)), int(rng.integers(0, n))))
        else:
            s = int(with_succ[int(rng.integers(0, with_succ.shape[0]))])
            pairs.append((s, _walk(rows.succ, s, int(rng.integers(1, 13)), rng)))
    for s in rng.integers(0, n, 50).tolist():
        far = nx_oracle.bfs_tree_nodes(rows, s, n)[-4:]
        pairs += [(s, t) for t in far]
    no_out = [v for v in range(n) if not rows.succ[v]]
    no_in = [v for v in range(n) if not rows.pred[v]]
    pairs += [(no_out[int(i)], int(t)) for i, t in zip(rng.integers(0, max(len(no_out), 1), 20 if no_out else 0), rng.integers(0, n, 20))]
    pairs += [(int(s), no_in[int(i)]) for s, i in zip(rng.integers(0, n, 20), rng.integers(0, max(len(no_in), 1), 20 if no_in else 0))]
    pairs += [(v, v) for v in rng.integers(0, n, 10).tolist()]
    hub = hub_of(rows)
    pairs += [(hub, _walk(rows.succ, hub, k, rng)) for k in range(1, 21)]
    pairs += [(_walk(rows.pred, hub, k, rng), hub) for k in range(1, 21)]
    return pairs


def hub_of(rows: nx_oracle.Rows) -> int:
    deg = [len(a) + len(b) for a, b in zip(rows.succ, rows.pred)]
    return int(np.argmax(deg))


@pytest.mark.parametrize("both_ways", [False, True], ids=["directed", "both-ways"])
def test_path_restatement_matches_networkx_on_the_estate(both_ways):
    """``nx.shortest_path`` on the 1 000-agent estate DiGraph, pair by pair.  On the directed estate every reachable pair has one
    answer whichever side the search expands first; with every edge both ways the fringe tie rule changes several answers."""
    nx = pytest.importorskip("networkx")
    from agent_bom_b200 import estate

    ops = estate_ops(1000, estate.Knobs(), both_ways=both_ways)
    c = replay(ops).csr
    rows, ids = nx_oracle.Rows.of(c), c.node_ids
    g = digraph(ops)
    assert list(g) == ids
    pairs = estate_pairs(rows, 1000)
    found = differ = 0
    for s, t in pairs:
        try:
            want = [c.index[v] for v in nx.shortest_path(g, ids[s], ids[t])]
        except nx.NetworkXNoPath:
            want = None
        assert nx_oracle.shortest_path(rows, s, t) == want, (s, t)
        found += want is not None
        differ += nx_oracle.shortest_path(rows, s, t, ties_forward=False) != want
    assert found > len(pairs) // 2
    if both_ways:
        assert differ >= 5


def scale_graph(n: int, m: int, hub_rows: int, hub_len: int, seed: int):
    """Seeded DiGraph edge list in insertion order (src, dst, weight): ``m`` random edges, ``hub_rows`` rows of ``hub_len``
    successors each and one sink with ``hub_len`` predecessors; no repeated (src, dst).  Weights are exact dyadic values across
    2^-20 .. 2^20 and every fifth node has no successors."""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m)
    src = src[src % 5 != 4]
    dst = rng.integers(0, n, src.shape[0])
    rows = np.flatnonzero(np.arange(n) % 5 != 4)
    hubs = rng.choice(rows, hub_rows, replace=False)
    sink = int(rng.integers(0, n))
    src = np.concatenate([src, np.repeat(hubs, hub_len), rng.choice(rows, hub_len, replace=False)])
    dst = np.concatenate([dst, *[rng.choice(n, hub_len, replace=False) for _ in range(hub_rows)], np.full(hub_len, sink)])
    _, first = np.unique(src.astype(np.int64) * n + dst, return_index=True)
    keep = np.sort(first)
    src, dst = src[keep].astype(np.int32), dst[keep].astype(np.int32)
    w = np.ldexp(rng.integers(1, 1 << 20, src.shape[0]).astype(np.float64), rng.integers(-40, 1, src.shape[0]))
    return src, dst, w


def arrays_of(n: int, src, dst, w) -> nx_oracle.DiGraphArrays:
    """The edge list as the oracle's rows: successors in insertion order."""
    order = np.argsort(src, kind="stable")
    foff = np.zeros(n + 1, dtype=np.int64)
    foff[1:] = np.cumsum(np.bincount(src, minlength=n))
    return nx_oracle.DiGraphArrays([str(i) for i in range(n)], foff, np.ascontiguousarray(dst[order]), np.ascontiguousarray(w[order]))


def test_oracle_pagerank_matches_networkx_at_scale():
    """300 000 nodes, two rows of 100 000 entries and a sink with 100 000 in-edges: the oracle is the device's yardstick at sizes
    networkx is too slow to rerun, so it is tied to networkx there."""
    nx = pytest.importorskip("networkx")
    n = 300_000
    src, dst, w = scale_graph(n, 600_000, 2, 100_000, 300)
    g = nx.DiGraph()
    g.add_nodes_from(range(n))
    g.add_weighted_edges_from(zip(src.tolist(), dst.tolist(), w.tolist()))
    assert max(d for _, d in g.out_degree()) >= 100_000 and max(d for _, d in g.in_degree()) >= 100_000
    want = nx.pagerank(g)
    pr, it = nx_oracle.pagerank(arrays_of(n, src, dst, w))
    assert it > 0
    assert_bitwise(pr, [want[v] for v in range(n)], "300 K nodes")
