"""The graph-constant exposure tables behind the exposure-path rows: every finding node's links and every vulnerable source's
template are built once per graph, and a call gathers its findings' rows from them.  Checks the device rows (count + fill), the
host API's factorised rows and the ranked pages (unfocused and focused) against the CPU oracle on batches that stress the
per-finding gather (duplicates, invalid ids, non-findings, findings without links), across several batches on one graph and
across a freed and rebuilt graph, and that count + fill replay from a CUDA graph (no host synchronisation) with the eager
result.  Needs a GPU.
"""

from __future__ import annotations

import numpy as np
import pytest

from golden_util import seeded_graph
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

ET_AGENT, ET_SERVER, ET_PACKAGE, ET_VULN, ET_MISCONF, ET_USER, ET_SA, GHOST = 0, 1, 2, 8, 9, 13, 17, 255
USES, DEPENDS_ON, PROVIDES_TOOL, EXPOSES_CRED, VULNERABLE_TO = 1, 2, 3, 4, 9


def exposure_graph():
    """A seeded graph plus hand-made findings: one with several vulnerable sources (a server among them, a package with a
    dependent-server hub longer than 64 entries, and a ghost source), one whose only source is a ghost, one without any source,
    and one with 70 sources (a long reverse row)."""
    src, dst, rel, flags, nt = seeded_graph(3000, 20000, 7)
    types, edges = list(nt), []

    def node(t):
        types.append(t)
        return len(types) - 1

    def edge(a, b, r, fl=1):
        edges.append((a, b, r, fl))

    hub, srv, pkg, ghost = node(ET_SERVER), node(ET_SERVER), node(ET_PACKAGE), node(GHOST)
    for i in range(90):
        edge(node((ET_AGENT, ET_USER, ET_SA)[i % 3]), hub, USES, 3 if i % 4 == 0 else 1)
    for k in range(5):
        edge(hub, node(10), EXPOSES_CRED if k % 2 else PROVIDES_TOOL)
    edge(node(ET_AGENT), srv, USES)
    edge(srv, pkg, 26)
    edge(srv, pkg, DEPENDS_ON)                     # not the pair's first edge
    deps = []
    for k in range(75):
        s = node(ET_SERVER)
        deps.append(s)
        for _ in range(k % 3):
            edge(node(ET_AGENT), s, USES)
        edge(s, pkg, DEPENDS_ON)
    several, ghost_only, no_source, wide = node(ET_VULN), node(ET_MISCONF), node(ET_VULN), node(ET_VULN)
    for s in (pkg, hub, ghost, srv):
        edge(s, several, VULNERABLE_TO)
    edge(hub, several, VULNERABLE_TO, 3)           # a second, bidirectional entry of the pair (hub, several)
    edge(ghost, ghost_only, VULNERABLE_TO)
    for s in [hub, srv, pkg] + deps[:67]:
        edge(s, wide, VULNERABLE_TO)
    e = np.asarray(edges, dtype=np.int64)
    src = np.concatenate([src, e[:, 0]]).astype(np.int32)
    dst = np.concatenate([dst, e[:, 1]]).astype(np.int32)
    rel = np.concatenate([rel, e[:, 2]]).astype(np.uint8)
    flags = np.concatenate([flags, e[:, 3]]).astype(np.uint8)
    nt = np.asarray(types, dtype=np.uint8)
    rank = np.random.default_rng(8).permutation(len(nt)).astype(np.int32)
    special = {"several": several, "ghost_only": ghost_only, "no_source": no_source, "wide": wide, "server": srv}
    return src, dst, rel, flags, nt, rank, special


@pytest.fixture(scope="module")
def graph():
    src, dst, rel, flags, nt, rank, special = exposure_graph()
    og = orc.build_csr(len(nt), src, dst, rel, flags, nt)
    return src, dst, rel, flags, nt, rank, special, og


def upload(graph):
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    src, dst, rel, flags, nt, rank, _special, _og = graph
    return DeviceGraph.upload(csrmod.from_arrays(None, nt, src, dst, rel, flags, node_rank=rank))


def batches(nt, special):
    """Several batches for one graph: duplicates, negative / out-of-range ids, non-finding nodes, findings without links."""
    n = len(nt)
    findings = np.flatnonzero((nt == ET_VULN) | (nt == ET_MISCONF)).astype(np.int32)
    s = special
    non_findings = np.flatnonzero((nt != ET_VULN) & (nt != ET_MISCONF))[:5].astype(np.int32)
    rng = np.random.default_rng(9)
    b1 = np.concatenate([[s["several"], -1, s["several"], n, s["ghost_only"], 2**31 - 1, s["no_source"], -2**31], non_findings,
                         findings[:200], [s["wide"], s["wide"]]]).astype(np.int32)
    b2 = rng.permutation(np.concatenate([findings, findings[::7], non_findings, [-5, n + 3]])).astype(np.int32)
    b3 = np.asarray([s["wide"]] * 3 + [s["several"], s["ghost_only"]], dtype=np.int32)
    b4 = np.asarray([s["no_source"], -1, n], dtype=np.int32)                # no rows at all
    return [b1, b2, b3, b4]


def expected_rows(og, f, rank):
    """Oracle rows and per-finding row counts (ids that are not valid nodes have no rows; the oracle is given only valid ones)."""
    n = og.n_nodes
    counts = np.zeros(len(f), dtype=np.int64)
    valid = (f >= 0) & (f < n)
    want = orc.derived_paths(og, f[valid], rank)
    per = np.asarray([orc.derived_paths(og, [x], rank).hops.shape[0] for x in f[valid]], dtype=np.int64)
    counts[valid] = per
    return want, np.concatenate([[0], np.cumsum(counts)])


def device_rows(dg, f):
    import torch

    from agent_bom_b200.torch_api import DevicePaths

    paths = DevicePaths(dg, len(f))
    f_dev = torch.from_numpy(f).cuda()
    rows = paths.run_fitted(f_dev, len(f))
    torch.cuda.synchronize()
    return (paths.f_off[: len(f) + 1].cpu().numpy(), paths.hops[: rows * 4].view(rows, 4).cpu().numpy(),
            paths.rels[: rows * 4].view(rows, 4).cpu().numpy(), paths.ncred[:rows].cpu().numpy(), paths.ntool[:rows].cpu().numpy())


def check_rows(dg, og, rank, f):
    want, off = expected_rows(og, f, rank)
    f_off, hops, rels, ncred, ntool = device_rows(dg, f)
    np.testing.assert_array_equal(f_off, off)
    np.testing.assert_array_equal(hops, want.hops)
    np.testing.assert_array_equal(rels[:, :3], want.rels)
    assert (rels[:, 3] == -2).all()
    np.testing.assert_array_equal(ncred, want.ncred)
    np.testing.assert_array_equal(ntool, want.ntool)
    host = dg.exposure_paths_many(f)
    np.testing.assert_array_equal(host.off, off)
    np.testing.assert_array_equal(host.hops, want.hops)
    np.testing.assert_array_equal(host.rels, want.rels)
    np.testing.assert_array_equal(host.ncred, want.ncred)
    np.testing.assert_array_equal(host.ntool, want.ntool)
    # factorised form: every link's rows are its source's template rows, the templates are distinct and in node order
    src = host.link_source
    _, first = np.unique(src, return_index=True)
    assert (np.diff(host.link_template[first]) >= 0).all()
    assert int(sum(host.link_row_off[i + 1] - host.link_row_off[i] for i in first)) == host.template.shape[0]
    for l in range(src.shape[0]):
        a, b, t0 = int(host.link_row_off[l]), int(host.link_row_off[l + 1]), int(host.link_template[l])
        np.testing.assert_array_equal(host.template[t0: t0 + b - a][:, :2], host.hops[a:b, :2])
    return want, off


def rank_inputs(nt, f):
    """Base risk per finding node, a dense-rank table and per-server label counts (arbitrary, seeded)."""
    n = len(nt)
    rng = np.random.default_rng(11)
    n_base = 3
    node_base = rng.integers(0, n_base, size=n).astype(np.int32)
    base_id = np.where((f >= 0) & (f < n), node_base[np.clip(f, 0, n - 1)], 0).astype(np.int32)
    table = rng.integers(0, 40, size=(n_base, 5, 15)).astype(np.uint32)
    ncu = rng.integers(0, 6, size=n).astype(np.int32)
    ntu = rng.integers(0, 6, size=n).astype(np.int32)
    return node_base, base_id, table, ncu, ntu


def check_ranked(dg, nt, f, want, off):
    from agent_bom_b200 import _lib

    node_base, base_id, table, ncu, ntu = rank_inputs(nt, f)
    h = want.hops
    n_rows = h.shape[0]
    fi = np.repeat(np.arange(len(f)), np.diff(off))
    rr = table[base_id[fi], np.minimum(want.ncred, 4), np.minimum(want.ntool, 14)].astype(np.int64)
    nh = np.where(h[:, 2] >= 0, 4, 3)
    order = np.lexsort((np.arange(n_rows), -ntu[h[:, 1]], -ncu[h[:, 1]], -nh, -rr))
    args = (f, base_id, table, ncu, ntu)
    for offset, limit in ((0, n_rows + 10), (n_rows // 3, 50)):
        page, rank, total = dg.rank_exposure_paths(*args, offset, limit)
        assert total == n_rows
        sel = order[offset: offset + limit]
        np.testing.assert_array_equal(page.hops, h[sel])
        np.testing.assert_array_equal(page.rels, want.rels[sel])
        np.testing.assert_array_equal(page.ncred, want.ncred[sel])
        np.testing.assert_array_equal(page.ntool, want.ntool[sel])
        np.testing.assert_array_equal(rank, rr[sel])
    if n_rows == 0:
        return
    focus = np.zeros(len(nt), dtype=np.uint8)
    focus[int(h[n_rows // 2, 0])] |= _lib.FOCUS_AGENT
    focus[int(h[0, 3])] |= _lib.FOCUS_CVE_FINDING
    vs = np.where(h[:, 2] >= 0, h[:, 2], h[:, 1])
    for need in (_lib.FOCUS_AGENT, _lib.FOCUS_CVE, _lib.FOCUS_CVE | _lib.FOCUS_AGENT):
        on_hops = focus[h[:, 0]] | focus[h[:, 1]] | focus[vs]
        on_hops = on_hops & np.uint8(~_lib.FOCUS_CVE_FINDING & 0xFF)
        on_f = focus[h[:, 3]]
        got = on_hops | on_f | np.where(on_f & _lib.FOCUS_CVE_FINDING, _lib.FOCUS_CVE, 0).astype(np.uint8)
        mask = (got & need) == need
        want_order = order[mask[order]]
        page, rank, total, matched = dg.rank_exposure_paths_focused(*args, focus, need, 0, n_rows)
        assert (total, matched) == (n_rows, int(mask.sum()))
        np.testing.assert_array_equal(page.hops, h[want_order])
        np.testing.assert_array_equal(page.rels, want.rels[want_order])


def test_batches_on_one_graph_match_the_oracle(graph):
    """Several batches through one device graph: the tables are built by the first and reused by the others."""
    src, dst, rel, flags, nt, rank, special, og = graph
    dg = upload(graph)
    try:
        seen = []
        for f in batches(nt, special):
            want, off = check_rows(dg, og, rank, f)
            check_ranked(dg, nt, f, want, off)
            seen.append(int(off[-1]))
        assert seen[0] > 0 and seen[-1] == 0
        # the cases the batches are built to hit
        s = special
        _, off = expected_rows(og, np.asarray([s["several"], s["ghost_only"], s["no_source"], s["wide"]], dtype=np.int32), rank)
        per = np.diff(off)
        assert per[0] > 64 and per[1] == 0 and per[2] == 0 and per[3] > 64
    finally:
        dg.close()


def test_freed_and_rebuilt_graph(graph):
    """A graph freed after its tables were built, then uploaded again: the new handle builds its own tables."""
    src, dst, rel, flags, nt, rank, special, og = graph
    f = batches(nt, special)[0]
    first = upload(graph)
    want, off = check_rows(first, og, rank, f)
    first.close()
    second = upload(graph)
    try:
        got_off, hops, rels, ncred, ntool = device_rows(second, f)
        np.testing.assert_array_equal(got_off, off)
        np.testing.assert_array_equal(hops, want.hops)
        np.testing.assert_array_equal(rels[:, :3], want.rels)
        check_ranked(second, nt, f, want, off)
    finally:
        second.close()


def test_count_and_fill_replay_from_a_cuda_graph(graph):
    """After a warm-up call, count + fill issue no host synchronisation and no allocation: both capture into a CUDA graph, and a
    replay on new findings (same batch size) writes what an eager call writes."""
    import torch

    from agent_bom_b200.torch_api import DevicePaths

    src, dst, rel, flags, nt, rank, special, og = graph
    dg = upload(graph)
    try:
        b1, b2 = batches(nt, special)[:2]
        nf = len(b2)
        f1 = np.resize(b1, nf).astype(np.int32)
        eager, _ = expected_rows(og, b2, rank)
        eager_off = device_rows(dg, b2)[0]
        need = int(max(eager_off[-1], device_rows(dg, f1)[0][-1]))
        paths = DevicePaths(dg, nf, row_cap=need)
        f_dev = torch.from_numpy(f1).cuda()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            paths.count(f_dev, stream=side)
            paths.fill(f_dev, stream=side)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            s = torch.cuda.current_stream()
            paths.count(f_dev, stream=s)
            paths.fill(f_dev, stream=s)
        f_dev.copy_(torch.from_numpy(b2))
        paths.hops.fill_(-7)
        cg.replay()
        torch.cuda.synchronize()
        rows = int(paths.f_off[nf].item())
        np.testing.assert_array_equal(paths.f_off[: nf + 1].cpu().numpy(), eager_off)
        np.testing.assert_array_equal(paths.hops[: rows * 4].view(rows, 4).cpu().numpy(), eager.hops)
        np.testing.assert_array_equal(paths.rels[: rows * 4].view(rows, 4)[:, :3].cpu().numpy(), eager.rels)
        np.testing.assert_array_equal(paths.ncred[:rows].cpu().numpy(), eager.ncred)
        np.testing.assert_array_equal(paths.ntool[:rows].cpu().numpy(), eager.ntool)
        del cg
    finally:
        dg.close()
