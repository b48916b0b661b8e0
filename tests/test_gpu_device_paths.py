"""The device-resident exposure-path rows (DevicePaths.count + fill, what the flagship bench times) against the CPU oracle.

The host API ships the factorised rows (links + templates) and expands them on the host; these tests check the flat rows the
fill pass writes to device memory: hops, relationships (4 bytes per row, the 4th is padding = -2), credential / tool counts and
per-finding offsets.  Needs a GPU.
"""

from __future__ import annotations

import numpy as np
import pytest

from golden_util import ALL_FIXTURES, edge_arrays, load, node_rank, seeded_graph
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

SEEDED = [(64, 300, 1), (2000, 12000, 2), (6000, 90000, 3), (30000, 400000, 4)]
ET_AGENT, ET_SERVER, ET_VULN, ET_MISCONF, ET_USER, ET_SA = 0, 1, 8, 9, 13, 17
USES, DEPENDS_ON, PROVIDES_TOOL, EXPOSES_CRED, VULNERABLE_TO = 1, 2, 3, 4, 9


def hub_graph():
    """A seeded graph plus reverse rows longer than the kernels' per-thread limit (64 entries), each handled by a whole warp:
    a server used by 100 principals (some through a pair whose first edge is not USES, some bidirectional, plus USES edges from
    non-principals), a package 80 servers depend on, and a finding with 70 vulnerable sources."""
    src, dst, rel, flags, nt = seeded_graph(2000, 12000, 2)
    rng = np.random.default_rng(31)
    types, edges = list(nt), []

    def node(t):
        types.append(t)
        return len(types) - 1

    def edge(a, b, r, fl=1):
        edges.append((a, b, r, fl))

    hub, quiet, pkg = node(ET_SERVER), node(ET_SERVER), node(3)
    for i in range(100):
        a = node((ET_AGENT, ET_USER, ET_SA)[i % 3])
        if i % 7 == 0:
            edge(a, hub, 13)                       # the pair's first edge: its relationship is the row's (agent, server) one
        edge(a, hub, USES, 3 if i % 5 == 0 else 1)
    for _ in range(6):
        edge(node(2), hub, USES)                   # not a principal
    for k in range(4):
        edge(hub, node(10), EXPOSES_CRED if k % 2 else PROVIDES_TOOL)
    edge(hub, pkg, DEPENDS_ON)
    edge(quiet, pkg, 26)
    edge(quiet, pkg, DEPENDS_ON)                   # not the pair's first edge
    servers = []
    for k in range(80):
        s = node(ET_SERVER)
        servers.append(s)
        for _ in range(k % 4):
            edge(node(ET_AGENT), s, USES)
        edge(s, pkg, DEPENDS_ON)
    findings = [node(ET_VULN if k % 2 else ET_MISCONF) for k in range(6)]
    for k, f in enumerate(findings):
        edge((pkg, hub, quiet)[k % 3], f, VULNERABLE_TO)
        edge(pkg if k % 3 else hub, f, VULNERABLE_TO, 3)
    wide = node(ET_VULN)
    for s in [hub, quiet, pkg] + servers[:67]:
        edge(s, wide, VULNERABLE_TO)
    e = np.asarray(edges, dtype=np.int64)
    src = np.concatenate([src, e[:, 0]]).astype(np.int32)
    dst = np.concatenate([dst, e[:, 1]]).astype(np.int32)
    rel = np.concatenate([rel, e[:, 2]]).astype(np.uint8)
    flags = np.concatenate([flags, e[:, 3]]).astype(np.uint8)
    nt = np.asarray(types, dtype=np.uint8)
    rank = rng.permutation(len(nt)).astype(np.int32)
    return src, dst, rel, flags, nt, rank


_cache: dict = {}


def graphs_for(key):
    if key in _cache:
        return _cache[key]
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    if key == "hub":
        src, dst, rel, flags, nt, rank = hub_graph()
    elif isinstance(key, str):
        doc = load(key)
        src, dst, rel, flags = edge_arrays(doc)
        nt = np.asarray(doc["node_types"], dtype=np.uint8)
        rank = node_rank(doc["node_ids"])
    else:
        n, e, seed = key
        src, dst, rel, flags, nt = seeded_graph(n, e, seed)
        rank = np.random.default_rng(seed + 1).permutation(n).astype(np.int32)
    og = orc.build_csr(len(nt), src, dst, rel, flags, nt)
    dg = DeviceGraph.upload(csrmod.from_arrays(None, nt, src, dst, rel, flags, node_rank=rank))
    _cache[key] = (og, dg, nt, rank)
    return _cache[key]


def device_rows(paths, findings_dev, n):
    """count + fill on the device, the rows copied back: (f_off, hops [R,4], rels [R,4], ncred, ntool)."""
    import torch

    rows = paths.run_fitted(findings_dev, n)
    torch.cuda.synchronize()
    f_off = paths.f_off[: n + 1].cpu().numpy()
    assert int(f_off[-1]) == rows
    return (f_off, paths.hops[: rows * 4].view(rows, 4).cpu().numpy(), paths.rels[: rows * 4].view(rows, 4).cpu().numpy(),
            paths.ncred[:rows].cpu().numpy(), paths.ntool[:rows].cpu().numpy())


def assert_rows_equal(got, want, f):
    f_off, hops, rels, ncred, ntool = got
    np.testing.assert_array_equal(hops, want.hops)
    np.testing.assert_array_equal(rels[:, :3], want.rels)
    assert (rels[:, 3] == -2).all()
    np.testing.assert_array_equal(ncred, want.ncred)
    np.testing.assert_array_equal(ntool, want.ntool)
    assert f_off[0] == 0 and (np.diff(f_off) >= 0).all()
    np.testing.assert_array_equal(np.repeat(np.asarray(f, dtype=np.int32), np.diff(f_off)), hops[:, 3])


@pytest.mark.parametrize("key", SEEDED + ALL_FIXTURES + ["hub"])
def test_device_rows_match_oracle(key):
    import torch

    from agent_bom_b200.torch_api import DevicePaths

    og, dg, nt, rank = graphs_for(key)
    findings = np.flatnonzero((nt == ET_VULN) | (nt == ET_MISCONF)).astype(np.int32)
    extra = np.asarray([0, og.n_nodes - 1, -1, -7], dtype=np.int32)   # non-findings / invalid ids yield no rows
    f = np.concatenate([findings[: len(findings) // 2], extra, findings[len(findings) // 2:]])
    paths = DevicePaths(dg, len(f))
    f_dev = torch.from_numpy(f).cuda()
    assert_rows_equal(device_rows(paths, f_dev, len(f)), orc.derived_paths(og, f, rank), f)
    # a second, smaller batch through the same (larger) buffers
    f2 = np.ascontiguousarray(f[::3][::-1])
    f2_dev = torch.from_numpy(f2).cuda()
    assert_rows_equal(device_rows(paths, f2_dev, len(f2)), orc.derived_paths(og, f2, rank), f2)


def test_hub_rows_through_the_host_api():
    """The long-reverse-row case through the host API's factorised rows as well."""
    og, dg, nt, rank = graphs_for("hub")
    f = np.flatnonzero((nt == ET_VULN) | (nt == ET_MISCONF)).astype(np.int32)
    want = orc.derived_paths(og, f, rank)
    got = dg.exposure_paths_many(f)
    assert int(np.diff(got.off).max()) > 64
    np.testing.assert_array_equal(got.hops, want.hops)
    np.testing.assert_array_equal(got.rels, want.rels)
    np.testing.assert_array_equal(got.ncred, want.ncred)
    np.testing.assert_array_equal(got.ntool, want.ntool)


@pytest.fixture(scope="module")
def scale():
    from agent_bom_b200 import estate
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    est = estate.generate(20_700, 2145, estate.BENCH_KNOBS, exact_rank=False)
    host = csrmod.from_arrays(None, est.node_type, est.src, est.dst, est.rel, est.flags, node_rank=est.node_rank)
    dg = DeviceGraph.upload(host)
    og = orc.OracleGraph(n_nodes=host.n_nodes, fwd_off=host.fwd_off, fwd_nbr=host.fwd_nbr, fwd_meta=host.fwd_meta, fwd_eid=host.fwd_eid,
                         rev_off=host.rev_off, rev_nbr=host.rev_nbr, rev_meta=host.rev_meta, rev_eid=host.rev_eid, node_type=host.node_type)
    yield est, dg, og
    dg.close()


def test_device_rows_at_scale(scale):
    """M2 estate, every finding: links with up to dozens of servers' rows, so a link's rows cross the fill pass's row tiles.
    All rows against the host API's expansion of the factorised rows; a sample against the oracle."""
    import torch

    from agent_bom_b200.torch_api import DevicePaths

    est, dg, og = scale
    f = np.ascontiguousarray(est.findings).astype(np.int32)
    paths = DevicePaths(dg, len(f))
    got = device_rows(paths, torch.from_numpy(f).cuda(), len(f))
    f_off, hops, rels, ncred, ntool = got
    host = dg.exposure_paths_many(f)
    np.testing.assert_array_equal(f_off, host.off)
    np.testing.assert_array_equal(hops, host.hops)
    np.testing.assert_array_equal(rels[:, :3], host.rels)
    np.testing.assert_array_equal(ncred, host.ncred)
    np.testing.assert_array_equal(ntool, host.ntool)
    rng = np.random.default_rng(41)
    idx = np.sort(rng.choice(len(f), size=3000, replace=False))
    sel = f[idx]
    want = orc.derived_paths(og, sel, est.node_rank)
    take = np.concatenate([np.arange(f_off[i], f_off[i + 1]) for i in idx]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum(np.diff(f_off)[idx])])
    assert_rows_equal((sub_off, hops[take], rels[take], ncred[take], ntool[take]), want, sel)
