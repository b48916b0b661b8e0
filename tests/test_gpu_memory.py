"""Freeing a graph returns all of its device memory.

A graph handle owns a workspace that grows on demand: walk arenas, exposure-path buffers, and the server row table that
the first exposure-path call builds.  A long-running store frees and re-uploads its graph whenever the topology changes,
so anything a freed handle kept would pile up until the device runs out.  The test runs the same upload / query / free
cycle three times and checks that free device memory after the last two cycles is where it was after the first (which
also loads the kernels).
"""

from __future__ import annotations

import numpy as np
import pytest

from golden_util import seeded_graph
from test_gpu_parity import REACH4, VULN_PKG, device_graph

pytestmark = pytest.mark.gpu

# 2 M nodes: the server row table's offsets alone take (n + 1) x 8 B (20 MB with DevBuf's growth slack), far above the tolerance
N_NODES, N_EDGES = 2_000_000, 4_000_000
TOLERANCE = 4 << 20


def cycle(dg, findings, agents, sources):
    try:
        dg.exposure_many(findings, 4)          # builds the server row table and the link arrays
        dg.finding_context(findings)
        dg.dependency_reach(agents, REACH4, VULN_PKG)
        dg.bottleneck_scores(sources)
    finally:
        dg.close()


def test_freed_graphs_return_their_device_memory():
    import torch

    from agent_bom_b200.engine import DeviceGraph

    src, dst, rel, flags, nt = seeded_graph(N_NODES, N_EDGES, 41, hub=False)
    rank = np.random.default_rng(42).permutation(N_NODES).astype(np.int32)
    rng = np.random.default_rng(43)
    findings = np.sort(rng.choice(np.flatnonzero((nt == 8) | (nt == 9)), 20_000, replace=False)).astype(np.int32)
    agents = np.sort(rng.choice(np.flatnonzero(nt == 0), 4_096, replace=False)).astype(np.int32)
    sources = findings[:4]

    torch.cuda.mem_get_info()
    dg, host = device_graph(src, dst, rel, flags, nt, rank)
    cycle(dg, findings, agents, sources)
    free_before, _ = torch.cuda.mem_get_info()
    for _ in range(2):
        cycle(DeviceGraph.upload(host), findings, agents, sources)
    free_after, _ = torch.cuda.mem_get_info()
    drop = free_before - free_after
    print(f"free device memory dropped by {drop / 2**20:.2f} MiB over two upload / query / free cycles")
    assert drop <= TOLERANCE, f"two freed graphs kept {drop / 2**20:.1f} MiB of device memory"
