"""Colliding frontier signatures for the de-duplication fallback tests, checked against a restatement of the hash.

Root-frontier de-duplication (dedup.cuh) groups a batch's sources by a 47-bit hash of their ordered level-1 frontier S' and
verifies each member against its group head element-wise.  COLLISIONS are pairs of different two-node frontiers with equal
hashes, found by ``oracle/make_signature_collisions.py --pairs 8``; test_gpu_dedup_fallbacks.py builds sources on them to force
the verification's fallback.  Here the hash is restated once more, independently of the generator, and every pair is checked to
collide; the GPU tests check the same restatement against the device's signatures.  No GPU needed.
"""

from __future__ import annotations

import pytest

from oracle.make_signature_collisions import signature as generator_signature

M64 = (1 << 64) - 1
SIG_INELIGIBLE = 1 << 47          # dedup.cuh: bit 47 marks a source walked on its own, the low bits are then its query index

# ((a, b), (c, d)): sources whose S' is (a, b) and sources whose S' is (c, d) land in one signature group
COLLISIONS = (
    ((464, 7571), (7781, 4027)),    # 0x3c56aeec016b
    ((2767, 5184), (7485, 7253)),   # 0x4e4879fdba0
    ((513, 7952), (3472, 4371)),    # 0x7fceba452389
    ((3674, 888), (6727, 7216)),    # 0x36ed6f0b101f
    ((402, 612), (2116, 2848)),     # 0x3c3c90a59f00
    ((984, 7159), (3082, 1807)),    # 0x1d4f2fc9d5bc
    ((2513, 6519), (7742, 1915)),   # 0x736cb2b47043
    ((1346, 5663), (6586, 3130)),   # 0x2f039f9e4d66
)
EXPECTED = (0x3c56aeec016b, 0x4e4879fdba0, 0x7fceba452389, 0x36ed6f0b101f, 0x3c3c90a59f00, 0x1d4f2fc9d5bc, 0x736cb2b47043, 0x2f039f9e4d66)


def mix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def frontier_signature(frontier) -> int:
    """``dedup_sig_kernel`` for an eligible source whose level-1 frontier is `frontier` (ordered node ids)."""
    h = mix64(0xABB200 + len(frontier))
    for i, v in enumerate(frontier):
        h = mix64(h ^ ((int(v) & 0xFFFFFFFF) + ((i + 1) << 32)))
    return h & (SIG_INELIGIBLE - 1)


@pytest.mark.parametrize("k", range(len(COLLISIONS)))
def test_committed_pairs_collide(k):
    f1, f2 = COLLISIONS[k]
    assert f1 != f2 and len(set(f1)) == len(set(f2)) == 2, "a frontier lists distinct nodes, and the two must differ"
    assert frontier_signature(f1) == frontier_signature(f2) == EXPECTED[k]
    # the same frontiers in the other order (and the frontiers crossed) are different lists with unrelated signatures
    assert frontier_signature(f1[::-1]) != EXPECTED[k] and frontier_signature(f2[::-1]) != EXPECTED[k]
    assert frontier_signature((f1[0], f2[1])) != EXPECTED[k]


def test_pairs_share_no_node():
    nodes = [v for f1, f2 in COLLISIONS for v in f1 + f2]
    assert len(nodes) == len(set(nodes)) == 4 * len(COLLISIONS)
    assert max(nodes) < 8192


def test_restatements_agree():
    """The generator's numpy form and this scalar form give the same hash, including for the empty frontier and a full one."""
    for f in ((), (0,), (7, 3), tuple(range(8)), (2**31 - 1, 5), COLLISIONS[0][0]):
        assert generator_signature(f) == frontier_signature(f)
    sigs = {frontier_signature(f) for f in ((), (0,), (1,), (0, 1), (1, 0))}
    assert len(sigs) == 5 and all(s < SIG_INELIGIBLE for s in sigs)
