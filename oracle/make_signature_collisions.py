"""Find pairs of two-node depth-1 frontiers whose de-duplication signatures collide (dedup.cuh ``dedup_sig_kernel``).

A single-source walk batch groups its sources by a 47-bit hash of their ordered level-1 frontier S' and verifies each group
element-wise; a member whose S' differs from its group head's is walked on its own.  Forcing that path needs two different
frontiers with the same hash.  This birthday search restates the hash in numpy and hashes every ordered frontier (a, b) with
a != b and both below ``--ids``; at 8192 ids that is 67 M frontiers and about 16 expected colliding pairs.  The search is
exhaustive and therefore deterministic: ``--seed`` only picks which of the pairs found are printed when ``--pairs`` asks for
fewer, so a test can take a reproducible sample.

    python oracle/make_signature_collisions.py                  # every colliding pair below 8192
    python oracle/make_signature_collisions.py --pairs 8        # 8 of them whose 32 node ids are all distinct

tests/test_dedup_signatures.py holds the committed constants; it checks them against the same restatement on the CPU, and the
GPU tests check the restatement against the device.
"""

from __future__ import annotations

import argparse

import numpy as np

SIG_BITS = 48
SIG_MASK = (1 << (SIG_BITS - 1)) - 1          # signatures live in the low 47 bits; bit 47 marks an ineligible source
SEED = 0xABB200


def mix64(x: np.ndarray) -> np.ndarray:
    """splitmix64's finaliser on uint64 arrays (wrapping arithmetic, as on the device)."""
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def signature(frontier) -> int:
    """The 47-bit signature of one ordered frontier (node ids), as ``dedup_sig_kernel`` computes it for an eligible source."""
    with np.errstate(over="ignore"):
        h = mix64(np.array([SEED + len(frontier)], dtype=np.uint64))
        for i, v in enumerate(frontier):
            h = mix64(h ^ np.uint64((int(v) & 0xFFFFFFFF) + ((i + 1) << 32)))
    return int(h[0]) & SIG_MASK


def pair_signatures(a0: int, a1: int, ids: int) -> np.ndarray:
    """Signatures of every frontier (a, b), a in [a0, a1), b in [0, ids), row-major."""
    with np.errstate(over="ignore"):
        h = mix64(np.full(a1 - a0, SEED + 2, dtype=np.uint64))
        h = mix64(h ^ (np.arange(a0, a1, dtype=np.uint64) + np.uint64(1 << 32)))
        b = np.arange(ids, dtype=np.uint64) + np.uint64(2 << 32)
        return mix64(h[:, None] ^ b[None, :]) & np.uint64(SIG_MASK)


def search(ids: int, block: int = 512) -> list[tuple[tuple[int, int], tuple[int, int]]]:
    """Every pair of distinct two-node frontiers (a, b), (c, d) with a != b, c != d, all ids below `ids`, and equal signatures."""
    sigs = np.concatenate([pair_signatures(a0, min(a0 + block, ids), ids).ravel() for a0 in range(0, ids, block)])
    s = np.sort(sigs)
    dup = np.unique(s[1:][s[1:] == s[:-1]])
    del s
    hits: dict[int, list[tuple[int, int]]] = {}
    for k in np.flatnonzero(np.isin(sigs, dup)).tolist():
        a, b = divmod(k, ids)
        if a != b:
            hits.setdefault(int(sigs[k]), []).append((a, b))
    out = []
    for fronts in hits.values():
        for i in range(len(fronts)):
            for j in range(i + 1, len(fronts)):
                out.append((fronts[i], fronts[j]))
    return sorted(out)


def disjoint_sample(pairs, n: int, seed: int):
    """Up to `n` pairs, in a seeded order, no two of which share a node id."""
    used: set[int] = set()
    out = []
    for k in np.random.default_rng(seed).permutation(len(pairs)).tolist():
        f1, f2 = pairs[k]
        nodes = set(f1) | set(f2)
        if len(nodes) == 4 and not nodes & used:
            used |= nodes
            out.append(pairs[k])
        if len(out) == n:
            break
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--ids", type=int, default=8192, help="node ids of both frontier elements are below this")
    ap.add_argument("--pairs", type=int, default=0, help="print only this many pairs with disjoint node ids (0: all)")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    pairs = search(args.ids)
    if args.pairs:
        pairs = disjoint_sample(pairs, args.pairs, args.seed)
    for f1, f2 in pairs:
        assert signature(f1) == signature(f2) and f1 != f2
        print(f"    ({f1}, {f2}),   # {signature(f1):#x}")


if __name__ == "__main__":
    main()
