"""ctypes front-end of the NetworkX centrality oracle (nx_oracle.c) and a replay of backend op sequences into a DiGraph.

TEST INFRASTRUCTURE ONLY: the tests pin it on the NetworkX goldens and compare the device with it on estates NetworkX is too slow
for.  Compiled separately from oracle.c, with floating-point contraction off, so that oracle.c's build and outputs are untouched.
"""

from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB_PATH = HERE / "libnxoracle.so"


def build_lib(force: bool = False) -> Path:
    src = HERE / "nx_oracle.c"
    if force or not LIB_PATH.exists() or LIB_PATH.stat().st_mtime < src.stat().st_mtime:
        cmd = ["gcc", "-O3", "-march=native", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", str(LIB_PATH), str(src), "-lm"]
        try:
            subprocess.run(cmd, check=True, capture_output=True, text=True)
        except subprocess.CalledProcessError:
            cmd.remove("-march=native")
            subprocess.run(cmd, check=True, capture_output=True, text=True)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build_lib()
        L = C.CDLL(str(LIB_PATH))
        vp = C.c_void_p
        L.nxo_pagerank.restype, L.nxo_pagerank.argtypes = C.c_int, [C.c_int32, vp, vp, vp, vp]
        L.nxo_betweenness.restype, L.nxo_betweenness.argtypes = C.c_int64, [C.c_int32, vp, vp, vp, vp, vp, C.c_int]
        _lib = L
    return _lib


class DiGraphArrays:
    """Node ids in node order and the forward rows (successors in dict order) with their weights."""

    def __init__(self, ids: list[str], foff: np.ndarray, fnbr: np.ndarray, w: np.ndarray):
        self.ids, self.foff, self.fnbr, self.w = ids, foff, fnbr, w

    @property
    def n(self) -> int:
        return len(self.ids)


def from_succ(succ: dict) -> DiGraphArrays:
    """``succ``: node -> {successor: weight} in the DiGraph's dict orders (every node a key)."""
    ids = list(succ)
    index = {v: i for i, v in enumerate(ids)}
    foff = np.zeros(len(ids) + 1, dtype=np.int64)
    foff[1:] = np.cumsum([len(r) for r in succ.values()])
    fnbr = np.fromiter((index[t] for r in succ.values() for t in r), dtype=np.int32, count=int(foff[-1]))
    w = np.fromiter((float(x) for r in succ.values() for x in r.values()), dtype=np.float64, count=int(foff[-1]))
    return DiGraphArrays(ids, foff, fnbr, w)


def replay(ops) -> DiGraphArrays:
    """Backend op sequence (``["n", id, kind, label, meta]`` / ``["e", s, t, kind, weight, directed, meta]``) replayed with
    nx.DiGraph semantics: endpoints created on first sight, a re-added edge keeps its place and takes the new weight."""
    succ: dict[str, dict[str, float]] = {}

    def edge(s, t, w):
        succ.setdefault(s, {})
        succ.setdefault(t, {})
        succ[s][t] = w

    for op in ops:
        if op[0] == "n":
            succ.setdefault(op[1], {})
        else:
            edge(op[1], op[2], op[4])
            if not op[5]:
                edge(op[2], op[1], op[4])
    return from_succ(succ)


def pagerank(g: DiGraphArrays) -> tuple[np.ndarray, int]:
    out = np.zeros(g.n, dtype=np.float64)
    it = lib().nxo_pagerank(g.n, g.foff.ctypes.data, g.fnbr.ctypes.data, g.w.ctypes.data, out.ctypes.data)
    return out, int(it)


def betweenness(g: DiGraphArrays, threads: int = 0) -> tuple[np.ndarray, int]:
    """Scores in node order and the forward adjacency entries scanned over all sources (the work Brandes' phase 1 does)."""
    row = np.repeat(np.arange(g.n, dtype=np.int32), np.diff(g.foff))
    order = np.argsort(g.fnbr, kind="stable")
    rnbr = np.ascontiguousarray(row[order])
    roff = np.zeros(g.n + 1, dtype=np.int64)
    roff[1:] = np.cumsum(np.bincount(g.fnbr, minlength=g.n))
    out = np.zeros(g.n, dtype=np.float64)
    scanned = lib().nxo_betweenness(g.n, g.foff.ctypes.data, g.fnbr.ctypes.data, roff.ctypes.data, rnbr.ctypes.data, out.ctypes.data, threads)
    return out, int(scanned)
