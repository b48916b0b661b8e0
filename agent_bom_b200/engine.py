"""DeviceGraph — a CSR resident in one H100's HBM plus the batched traversal calls on it.

Thin Python face of the C ABI (include/abb200.h): every method stages its
integer inputs, calls one ``abb_*_host`` entry point (H2D → sm_90a kernels →
D2H inside the library) and wraps the pinned result arrays as numpy.  There is
no CPU path: constructing a DeviceGraph without a CUDA device raises
``EngineUnavailable``.
"""

from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass

import numpy as np

from . import _lib
from .graph.csr import HostCSR
from .graph.schema import ENTITY_VALUES, N_ENTITY_TYPES

_vp = C.c_void_p


class _Owner:
    """Keeps a C result object alive for as long as any numpy view of its pinned host arrays exists."""

    def __init__(self, free, handle):
        self._free, self._handle = free, handle

    def __del__(self):
        try:
            if self._handle:
                self._free(self._handle)
                self._handle = None
        except Exception:
            pass


def _view(ptr, n: int, dtype, owner: _Owner | None = None) -> np.ndarray:
    """``n`` items at a C pointer as a numpy array: a copy by default; with ``owner`` a zero-copy view of the library's
    pinned host block whose buffer object holds a reference to the owner (so the block outlives every slice of it)."""
    if not ptr or n <= 0:
        return np.zeros(max(n, 0), dtype=dtype)
    nbytes = n * np.dtype(dtype).itemsize
    buf = (C.c_char * nbytes).from_address(ptr)
    if owner is None:
        return np.frombuffer(buf, dtype=dtype).copy()
    buf._owner = owner
    arr = np.frombuffer(buf, dtype=dtype)
    arr.flags.writeable = False
    return arr


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


@dataclass
class WalkResult:
    """Ragged result of a batch of traversals.  Slice of query q = ``nodes[start[q] : start[q] + count[q]]``."""

    start: np.ndarray
    count: np.ndarray
    maxd: np.ndarray
    flags: np.ndarray
    nodes: np.ndarray
    parent: np.ndarray | None = None
    depth: np.ndarray | None = None
    estart: np.ndarray | None = None
    ecount: np.ndarray | None = None
    edges: np.ndarray | None = None
    h2d_bytes: int = 0
    d2h_bytes: int = 0
    kernel_ms: float = 0.0
    # entity-type histograms as they crossed PCIe: the columns that are non-zero somewhere in the batch (``hist_cols``), uint16 unless a
    # count needs more; ``hist`` is the dense [n_queries, N_ENTITY_TYPES] uint32 table, built on first access
    hist_packed: np.ndarray | None = None
    hist_cols: np.ndarray | None = None
    _hist: np.ndarray | None = None

    @property
    def hist(self) -> np.ndarray | None:
        if self._hist is None and self.hist_packed is not None:
            dense = np.zeros((len(self), N_ENTITY_TYPES), np.uint32)
            if self.hist_cols.size:
                dense[:, self.hist_cols] = self.hist_packed
            self._hist = dense
        return self._hist

    @hist.setter
    def hist(self, value) -> None:
        self._hist = value

    def __len__(self) -> int:
        return int(self.count.shape[0])

    def slice(self, q: int) -> np.ndarray:
        s = int(self.start[q])
        return self.nodes[s: s + int(self.count[q])]

    def aux(self, q: int, which: str) -> np.ndarray:
        s = int(self.start[q])
        return getattr(self, which)[s: s + int(self.count[q])]

    def edge_slice(self, q: int) -> np.ndarray:
        s = int(self.estart[q])
        return self.edges[s: s + int(self.ecount[q])]

    def hist_dict(self, q: int) -> dict[str, int]:
        if self._hist is None and self.hist_packed is not None:
            return {ENTITY_VALUES[int(t)]: int(c) for t, c in zip(self.hist_cols, self.hist_packed[q]) if c}
        return {ENTITY_VALUES[t]: int(c) for t, c in enumerate(self.hist[q]) if c}


@dataclass
class FindingContext:
    """What the OCSF export's ``graph_context`` needs per finding q, from ``DeviceGraph.finding_context``: the impact walk's
    ``count`` / ``maxd`` / ``flags`` / type histogram (no node slices), and the finding's in-neighbours of the four listed kinds —
    ``sources(q, bucket)`` with ``bucket`` one of ``_lib.CTX_AGENT`` / ``CTX_SERVER`` / ``CTX_PACKAGE`` / ``CTX_CREDENTIAL``, in
    ``reverse_adjacency`` order with duplicates kept."""

    count: np.ndarray
    maxd: np.ndarray
    flags: np.ndarray
    start: np.ndarray              # int64 [n] first source of finding q
    bucket_counts: np.ndarray      # int32 [n, CTX_BUCKETS]
    source_nodes: np.ndarray       # int32, bucket-major within a finding
    h2d_bytes: int = 0
    d2h_bytes: int = 0
    kernel_ms: float = 0.0         # the impact walk's kernels
    context_ms: float = 0.0        # the context kernels (count + fill passes; they overlap the walk on another stream)
    hist_packed: np.ndarray | None = None
    hist_cols: np.ndarray | None = None
    _hist: np.ndarray | None = None

    hist = WalkResult.hist
    hist_dict = WalkResult.hist_dict

    def __len__(self) -> int:
        return int(self.count.shape[0])

    def sources(self, q: int, bucket: int) -> np.ndarray:
        bc = self.bucket_counts[q]
        s = int(self.start[q]) + int(bc[:bucket].sum())
        return self.source_nodes[s: s + int(bc[bucket])]


@dataclass
class PathRows:
    """Exposure-path rows in the reference's emission order (before risk ranking)."""

    off: np.ndarray     # int64 [F+1] rows of finding i = [off[i], off[i+1])
    hops: np.ndarray    # int32 [P,4] agent, server, vulnerable_source (-1 = the server), finding
    rels: np.ndarray    # int8 [P,3]  relationship code per hop pair; -1 no edge; -2 n/a
    ncred: np.ndarray
    ntool: np.ndarray
    h2d_bytes: int = 0
    d2h_bytes: int = 0
    kernel_ms: float = 0.0
    # factorised form (what actually crossed PCIe): rows of finding i = for each link l in [link_off[i], link_off[i+1]):
    # the template rows [link_template[l], +link_row_off[l+1]-link_row_off[l]) of vulnerable source link_source[l]
    link_off: np.ndarray | None = None
    link_source: np.ndarray | None = None
    link_rel: np.ndarray | None = None
    link_row_off: np.ndarray | None = None
    link_template: np.ndarray | None = None
    template: np.ndarray | None = None       # int32 [T,4] agent, server, ncred, ntool
    template_rel: np.ndarray | None = None   # int8 [T,2]


class DeviceGraph:
    """Owns one ``abb_graph`` handle.  Thread-safe (the library serialises use of its workspace)."""

    def __init__(self, handle: int, n_nodes: int, n_entries: int, device: int, keepalive=None):
        self._h = _vp(handle)
        self.n_nodes = n_nodes
        self.n_entries = n_entries
        self.device = device
        self._keepalive = keepalive
        self._lock = threading.Condition()
        self._users = 0          # library calls in flight on this handle (ctypes releases the GIL inside them)
        self._closing = False

    # ── construction ────────────────────────────────────────────────────
    @classmethod
    def upload(cls, csr: HostCSR, device: int = 0) -> "DeviceGraph":
        lib = _lib.load()
        _lib.require_device()
        c = csr.c_struct()
        h = _vp()
        _lib.check(lib.abb_graph_upload(device, C.byref(c), C.byref(h)))
        return cls(h.value, csr.n_nodes, csr.n_entries, device)

    @classmethod
    def adopt(cls, tensors: dict, n_nodes: int, n_entries: int, device: int) -> "DeviceGraph":
        """Wrap device arrays owned by the caller (torch tensors, e.g. after an NCCL broadcast)."""
        lib = _lib.load()
        _lib.require_device()
        c = _lib.Csr()
        c.n_nodes, c.n_entries = n_nodes, n_entries
        for name in ("fwd_off", "fwd_nbr", "fwd_meta", "fwd_eid", "rev_off", "rev_nbr", "rev_meta", "rev_eid", "node_type", "node_rank"):
            t = tensors.get(name)
            setattr(c, name, t.data_ptr() if t is not None else None)
        h = _vp()
        _lib.check(lib.abb_graph_adopt(device, C.byref(c), C.byref(h)))
        return cls(h.value, n_nodes, n_entries, device, keepalive=tensors)

    def close(self) -> None:
        """Free the device graph.  Waits for library calls still running on other threads (a REST worker inside a traversal
        while another thread re-saves the snapshot): the handle is never freed under a caller."""
        with self._lock:
            if not self._h:
                return
            self._closing = True
            while self._users:
                self._lock.wait()
            h, self._h = self._h, None
        _lib.load().abb_graph_free(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        """The raw handle, for calls made while the caller otherwise guarantees the graph stays open."""
        if not self._h:
            raise RuntimeError("DeviceGraph is closed")
        return self._h

    class _Use:
        def __init__(self, dg):
            self.dg = dg

        def __enter__(self):
            dg = self.dg
            with dg._lock:
                if not dg._h or dg._closing:
                    raise RuntimeError("DeviceGraph is closed")
                dg._users += 1
            return dg._h

        def __exit__(self, *exc):
            dg = self.dg
            with dg._lock:
                dg._users -= 1
                if not dg._users:
                    dg._lock.notify_all()

    def _use(self):
        """Context manager around a library call: pins the handle against a concurrent ``close()``."""
        return DeviceGraph._Use(self)

    def set_dedup(self, enabled: bool) -> None:
        """Toggle root-frontier de-duplication of single-source batches (results are identical either way)."""
        _lib.check(_lib.load().abb_graph_set_dedup(self.handle, int(bool(enabled))))

    def set_option(self, name: str, value: int) -> None:
        """Tuning / test switch of the handle (``abb_graph_set_option``): block_tiers, mid_qcap, big_qcap, dedup, zero_copy."""
        _lib.check(_lib.load().abb_graph_set_option(self.handle, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        return int(_lib.load().abb_graph_get_option(self.handle, name.encode()))

    @property
    def nbytes(self) -> int:
        return int(_lib.load().abb_graph_bytes(self.handle))

    # ── specs (reference function -> walk spec; the mapping lives in the C library) ──
    @staticmethod
    def spec_impact_of(max_depth: int = 4):
        return _lib.load().abb_spec_impact_of(max_depth)

    @staticmethod
    def spec_bfs(max_depth: int = 4, traversable_only: bool = True):
        return _lib.load().abb_spec_bfs(max_depth, int(traversable_only))

    @staticmethod
    def spec_reachable_from(max_depth: int = 6, traversable_only: bool = False):
        return _lib.load().abb_spec_reachable_from(max_depth, int(traversable_only))

    @staticmethod
    def spec_shortest_path():
        return _lib.load().abb_spec_shortest_path()

    @staticmethod
    def spec_traverse(direction: int, max_depth: int, max_nodes: int, max_edges: int, traversable_only: bool, rel_mask: int,
                      static_only: bool, dynamic_only: bool, include_roots: bool):
        return _lib.load().abb_spec_traverse_subgraph(direction, max_depth, max_nodes, max_edges, int(traversable_only), rel_mask & 0xFFFFFFFF,
                                                      int(static_only), int(dynamic_only), int(include_roots))

    @staticmethod
    def spec_distances(rel_mask: int, emit_types: int = 0xFFFFFFFF):
        return _lib.load().abb_spec_distances_along(rel_mask & 0xFFFFFFFF, emit_types & 0xFFFFFFFF)

    # ── batched walk ────────────────────────────────────────────────────
    def walk(self, spec, roots, root_off=None, targets=None, zero_copy: bool = False) -> WalkResult:
        """One batched traversal through the host-buffer C call.  ``zero_copy=True`` returns read-only numpy views of the
        library's pinned result blocks instead of copies (the blocks are recycled when the last view is dropped)."""
        lib = _lib.load()
        roots = _i32(roots)
        if root_off is not None:
            root_off = np.ascontiguousarray(root_off, dtype=np.int64)
            nq = int(root_off.shape[0]) - 1
        else:
            nq = int(roots.shape[0])
        tg = _i32(targets) if targets is not None else None
        res = _vp()
        with self._use() as h:
            _lib.check(lib.abb_walk_host(h, C.byref(spec), roots.ctypes.data, root_off.ctypes.data if root_off is not None else None,
                                         tg.ctypes.data if tg is not None else None, nq, C.byref(res)))
        if zero_copy:
            out = self._collect_walk(res, spec.flags, _Owner(lib.abb_walk_result_free, res))
        else:
            try:
                out = self._collect_walk(res, spec.flags)
            finally:
                lib.abb_walk_result_free(res)
        out.kernel_ms = float(lib.abb_last_walk_ms(self.handle))
        return out

    @staticmethod
    def _collect_walk(res, flags: int, owner: _Owner | None = None) -> WalkResult:
        lib = _lib.load()
        nq = int(lib.abb_walk_result_queries(res))
        tn = int(lib.abb_walk_result_total_nodes(res))
        te = int(lib.abb_walk_result_total_edges(res))
        out = WalkResult(
            start=_view(lib.abb_walk_result_start(res), nq, np.int64, owner), count=_view(lib.abb_walk_result_count(res), nq, np.int32, owner),
            maxd=_view(lib.abb_walk_result_maxd(res), nq, np.int32, owner), flags=_view(lib.abb_walk_result_flags(res), nq, np.int32, owner),
            nodes=_view(lib.abb_walk_result_nodes(res), tn, np.int32, owner),
            h2d_bytes=int(lib.abb_walk_result_h2d_bytes(res)), d2h_bytes=int(lib.abb_walk_result_d2h_bytes(res)),
        )
        if flags & _lib.WALK_PARENTS:
            out.parent = _view(lib.abb_walk_result_parent(res), tn, np.int32, owner)
        if flags & _lib.WALK_DEPTHS:
            out.depth = _view(lib.abb_walk_result_depth(res), tn, np.int32, owner)
        if flags & _lib.WALK_HIST:
            mask, width = C.c_uint32(0), C.c_int32(0)
            packed = lib.abb_walk_result_hist_packed(res, C.byref(mask), C.byref(width))
            if packed:
                cols = np.array([t for t in range(N_ENTITY_TYPES) if mask.value >> t & 1], dtype=np.int64)
                out.hist_cols = cols
                dt = np.uint16 if width.value == 2 else np.uint32
                out.hist_packed = (_view(packed, nq * len(cols), dt, owner) if len(cols) else np.zeros(0, dt)).reshape(nq, len(cols))
            else:
                out.hist = _view(lib.abb_walk_result_hist(res), nq * N_ENTITY_TYPES, np.uint32, owner).reshape(nq, N_ENTITY_TYPES)
        if flags & _lib.WALK_EDGES:
            out.estart = _view(lib.abb_walk_result_estart(res), nq, np.int64, owner)
            out.ecount = _view(lib.abb_walk_result_ecount(res), nq, np.int64, owner)
            out.edges = _view(lib.abb_walk_result_edges(res), te, np.uint32, owner)
        return out

    # convenience wrappers named after the reference functions
    def impact_many(self, sources, max_depth: int = 4) -> WalkResult:
        return self.walk(self.spec_impact_of(max_depth), sources)

    def bfs_many(self, sources, max_depth: int = 4, traversable_only: bool = True) -> WalkResult:
        return self.walk(self.spec_bfs(max_depth, traversable_only), sources)

    def reachable_many(self, sources, max_depth: int = 6, traversable_only: bool = False) -> WalkResult:
        return self.walk(self.spec_reachable_from(max_depth, traversable_only), sources)

    def shortest_path_many(self, sources, targets) -> WalkResult:
        return self.walk(self.spec_shortest_path(), sources, targets=targets)

    # ── exposure-path rows ──────────────────────────────────────────────
    @staticmethod
    def _collect_paths(res, nf: int, owner: _Owner | None = None, expand: bool = True) -> PathRows:
        """``expand=False`` leaves the flat row arrays empty (only the factorised form — what crossed PCIe — is wrapped)."""
        lib = _lib.load()
        rows = int(lib.abb_paths_result_rows(res))
        nl, nt = int(lib.abb_paths_result_links(res)), int(lib.abb_paths_result_template_rows(res))
        if expand:
            hops = _view(lib.abb_paths_result_hops(res), rows * 4, np.int32, owner).reshape(rows, 4)
            rels = np.ascontiguousarray(_view(lib.abb_paths_result_rels(res), rows * 4, np.int8, owner).reshape(rows, 4)[:, :3])
            ncred, ntool = _view(lib.abb_paths_result_ncred(res), rows, np.int32, owner), _view(lib.abb_paths_result_ntool(res), rows, np.int32, owner)
        else:
            hops, rels = np.zeros((0, 4), np.int32), np.zeros((0, 3), np.int8)
            ncred = ntool = np.zeros(0, np.int32)
        return PathRows(
            off=_view(lib.abb_paths_result_off(res), nf + 1, np.int64, owner), hops=hops, rels=rels, ncred=ncred, ntool=ntool,
            h2d_bytes=int(lib.abb_paths_result_h2d_bytes(res)), d2h_bytes=int(lib.abb_paths_result_d2h_bytes(res)),
            link_off=_view(lib.abb_paths_result_link_off(res), nf + 1, np.int64, owner),
            link_source=_view(lib.abb_paths_result_link_source(res), nl, np.int32, owner),
            link_rel=_view(lib.abb_paths_result_link_rel(res), nl, np.int8, owner),
            link_row_off=_view(lib.abb_paths_result_link_row_off(res), nl + 1, np.int64, owner),
            link_template=_view(lib.abb_paths_result_link_template(res), nl, np.int64, owner),
            template=_view(lib.abb_paths_result_template(res), nt * 4, np.int32, owner).reshape(-1, 4),
            template_rel=_view(lib.abb_paths_result_template_rel(res), nt * 2, np.int8, owner).reshape(-1, 2),
        )

    def exposure_paths_many(self, findings) -> PathRows:
        lib = _lib.load()
        f = _i32(findings)
        res = _vp()
        with self._use() as h:
            _lib.check(lib.abb_paths_host(h, f.ctypes.data, int(f.shape[0]), C.byref(res)))
        try:
            out = self._collect_paths(res, int(f.shape[0]))
        finally:
            lib.abb_paths_result_free(res)
        out.kernel_ms = float(lib.abb_last_paths_ms(self.handle))
        return out

    def exposure_many(self, findings, max_depth: int = 4, collect: bool = True, zero_copy: bool = False):
        """One exposure traversal per finding: impact_of + derived exposure-path rows (BASELINE.json's unit of work).

        ``zero_copy=True``: read-only numpy views of the pinned result blocks, exposure-path rows in their factorised form
        (links + templates; ``PathRows.hops`` etc. stay empty — expand with ``exposure_paths_many`` or from the factors)."""
        lib = _lib.load()
        f = _i32(findings)
        wres, pres = _vp(), _vp()
        with self._use() as h:
            _lib.check(lib.abb_exposure_host(h, f.ctypes.data, int(f.shape[0]), max_depth, C.byref(wres), C.byref(pres)))
        if zero_copy:
            w = self._collect_walk(wres, _lib.WALK_HIST, _Owner(lib.abb_walk_result_free, wres))
            p = self._collect_paths(pres, int(f.shape[0]), _Owner(lib.abb_paths_result_free, pres), expand=False)
            return w, p
        try:
            if collect:
                w = self._collect_walk(wres, _lib.WALK_HIST)
                p = self._collect_paths(pres, int(f.shape[0]))
            else:  # bench: results are already in pinned host memory; report sizes only
                w = (int(lib.abb_walk_result_total_nodes(wres)), int(lib.abb_walk_result_h2d_bytes(wres)), int(lib.abb_walk_result_d2h_bytes(wres)))
                p = (int(lib.abb_paths_result_rows(pres)), int(lib.abb_paths_result_h2d_bytes(pres)), int(lib.abb_paths_result_d2h_bytes(pres)))
        finally:
            lib.abb_walk_result_free(wres)
            lib.abb_paths_result_free(pres)
        return w, p

    def finding_context(self, findings, max_depth: int = 4) -> FindingContext:
        """Per finding: ``impact_of``'s count, depth, flags and type histogram plus its typed in-neighbour lists
        (``abb_finding_context_host``).  The walk's node slices stay on the device."""
        lib = _lib.load()
        f = _i32(findings)
        nq = int(f.shape[0])
        res = _vp()
        with self._use() as h:
            _lib.check(lib.abb_finding_context_host(h, int(max_depth), f.ctypes.data, nq, C.byref(res)))
        try:
            total = int(lib.abb_finding_context_result_total_sources(res))
            out = FindingContext(
                count=_view(lib.abb_finding_context_result_count(res), nq, np.int32), maxd=_view(lib.abb_finding_context_result_maxd(res), nq, np.int32),
                flags=_view(lib.abb_finding_context_result_flags(res), nq, np.int32), start=_view(lib.abb_finding_context_result_start(res), nq, np.int64),
                bucket_counts=_view(lib.abb_finding_context_result_bucket_counts(res), nq * _lib.CTX_BUCKETS, np.int32).reshape(nq, _lib.CTX_BUCKETS),
                source_nodes=_view(lib.abb_finding_context_result_sources(res), total, np.int32),
                h2d_bytes=int(lib.abb_finding_context_result_h2d_bytes(res)), d2h_bytes=int(lib.abb_finding_context_result_d2h_bytes(res)),
                kernel_ms=float(lib.abb_finding_context_result_walk_ms(res)), context_ms=float(lib.abb_finding_context_result_context_ms(res)),
            )
            mask, width = C.c_uint32(0), C.c_int32(0)
            packed = lib.abb_finding_context_result_hist_packed(res, C.byref(mask), C.byref(width))
            if packed:
                cols = np.array([t for t in range(N_ENTITY_TYPES) if mask.value >> t & 1], dtype=np.int64)
                dt = np.uint16 if width.value == 2 else np.uint32
                out.hist_cols = cols
                out.hist_packed = (_view(packed, nq * len(cols), dt) if len(cols) else np.zeros(0, dt)).reshape(nq, len(cols))
            else:
                out.hist = _view(lib.abb_finding_context_result_hist(res), nq * N_ENTITY_TYPES, np.uint32).reshape(nq, N_ENTITY_TYPES)
            return out
        finally:
            lib.abb_finding_context_result_free(res)

    def rank_exposure_paths(self, findings, base_id, risk_rank, ncu, ntu, offset: int = 0, limit: int = 100):
        """Page [offset, offset+limit) of the exposure-path rows in the reference's ranking order; returns (PathRows-like, risk_rank, total)."""
        rows, rank, total, _matched = self.rank_exposure_paths_focused(findings, base_id, risk_rank, ncu, ntu, None, 0, offset, limit)
        return rows, rank, total

    def rank_exposure_paths_focused(self, findings, base_id, risk_rank, ncu, ntu, node_focus, need: int, offset: int = 0, limit: int = 100):
        """Like ``rank_exposure_paths``, restricted to the rows whose hops carry every focus category in ``need``
        (``node_focus``: uint8 ``_lib.FOCUS_*`` bits per node, ``None`` = every row).  The page is taken from the matched rows in
        ranking order; returns (PathRows-like, risk_rank, total rows, matched rows)."""
        lib = _lib.load()
        f, b = _i32(findings), _i32(base_id)
        table = np.ascontiguousarray(risk_rank, dtype=np.uint32)
        cu, tu = _i32(ncu), _i32(ntu)
        assert table.size % 75 == 0 and cu.shape[0] == self.n_nodes and tu.shape[0] == self.n_nodes and b.shape[0] == f.shape[0]
        focus = None if node_focus is None else np.ascontiguousarray(node_focus, dtype=np.uint8)
        assert focus is None or focus.shape[0] == self.n_nodes
        res = _vp()
        with self._use() as h:
            if focus is None:
                _lib.check(lib.abb_paths_rank_host(h, f.ctypes.data, int(f.shape[0]), b.ctypes.data, table.ctypes.data, table.size // 75, cu.ctypes.data,
                                                   tu.ctypes.data, int(offset), int(limit), C.byref(res)))
            else:
                _lib.check(lib.abb_paths_rank_focus_host(h, f.ctypes.data, int(f.shape[0]), b.ctypes.data, table.ctypes.data, table.size // 75,
                                                         cu.ctypes.data, tu.ctypes.data, focus.ctypes.data, int(need), int(offset), int(limit), C.byref(res)))
        try:
            k = int(lib.abb_rank_result_count(res))
            rows = PathRows(
                off=np.zeros(0, dtype=np.int64), hops=_view(lib.abb_rank_result_hops(res), k * 4, np.int32).reshape(k, 4),
                rels=np.ascontiguousarray(_view(lib.abb_rank_result_rels(res), k * 4, np.int8).reshape(k, 4)[:, :3]),
                ncred=_view(lib.abb_rank_result_ncred(res), k, np.int32), ntool=_view(lib.abb_rank_result_ntool(res), k, np.int32),
            )
            return rows, _view(lib.abb_rank_result_risk_rank(res), k, np.uint32), int(lib.abb_rank_result_total(res)), int(lib.abb_rank_result_matched(res))
        finally:
            lib.abb_rank_result_free(res)

    # ── dependency reach ────────────────────────────────────────────────
    def dependency_reach(self, agents, rel_mask: int, vuln_pkg_mask: int) -> dict:
        lib = _lib.load()
        a = _i32(agents)
        res = _vp()
        with self._use() as h:
            _lib.check(lib.abb_dependency_reach_host(h, a.ctypes.data, int(a.shape[0]), rel_mask & 0xFFFFFFFF, vuln_pkg_mask & 0xFFFFFFFF, C.byref(res)))
        try:
            npk = int(lib.abb_reach_n_packages(res))
            nv = int(lib.abb_reach_n_vulns(res))
            pkg_off = _view(lib.abb_reach_pkg_off(res), npk + 1, np.int64)
            vpo = _view(lib.abb_reach_vuln_poff(res), nv + 1, np.int64)
            vao = _view(lib.abb_reach_vuln_aoff(res), nv + 1, np.int64)
            return dict(
                pkg_ids=_view(lib.abb_reach_pkg_ids(res), npk, np.int32), pkg_off=pkg_off,
                pkg_agents=_view(lib.abb_reach_pkg_agents(res), int(pkg_off[-1]) if npk else 0, np.int32),
                pkg_minhop=_view(lib.abb_reach_pkg_minhop(res), npk, np.int32),
                vuln_ids=_view(lib.abb_reach_vuln_ids(res), nv, np.int32), vuln_poff=vpo,
                vuln_pkgs=_view(lib.abb_reach_vuln_pkgs(res), int(vpo[-1]) if nv else 0, np.int32), vuln_aoff=vao,
                vuln_agents=_view(lib.abb_reach_vuln_agents(res), int(vao[-1]) if nv else 0, np.int32),
                vuln_minhop=_view(lib.abb_reach_vuln_minhop(res), nv, np.int32),
            )
        finally:
            lib.abb_reach_result_free(res)

    # ── sampled bottleneck score ────────────────────────────────────────
    def bottleneck_scores(self, sources) -> np.ndarray:
        """uint64 per node: over all sources, the number of BFS-tree paths the node lies strictly inside (``abb_bottleneck_host``)."""
        src = _i32(sources)
        out = np.zeros(self.n_nodes, dtype=np.uint64)
        with self._use() as h:
            _lib.check(_lib.load().abb_bottleneck_host(h, src.ctypes.data, int(src.shape[0]), out.ctypes.data))
        return out

    # ── NetworkX analysis backend ───────────────────────────────────────
    def pagerank(self, weights) -> tuple[np.ndarray, int]:
        """``nx.pagerank`` of the graph as a DiGraph (``abb_pagerank_host``): f64 score per node and the power iterations run.
        ``weights``: f64 edge weight per forward adjacency entry."""
        w = np.ascontiguousarray(weights, dtype=np.float64)
        if w.shape[0] != self.n_entries:
            raise ValueError("pagerank needs one weight per adjacency entry")
        out = np.zeros(self.n_nodes, dtype=np.float64)
        iters = C.c_int32(0)
        with self._use() as h:
            _lib.check(_lib.load().abb_pagerank_host(h, w.ctypes.data, out.ctypes.data, C.byref(iters)))
        return out, int(iters.value)

    def build_clusters(self, k: int, codes, level, risk, etype) -> dict[str, np.ndarray]:
        """Build the graph's semantic-cluster tables (``abb_clusters_build_host``), replacing earlier ones, and return the per-cluster
        summaries: ``count``, ``max_risk``, ``hist`` [k, 5], ``type_mask`` and ``rel_nnz``.  ``codes``: int32 [n_nodes, 2]
        (-1 = none); ``level`` / ``risk`` / ``etype``: per node."""
        n = self.n_nodes
        codes = np.ascontiguousarray(codes, dtype=np.int32).reshape(n, 2)
        level = np.ascontiguousarray(level, dtype=np.uint8)
        risk = np.ascontiguousarray(risk, dtype=np.float64)
        etype = np.ascontiguousarray(etype, dtype=np.uint8)
        if level.shape != (n,) or risk.shape != (n,) or etype.shape != (n,):
            raise ValueError("cluster inputs need one entry per node")
        out = {"count": np.zeros(k, np.int64), "max_risk": np.zeros(k, np.float64), "hist": np.zeros((k, 5), np.int64),
               "type_mask": np.zeros(k, np.uint64), "rel_nnz": np.zeros(k, np.int64)}
        with self._use() as h:
            _lib.check(_lib.load().abb_clusters_build_host(h, k, codes.ctypes.data, level.ctypes.data, risk.ctypes.data, etype.ctypes.data,
                                                           *(out[f].ctypes.data for f in ("count", "max_risk", "hist", "type_mask", "rel_nnz"))))
        return out

    def fetch_clusters(self, sel, n_members: int, n_pairs: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Members (node indices in id order) and (relationship code, edge count) pairs of the selected clusters, concatenated in
        selection order (``abb_clusters_fetch_host``); the caller sizes the outputs from the build's ``count`` and ``rel_nnz``."""
        sel = _i32(sel)
        members = np.empty(n_members, np.int32)
        rel = np.empty(n_pairs, np.uint8)
        cnt = np.empty(n_pairs, np.int64)
        with self._use() as h:
            _lib.check(_lib.load().abb_clusters_fetch_host(h, sel.shape[0], sel.ctypes.data, members.ctypes.data, rel.ctypes.data, cnt.ctypes.data))
        return members, rel, cnt

    def build_delta_table(self, n_real: int, ids: bytes, id_off, perm, labels: bytes, label_off, status, severity, risk, erel, eflag, weight=None) -> None:
        """Store the graph's snapshot-diff tables (``abb_delta_table_host``), replacing earlier ones; freed with the graph."""
        id_off, label_off = np.ascontiguousarray(id_off, np.int64), np.ascontiguousarray(label_off, np.int64)
        perm = _i32(perm)
        status, severity = np.ascontiguousarray(status, np.uint8), np.ascontiguousarray(severity, np.uint8)
        risk = np.ascontiguousarray(risk, np.float64)
        erel, eflag = np.ascontiguousarray(erel, np.uint8), np.ascontiguousarray(eflag, np.uint8)
        if weight is not None:
            weight = np.ascontiguousarray(weight, np.float64)
        if id_off.shape != (self.n_nodes + 1,) or perm.shape != (self.n_nodes,) or label_off.shape != (n_real + 1,) or \
                status.shape != (n_real,) or severity.shape != (n_real,) or risk.shape != (n_real,) or eflag.shape != erel.shape or \
                (weight is not None and weight.shape != erel.shape):
            raise ValueError("delta table inputs have the wrong shapes")
        ids_buf = np.frombuffer(ids, np.uint8) if ids else np.zeros(1, np.uint8)
        lbl_buf = np.frombuffer(labels, np.uint8) if labels else np.zeros(1, np.uint8)
        with self._use() as h:
            _lib.check(_lib.load().abb_delta_table_host(h, n_real, ids_buf.ctypes.data, id_off.ctypes.data, perm.ctypes.data, lbl_buf.ctypes.data,
                                                        label_off.ctypes.data, status.ctypes.data, severity.ctypes.data, risk.ctypes.data, erel.shape[0],
                                                        erel.ctypes.data, eflag.ctypes.data, None if weight is None else weight.ctypes.data))

    def delta_table_bytes(self) -> int:
        with self._use() as h:
            return int(_lib.load().abb_delta_table_bytes(h))

    def diff(self, old: "DeviceGraph", relmap_old, relmap_new) -> dict[str, np.ndarray]:
        """Diff ``old`` -> this graph on the device (``abb_delta_build_host`` + ``abb_delta_fetch_host``); both need delta tables.
        Returns ``nodes_added`` (this graph's indices) / ``nodes_removed`` (old's) in id order, ``changed_new`` / ``changed_old`` /
        ``changed_flag`` node pairs in id order, ``edges_added`` / ``edges_removed`` edge indices and ``echanged_new`` /
        ``echanged_old`` edge pairs in (source, target, relationship) order."""
        rm_old = np.zeros(64, np.uint8)
        rm_new = np.zeros(64, np.uint8)
        rm_old[: len(relmap_old)] = relmap_old
        rm_new[: len(relmap_new)] = relmap_new
        sizes = np.zeros(6, np.int64)
        lib = _lib.load()
        res = _vp()
        with self._use() as h, old._use() as ho:
            _lib.check(lib.abb_delta_build_host(ho, h, rm_old.ctypes.data, rm_new.ctypes.data, C.byref(res), sizes.ctypes.data))
        try:
            na, nr, nc, ea, er, ec = (int(x) for x in sizes)
            out = {"nodes_added": np.empty(na, np.int32), "nodes_removed": np.empty(nr, np.int32), "changed_new": np.empty(nc, np.int32),
                   "changed_old": np.empty(nc, np.int32), "changed_flag": np.empty(nc, np.uint8), "edges_added": np.empty(ea, np.int32),
                   "edges_removed": np.empty(er, np.int32), "echanged_new": np.empty(ec, np.int32), "echanged_old": np.empty(ec, np.int32)}
            _lib.check(lib.abb_delta_fetch_host(res, *(out[k].ctypes.data for k in ("nodes_added", "nodes_removed", "changed_new", "changed_old", "changed_flag",
                                                                                     "edges_added", "edges_removed", "echanged_new", "echanged_old"))))
        finally:
            lib.abb_delta_result_free(res)
        return out

    def betweenness(self) -> np.ndarray:
        """``nx.betweenness_centrality`` of the graph as a DiGraph (``abb_betweenness_host``): f64 per node."""
        out = np.zeros(self.n_nodes, dtype=np.float64)
        with self._use() as h:
            _lib.check(_lib.load().abb_betweenness_host(h, out.ctypes.data))
        return out

    def bidirectional_paths(self, sources, targets) -> list[np.ndarray | None]:
        """``nx.shortest_path(G, s, t)`` per pair (``abb_bidir_paths_host``): node indices source first, ``None`` when there is no path."""
        lib = _lib.load()
        s, t = _i32(sources), _i32(targets)
        if s.shape != t.shape:
            raise ValueError("sources and targets differ in length")
        res = _vp()
        with self._use() as h:
            _lib.check(lib.abb_bidir_paths_host(h, s.ctypes.data, t.ctypes.data, int(s.shape[0]), C.byref(res)))
        try:
            n = int(s.shape[0])
            start = _view(lib.abb_bidir_result_start(res), n, np.int64)
            length = _view(lib.abb_bidir_result_length(res), n, np.int32)
            nodes = _view(lib.abb_bidir_result_nodes(res), int(lib.abb_bidir_result_total(res)), np.int32)
        finally:
            lib.abb_bidir_result_free(res)
        return [nodes[a: a + k] if k else None for a, k in zip(start.tolist(), length.tolist())]

    # ── timing hooks used by bench.py ───────────────────────────────────
    def last_walk_ms(self) -> float:
        return float(_lib.load().abb_last_walk_ms(self.handle))

    def last_walk_stats(self) -> dict:
        """Sharing statistics of the most recent walk: how many sources collapsed into how many traversals."""
        out = (C.c_int64 * 4)()
        _lib.check(_lib.load().abb_last_walk_stats(self.handle, out))
        return {"queries": int(out[0]), "groups": int(out[1]), "individual": int(out[2]), "eligible": int(out[3])}

    def last_walk_tier_counts(self) -> dict:
        """Queries each storage tier of the most recent walk handed to the next tier (first pass / individual pass)."""
        out = (C.c_int64 * 8)()
        _lib.check(_lib.load().abb_last_walk_tier_counts(self.handle, out))
        names = ("s1", "s1_heavy", "mid", "g1")
        return {"first": dict(zip(names, [int(x) for x in out[0:4]])), "individual": dict(zip(names, [int(x) for x in out[4:8]]))}

    def last_paths_ms(self) -> float:
        return float(_lib.load().abb_last_paths_ms(self.handle))


def group_union(member_off, members, item_off, items, w0=None, w1=None, *, device: int = 0):
    """Per group: sorted de-duplicated union of its members' item lists and the maxima of two per-member byte weights
    (``abb_group_union_host``; the device reduction behind effective-reach scoring).  Returns ``(off, items, w0max, w1max, ms)``."""
    lib = _lib.load()
    moff = np.ascontiguousarray(member_off, dtype=np.int64)
    mem = _i32(members)
    ioff = np.ascontiguousarray(item_off, dtype=np.int64)
    it = _i32(items)
    n_groups, n_members = int(moff.shape[0]) - 1, int(ioff.shape[0]) - 1
    if n_groups < 0 or n_members < 0:
        raise ValueError("offset arrays need at least one entry")
    a0 = np.ascontiguousarray(w0, dtype=np.uint8) if w0 is not None else None
    a1 = np.ascontiguousarray(w1, dtype=np.uint8) if w1 is not None else None
    for w in (a0, a1):
        if w is not None and int(w.shape[0]) != n_members:
            raise ValueError("weights must have one byte per member")
    res = _vp()
    _lib.check(lib.abb_group_union_host(device, n_groups, moff.ctypes.data, mem.ctypes.data, n_members, ioff.ctypes.data, it.ctypes.data,
                                        a0.ctypes.data if a0 is not None else None, a1.ctypes.data if a1 is not None else None, C.byref(res)))
    try:
        off = _view(lib.abb_union_result_off(res), n_groups + 1, np.int64)          # _view copies out of the result object
        out = _view(lib.abb_union_result_items(res), int(off[-1]), np.int32)
        g0 = _view(lib.abb_union_result_w0(res), n_groups, np.uint8)
        g1 = _view(lib.abb_union_result_w1(res), n_groups, np.uint8)
        return off, out, g0, g1, float(lib.abb_union_result_ms(res))
    finally:
        lib.abb_union_result_free(res)
