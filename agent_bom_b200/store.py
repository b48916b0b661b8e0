"""B200GraphStore — GraphStoreProtocol drop-in whose traversal methods run on the GPU.

Boundary (SURVEY.md §8b): the reference's REST / MCP graph surfaces talk to a
``GraphStoreProtocol`` object (``/root/reference/src/agent_bom/api/graph_store.py:102-256``)
chosen in ``api/stores.py:437-465`` (``set_graph_store(store)``).  This class
implements the traversal subset natively — ``bfs_paths`` (:182-190),
``impact_of`` (:192-199), ``traverse_subgraph`` (:201-217),
``attack_paths_for_sources`` (:219-225), ``attack_paths`` (:227-234) — with the
in-memory engine's semantics (what ``PostgresGraphStore`` does by delegation,
``api/postgres_graph.py:864-931``) and forwards every other method
(snapshots, search, presets, diffs …) to a wrapped default store.

Conventions kept: keyword-only arguments; a missing snapshot / node yields
``None`` / ``([], set())`` / an empty graph, never an exception; methods are
thread-safe (REST calls arrive on worker threads via ``asyncio.to_thread``).
Batched extensions (``impact_of_many``, ``exposure_paths_many``,
``fix_first_view``, ``ocsf_events``, ``dependency_reach``) expose what a GPU is actually good at.
"""

from __future__ import annotations

import threading
from typing import Any

from .graph.clusters import semantic_clusters_view
from .graph.container import UnifiedGraph
from .graph.dependency_reach import ReachabilityReport, compute_dependency_reach
from .graph.exposure import exposure_path_rows, materialize_attack_paths, ranked_attack_paths
from .graph.fix_first import fix_first_view
from .graph.ocsf import iter_ocsf_events


class B200UnsupportedOperationError(NotImplementedError):
    """Raised for store operations this backend does not implement and has no inner store to delegate to
    (the Neptune adapter's convention: reference api/neptune_graph.py:26-27, 408-411)."""


DEFAULT_TENANT = "default"


def normalize_tenant(tenant_id: str | None) -> str:
    """Blank tenants are the default bucket (reference db/graph_store.py:169-172 ``normalize_graph_tenant_id``)."""
    return (tenant_id or "").strip() or DEFAULT_TENANT


class B200GraphStore:
    """``max_graphs`` bounds the snapshot cache: every cached snapshot pins a device CSR plus its walk workspace in HBM, so the
    least recently used one is dropped (and freed once no caller is inside it) when a new snapshot would exceed the bound."""

    def __init__(self, inner=None, *, device: int = 0, max_graphs: int = 4):
        self._inner = inner
        self._device = device
        self._max_graphs = max(1, int(max_graphs))
        self._lock = threading.RLock()
        self._graphs: "dict[tuple[str, str], UnifiedGraph]" = {}     # insertion order = recency (re-inserted on use)
        self._latest: dict[str, str] = {}                             # only when there is no inner store to ask

    # ── snapshot cache: the device CSR is a cache of a snapshot, keyed (tenant, scan_id) ──
    def _remember(self, key: tuple[str, str], g: UnifiedGraph) -> None:
        """Insert as most recent; evict beyond the bound.  A replaced / evicted graph is only dereferenced: its device memory is
        released when the last holder lets go (``DeviceGraph.__del__`` → ``close()``, which itself waits for calls in flight),
        so a REST worker still inside a traversal of the old snapshot keeps a valid handle."""
        self._graphs.pop(key, None)
        self._graphs[key] = g
        while len(self._graphs) > self._max_graphs:
            del self._graphs[next(iter(self._graphs))]

    def save_graph(self, graph) -> None:
        g = graph if isinstance(graph, UnifiedGraph) else UnifiedGraph.from_graph(graph, device=self._device)
        tenant = normalize_tenant(g.tenant_id)
        with self._lock:
            self._remember((tenant, g.scan_id or ""), g)
            self._latest[tenant] = g.scan_id or ""
        if self._inner is not None:
            self._inner.save_graph(graph)

    def latest_snapshot_id(self, *, tenant_id: str = "") -> str:
        latest = getattr(self._inner, "latest_snapshot_id", None) if self._inner is not None else None
        if latest is not None:                # the inner store is the source of truth: another process may have written a newer snapshot
            return latest(tenant_id=tenant_id)
        with self._lock:
            return self._latest.get(normalize_tenant(tenant_id), "")

    def _graph(self, tenant_id: str, scan_id: str) -> UnifiedGraph | None:
        tenant = normalize_tenant(tenant_id)
        sid = scan_id or self.latest_snapshot_id(tenant_id=tenant_id)
        with self._lock:
            g = self._graphs.get((tenant, sid))
            if g is not None:
                self._graphs[(tenant, sid)] = self._graphs.pop((tenant, sid))      # most recently used
                return g
        if self._inner is None:
            return None
        g = self._load_topology_first(tenant_id, sid)
        if g is None:
            loaded = self._inner.load_graph(tenant_id=tenant_id, scan_id=sid)
            if loaded is None or not getattr(loaded, "nodes", None):
                return None
            g = UnifiedGraph.from_graph(loaded, device=self._device)
        with self._lock:
            self._remember((tenant, g.scan_id or sid), g)
        return g

    def _load_topology_first(self, tenant_id: str, scan_id: str) -> UnifiedGraph | None:
        """Cache miss over a SQLite-backed inner store (reference api/graph_store.py:259-263 keeps ``_db_path``): scan the
        topology columns only (graph/snapshot.py) instead of materialising every node / edge record."""
        db_path = getattr(self._inner, "_db_path", None)
        if db_path is None:
            return None
        from pathlib import Path

        from .graph.snapshot import load_snapshot

        if not Path(db_path).exists():
            return None
        g = load_snapshot(db_path, tenant_id=tenant_id, scan_id=scan_id, device=self._device)
        return g if g.nodes else None

    def load_graph(self, *, tenant_id: str = "", scan_id: str = "", entity_types: set[str] | None = None, min_severity_rank: int = 0):
        if (entity_types or min_severity_rank) and self._inner is not None:
            return self._inner.load_graph(tenant_id=tenant_id, scan_id=scan_id, entity_types=entity_types, min_severity_rank=min_severity_rank)
        g = self._graph(tenant_id, scan_id)
        return g if g is not None else UnifiedGraph(scan_id=scan_id, tenant_id=tenant_id)

    # ── traversal subset (GPU) ──────────────────────────────────────────
    def bfs_paths(self, *, tenant_id: str = "", scan_id: str = "", source: str, max_depth: int = 4, traversable_only: bool = True):
        g = self._graph(tenant_id, scan_id)
        if g is None or not g.has_node(source):
            return [], set()
        paths = g.bfs(source, max_depth=max_depth, traversable_only=traversable_only)
        reachable = g.reachable_from(source, max_depth=max_depth, traversable_only=traversable_only, include_source=False)
        return paths, reachable

    def impact_of(self, *, tenant_id: str = "", scan_id: str = "", node_id: str, max_depth: int = 4) -> dict[str, Any] | None:
        g = self._graph(tenant_id, scan_id)
        if g is None or not g.has_node(node_id):
            return None
        return g.impact_of(node_id, max_depth=max_depth)

    def traverse_subgraph(self, *, tenant_id: str = "", scan_id: str = "", roots: list[str], direction: str = "forward", max_depth: int = 4,
                          max_nodes: int = 500, max_edges: int = 10_000, deadline_monotonic: float | None = None, traversable_only: bool = False,
                          relationship_types=None, static_only: bool = False, dynamic_only: bool = False, include_roots: bool = True):
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return UnifiedGraph(scan_id=scan_id, tenant_id=tenant_id), {}, False
        return g.traverse_subgraph(roots, direction=direction, max_depth=max_depth, max_nodes=max_nodes, max_edges=max_edges,
                                   deadline_monotonic=deadline_monotonic, traversable_only=traversable_only, relationship_types=relationship_types,
                                   static_only=static_only, dynamic_only=dynamic_only, include_roots=include_roots)

    def attack_paths_for_sources(self, *, tenant_id: str = "", scan_id: str = "", source_ids: set[str]):
        """Materialised attack-path rows of the snapshot whose source is in ``source_ids`` — exactly what the reference stores
        return (api/graph_store.py:792-834: persisted rows only, ``[]`` for an empty source set); nothing is derived here."""
        if not source_ids:
            return []
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return []
        return [p for p in g.attack_paths if p.source in source_ids]

    def attack_paths(self, *, tenant_id: str = "", scan_id: str = "", offset: int = 0, limit: int = 100):
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return scan_id, "", [], 0
        if g.attack_paths:     # materialised rows: the stores' order (api/graph_store.py:836-887 ORDER BY composite_risk DESC)
            paths = sorted(g.attack_paths, key=lambda p: (-p.composite_risk, p.source, p.target))
            return g.scan_id, g.created_at, paths[offset: offset + limit], len(paths)
        # no materialised rows: the derived paths in their own ranking (api/routes/graph.py:1221-1230), ranked on the device —
        # only the requested page becomes Python objects
        page, total = ranked_attack_paths(g, offset, limit)
        return g.scan_id, g.created_at, page, total

    # ── batched extensions ──────────────────────────────────────────────
    def impact_of_many(self, *, tenant_id: str = "", scan_id: str = "", node_ids: list[str], max_depth: int = 4) -> list[dict[str, Any] | None]:
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return [None] * len(node_ids)
        res = g.impact_of_many(node_ids, max_depth)
        return [r if g.has_node(n) else None for n, r in zip(node_ids, res)]

    def exposure_paths_many(self, *, tenant_id: str = "", scan_id: str = "", finding_ids: list[str] | None = None):
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return []
        return materialize_attack_paths(g, exposure_path_rows(g, finding_ids))

    def fix_first_view(self, *, tenant_id: str = "", scan_id: str = "", cve: str = "", package: str = "", agent: str = "", limit: int = 8) -> dict[str, Any]:
        """The body of ``GET /v1/graph/views/fix-first`` (reference api/routes/graph.py:1110-1166) for the resolved snapshot, ranked on
        the device; a missing snapshot gives the view of an empty graph, as the route's ``load_graph`` does.  The route keeps its own
        503 when there is no snapshot at all."""
        g = self._graph(tenant_id, scan_id)
        if g is None:
            g = UnifiedGraph(scan_id=scan_id, tenant_id=tenant_id)
        return fix_first_view(g, cve=cve, package=package, agent=agent, limit=limit)

    def semantic_clusters_view(self, *, tenant_id: str = "", scan_id: str = "", kinds=None, min_members: int = 2, limit: int = 250) -> dict[str, Any]:
        """The body of ``GET /v1/graph/clusters`` (reference api/routes/graph.py:1485-1528) for the resolved snapshot, rolled up on the
        device; a missing snapshot gives the view of an empty graph, as the route's ``load_graph`` does.  The route keeps its own 503
        when there is no snapshot at all, and turns the ``ValueError`` of an unknown kind into its 400."""
        g = self._graph(tenant_id, scan_id)
        if g is None:
            g = UnifiedGraph(scan_id=scan_id, tenant_id=tenant_id)
        return semantic_clusters_view(g, kinds=kinds, min_members=min_members, limit=limit)

    def ocsf_events(self, *, tenant_id: str = "", scan_id: str = "", product_version: str = "0.0.0", enrich_neighbors: bool = True, offset: int = 0,
                    limit: int | None = None) -> list[dict[str, Any]]:
        """Page [offset, offset+limit) of the snapshot's OCSF finding events (``UnifiedGraph.to_ocsf_events`` order; ``limit=None``:
        to the end), computed only for that page; ``[]`` for a missing snapshot."""
        g = self._graph(tenant_id, scan_id)
        if g is None:
            return []
        return list(iter_ocsf_events(g, product_version, enrich_neighbors=enrich_neighbors, offset=offset, limit=limit))

    def dependency_reach(self, *, tenant_id: str = "", scan_id: str = "") -> ReachabilityReport | None:
        g = self._graph(tenant_id, scan_id)
        return None if g is None else compute_dependency_reach(g)

    def diff_snapshots(self, scan_id_old: str, scan_id_new: str, *, tenant_id: str = "") -> dict[str, Any]:
        """The body of ``GET /v1/graph/diff`` (reference db/graph_store.py:671-738), diffed on the device when the inner store is
        SQLite-backed (``_db_path``, as for topology-first loading); otherwise the inner store's own ``diff_snapshots``.  A blank or
        missing scan id is an empty snapshot: like the reference's ``scan_id = ?`` query, it never resolves to the latest one."""
        from pathlib import Path

        from .graph.delta import snapshot_diff

        db_path = getattr(self._inner, "_db_path", None) if self._inner is not None else None
        if db_path is None or not Path(db_path).exists():
            inner = getattr(self._inner, "diff_snapshots", None) if self._inner is not None else None
            if inner is None:
                raise B200UnsupportedOperationError("B200GraphStore has no inner store to serve diff_snapshots()")
            return inner(scan_id_old, scan_id_new, tenant_id=tenant_id)
        tenant = normalize_tenant(tenant_id)

        def snapshot(scan_id: str) -> UnifiedGraph:
            g = self._graph(tenant, scan_id) if scan_id else None
            return g if g is not None else UnifiedGraph(scan_id=scan_id, tenant_id=tenant, device=self._device)

        return snapshot_diff(snapshot(scan_id_old), snapshot(scan_id_new), db_path=db_path, tenant_id=tenant)

    # ── everything else: the wrapped default store ──────────────────────
    def __getattr__(self, name: str):
        inner = self.__dict__.get("_inner")
        if inner is not None and hasattr(inner, name):
            return getattr(inner, name)
        if name.startswith("_"):
            raise AttributeError(name)

        def unsupported(*_a, **_k):
            raise B200UnsupportedOperationError(f"B200GraphStore has no inner store to serve {name}()")

        return unsupported
