"""Lateral-movement paths over the legacy context graph, searched on the device (SURVEY §8 row f4).

Reference: ``/root/reference/src/agent_bom/context_graph.py`` — ``find_lateral_paths`` (:397-477) and
``_build_lateral_path`` (:480-593).  The order-sensitive queue search (100-path / 10 000-queue caps, per-path cycle
check, duplicate node sequences extended instead of recorded) runs in ``csrc/lateral.cuh``, one warp per source, so a
whole fleet is searched in one launch (the CLI and the REST route loop over every agent, ``cli/agents/__init__.py:1745``,
``api/routes/scan.py:701-705``).  What each found path folds in — the credential / tool / vulnerability label lists, the
execute-tool count and the highest severity (:495-572) — is computed on the device too, for every path of the call at once
(``abb_lateral_enrich_host``): a ``shares_server`` hop stands for every server with the link's server name, so on a fleet with
large shared-server cliques this is where the reference spends ~98 % of a search.  The host keeps the composite formula, the
summary string, the id -> label mapping and the per-source stable sort.  ``build_lateral_path`` is the single-path host
restatement, kept as the reference the device pass is tested against (and used to re-derive a path whose execute test or
severity lookup raised, so the caller sees the reference's exception).
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Any, Iterable

import numpy as np

from . import _lib
from .context_graph import kind_value

MAX_PATHS = 100                      # _MAX_PATHS (context_graph.py:393)
SEVERITY_RISK_SCORE = {"critical": 8.0, "high": 6.0, "medium": 4.0, "low": 2.0, "info": 0.5, "informational": 0.5, "none": 0.0, "unknown": 0.0}
_NODE_KIND_CODE = {"agent": 0, "server": 1, "credential": 2, "tool": 3, "vulnerability": 4, "iam_role": 5}
_GHOST = 255


@dataclass
class LateralPath:
    source: str
    target: str
    hops: list[str]
    edges: list[Any]
    composite_risk: float
    summary: str
    credential_exposure: list[str] = field(default_factory=list)
    tool_exposure: list[str] = field(default_factory=list)
    vuln_ids: list[str] = field(default_factory=list)


class LateralSearchOverflow(RuntimeError):
    """A source exhausted the search's safety valve; its result would be incomplete, so none is returned."""


class _Arrays:
    """``graph.adjacency`` as rows of (target, kind) and the per-node facts the target test reads."""

    def __init__(self, graph):
        nodes, adjacency = graph.nodes, graph.adjacency
        self.ids = list(nodes)
        index = {nid: i for i, nid in enumerate(self.ids)}
        rows = list(adjacency.items()) if hasattr(adjacency, "items") else []
        for nid, lst in rows:                                         # ids that only exist as adjacency keys / targets
            if nid not in index:
                index[nid] = len(self.ids)
                self.ids.append(nid)
            for e in lst:
                if e.target not in index:
                    index[e.target] = len(self.ids)
                    self.ids.append(e.target)
        n = len(self.ids)
        self.index = index
        self.kind_objs: list[Any] = []
        kind_code: dict[str, int] = {}
        counts = np.zeros(n + 1, dtype=np.int64)
        for nid, lst in rows:
            counts[index[nid] + 1] = len(lst)
        self.off = np.cumsum(counts)
        nbr = np.zeros(int(self.off[-1]), dtype=np.int32)
        ek = np.zeros(int(self.off[-1]), dtype=np.uint8)
        for nid, lst in rows:
            p = int(self.off[index[nid]])
            for e in lst:
                kv = kind_value(e.kind)
                code = kind_code.get(kv)
                if code is None:
                    code = kind_code[kv] = len(self.kind_objs)
                    self.kind_objs.append(e.kind)
                    if code > 15:
                        raise ValueError("more than 16 distinct edge kinds")
                nbr[p], ek[p] = index[e.target], code
                p += 1
        self.nbr, self.ek = nbr, ek
        self.kind_code = kind_code
        self._rows = rows
        self._enrich: _Enrichment | None = None
        self.keys: dict[Any, int] = {}
        self.nkind = np.full(n, _GHOST, dtype=np.uint8)
        self.nkey = np.full(n, -1, dtype=np.int32)
        for nid, node in nodes.items():
            i = index[nid]
            kv = kind_value(node.kind)
            self.nkind[i] = _NODE_KIND_CODE.get(kv, 6)
            if kv == "agent":
                self.nkey[i] = self.key_id(node.label)
            elif kv in ("credential", "tool"):
                owner = node.metadata.get("agent", "")
                if owner:
                    self.nkey[i] = self.key_id(owner)

    def key_id(self, value) -> int:
        return self.keys.setdefault(value, len(self.keys))

    def enrichment(self, graph) -> "_Enrichment":
        """The per-node and per-entry facts the device enrichment reads; built on first use, cached with the adjacency encoding."""
        if self._enrich is None:
            self._enrich = _Enrichment(graph, self)
        return self._enrich


_CAT_CRED, _CAT_TOOL, _CAT_VULN = 0, 1, 2
_SURFACE_PAIRS = {("exposes", "credential"): _CAT_CRED, ("provides", "tool"): _CAT_TOOL, ("vulnerable_to", "vulnerability"): _CAT_VULN}


def _execute_value(node) -> float:
    """1 when the reference counts the tool as execute-capable (``"execute" in caps``: a string does a substring test), -1 when
    that test raises."""
    try:
        return 1.0 if "execute" in node.metadata.get("capabilities", []) else 0.0
    except Exception:
        return -1.0


def _severity_value(node) -> float:
    """The severity score the reference takes for a vulnerability node, -1 when its lookup raises."""
    try:
        return float(SEVERITY_RISK_SCORE.get(node.metadata.get("severity", ""), 0))
    except Exception:
        return -1.0


class _Enrichment:
    """Label ids per category (credential names carried by ``shares_credential`` links share the credential ids), per-node
    execute flag / severity score, per-server surfaces, one surface per shared server name (every server with that label, in
    node order) and per-entry name ids for the sharing kinds.  Every surface is de-duplicated by label keeping its first node,
    which is the node that would first add the label if the path has not added it earlier."""

    def __init__(self, graph, arr: _Arrays):
        nodes, index = graph.nodes, arr.index
        n = len(arr.ids)
        self._nkind = arr.nkind
        self.label_ids: list[dict] = [{}, {}, {}]
        self.labels: list[list] = [[], [], []]
        self.node_label = np.full(n, -1, dtype=np.int32)
        self.node_value = np.zeros(n, dtype=np.float32)
        self.node_surface = np.full(n, -1, dtype=np.int32)
        servers_by_label: dict[Any, list[str]] = {}
        cat_of = {"credential": _CAT_CRED, "tool": _CAT_TOOL, "vulnerability": _CAT_VULN}
        for nid, node in nodes.items():
            i = index[nid]
            kv = kind_value(node.kind)
            cat = cat_of.get(kv)
            if cat is not None:
                self.node_label[i] = self._intern(cat, node.label)
                if cat == _CAT_TOOL:
                    self.node_value[i] = _execute_value(node)
                elif cat == _CAT_VULN:
                    self.node_value[i] = _severity_value(node)
            elif kv == "server":
                try:
                    servers_by_label.setdefault(node.label, []).append(nid)
                except TypeError:          # an unhashable label equals no name a link can carry here
                    pass
        surfaces: list[list[int]] = []
        server_surface: dict[str, list[int]] = {}
        for nid in (sid for sids in servers_by_label.values() for sid in sids):
            items = []
            for e in graph.adjacency.get(nid, []):
                other = nodes.get(e.target)
                if not other:
                    continue
                cat = _SURFACE_PAIRS.get((kind_value(e.kind), kind_value(other.kind)))
                if cat is not None:
                    items.append(index[e.target])
            server_surface[nid] = items = self._dedup(items)
            if items:
                self.node_surface[index[nid]] = len(surfaces)
                surfaces.append(items)
        # per entry of the sharing kinds: the shared server name's surface, or the shared credential name's id
        name_surface: dict[Any, int] = {}
        self.entry_name = np.full(len(arr.nbr), -1, dtype=np.int32)
        for nid, lst in arr._rows:
            p = int(arr.off[index[nid]])
            for e in lst:
                ek = kind_value(e.kind)
                meta = getattr(e, "metadata", None)
                if ek == "shares_server" and hasattr(meta, "get"):
                    name = meta.get("server", "")
                    if name:
                        try:
                            s = name_surface.get(name)
                            if s is None:
                                items = self._dedup([v for sid in servers_by_label.get(name, ()) for v in server_surface[sid]])
                                s = name_surface[name] = len(surfaces) if items else -1
                                if items:
                                    surfaces.append(items)
                            self.entry_name[p] = s
                        except TypeError:
                            pass
                elif ek == "shares_credential" and hasattr(meta, "get"):
                    name = meta.get("credential", "")
                    if name:
                        self.entry_name[p] = self._intern(_CAT_CRED, name)
                p += 1
        self.surface_off = np.zeros(len(surfaces) + 1, dtype=np.int64)
        self.surface_off[1:] = np.cumsum([len(x) for x in surfaces], dtype=np.int64)
        self.surface_node = np.asarray([v for x in surfaces for v in x], dtype=np.int32)
        self.code_ss = arr.kind_code.get("shares_server", -1)
        self.code_sc = arr.kind_code.get("shares_credential", -1)

    def _intern(self, cat: int, label) -> int:
        ids = self.label_ids[cat]
        i = ids.get(label)
        if i is None:
            i = ids[label] = len(self.labels[cat])
            self.labels[cat].append(label)
            if i >= 1 << 30:
                raise ValueError("more than 2^30 distinct labels in one category")
        return i

    def _dedup(self, items: list[int]) -> list[int]:
        seen, out = set(), []
        for v in items:
            key = (int(self._nkind[v]), int(self.node_label[v]))       # the node kind stands for the category
            if key not in seen:
                seen.add(key)
                out.append(v)
        return out


def _add(lst: list, item) -> bool:
    if item in lst:
        return False
    lst.append(item)
    return True


def build_lateral_path(graph, source_id: str, target_id: str, hops: list[str], edges: list) -> LateralPath:
    """Exposure lists, composite and summary of one found path (:480-593)."""
    nodes, adjacency = graph.nodes, graph.adjacency
    creds: list[str] = []
    tools: list[str] = []
    vulns: list[str] = []
    state = {"sev": 0.0, "exec": 0}

    def see_tool(node) -> None:
        if _add(tools, node.label) and "execute" in node.metadata.get("capabilities", []):
            state["exec"] += 1

    def see_vuln(node) -> None:
        if _add(vulns, node.label):
            state["sev"] = max(state["sev"], SEVERITY_RISK_SCORE.get(node.metadata.get("severity", ""), 0))

    def see_server_surface(server_id: str) -> None:
        """What a server exposes, provides and is vulnerable to, in adjacency order."""
        for e in adjacency.get(server_id, []):
            other = nodes.get(e.target)
            if not other:
                continue
            ek, ok = kind_value(e.kind), kind_value(other.kind)
            if ek == "exposes" and ok == "credential":
                _add(creds, other.label)
            elif ek == "provides" and ok == "tool":
                see_tool(other)
            elif ek == "vulnerable_to" and ok == "vulnerability":
                see_vuln(other)

    for nid in hops:
        node = nodes.get(nid)
        if not node:
            continue
        kv = kind_value(node.kind)
        if kv == "credential":
            _add(creds, node.label)
        elif kv == "tool":
            see_tool(node)
        elif kv == "vulnerability":
            see_vuln(node)
        elif kv == "server":
            see_server_surface(nid)
    # agent <-> agent sharing hops bypass the server node: fold in what the shared server / credential stands for (:538-572)
    for i, kind in enumerate(edges):
        if i >= len(hops) - 1:
            continue
        ek = kind_value(kind)
        if ek not in ("shares_server", "shares_credential"):
            continue
        link = next((e for e in adjacency.get(hops[i], []) if e.target == hops[i + 1] and kind_value(e.kind) == ek), None)
        if link is None:
            continue
        if ek == "shares_server":
            name = link.metadata.get("server", "")
            if name:
                for nid, node in nodes.items():
                    if kind_value(node.kind) == "server" and node.label == name:
                        see_server_surface(nid)
        else:
            name = link.metadata.get("credential", "")
            if name:
                _add(creds, name)
    composite = min(state["sev"] + len(creds) * 0.3 + state["exec"] * 0.2, 10.0)
    summary = " → ".join(nodes[n].label for n in hops if nodes.get(n))
    return LateralPath(source=source_id, target=target_id, hops=hops, edges=edges, composite_risk=round(composite, 1), summary=summary,
                       credential_exposure=creds, tool_exposure=tools, vuln_ids=vulns)



_ARRAYS_CACHE: dict[int, tuple[tuple, "_Arrays"]] = {}


def _arrays_for(graph) -> "_Arrays":
    """The array encoding of ``graph.adjacency`` is reused across calls on the same, unchanged graph (it was >99 % of a call:
    1.29 s of Python against 0.64 ms of device time for a 4 000-agent fleet); a change in node / edge / adjacency-row counts
    rebuilds it.  Entries die with their graph."""
    import weakref

    stamp = (len(graph.nodes), len(getattr(graph, "edges", ()) or ()), len(graph.adjacency), sum(map(len, graph.adjacency.values())) if len(graph.adjacency) < 4096 else -1)
    key = id(graph)
    hit = _ARRAYS_CACHE.get(key)
    if hit is not None and hit[0] == stamp:
        return hit[1]
    arr = _Arrays(graph)
    _ARRAYS_CACHE[key] = (stamp, arr)
    try:
        weakref.finalize(graph, _ARRAYS_CACHE.pop, key, None)
    except TypeError:          # not weak-referenceable: do not keep it
        _ARRAYS_CACHE.pop(key, None)
    return arr


def _search_records(graph, source_ids: list, max_depth: int, device: int, max_pops: int = 0):
    """One device search for every source: (encoding, per-source record offsets, records [total][W+2], W, device ms)."""
    lib = _lib.load()
    arr = _arrays_for(graph)
    src = np.full(len(source_ids), -1, dtype=np.int32)
    skey = np.zeros(len(source_ids), dtype=np.int32)
    for q, sid in enumerate(source_ids):
        node = graph.nodes.get(sid) if sid in graph.nodes else None
        if node is None:
            continue
        src[q] = arr.index[sid]
        skey[q] = arr.key_id(node.label if kind_value(node.kind) == "agent" else node.metadata.get("agent", ""))
    res = C.c_void_p()
    off64 = np.ascontiguousarray(arr.off, dtype=np.int64)
    _lib.check(lib.abb_lateral_paths_host(device, len(arr.ids), off64.ctypes.data, arr.nbr.ctypes.data, arr.ek.ctypes.data, arr.nkind.ctypes.data,
                                          arr.nkey.ctypes.data, len(source_ids), src.ctypes.data, skey.ctypes.data, int(max_depth), int(max_pops), C.byref(res)))
    try:
        nq = len(source_ids)
        W = int(lib.abb_lateral_result_width(res))
        R = W + 2
        off = np.ctypeslib.as_array(C.cast(lib.abb_lateral_result_off(res), C.POINTER(C.c_int64)), shape=(nq + 1,)).copy() if nq else np.zeros(1, np.int64)
        total = int(off[-1])
        rec = (np.ctypeslib.as_array(C.cast(lib.abb_lateral_result_records(res), C.POINTER(C.c_int32)), shape=(total * R,)).copy().reshape(total, R)
               if total else np.zeros((0, R), np.int32))
        flags = np.ctypeslib.as_array(C.cast(lib.abb_lateral_result_flags(res), C.POINTER(C.c_int32)), shape=(nq,)).copy() if nq else np.zeros(0, np.int32)
        ms = float(lib.abb_lateral_result_ms(res))
    finally:
        lib.abb_lateral_result_free(res)
    if flags.any():
        raise LateralSearchOverflow(f"search from {source_ids[int(np.flatnonzero(flags)[0])]!r} exceeded the safety valve")
    return arr, off, rec, W, ms


def search_many(graph, source_ids: Iterable[str], max_depth: int = 4, *, device: int = 0, max_pops: int = 0):
    """Raw device result per source: list of ``(hops, edge kinds)`` in discovery order."""
    source_ids = list(source_ids)
    arr, off, rec, _W, ms = _search_records(graph, source_ids, max_depth, device, max_pops)
    out = []
    for q in range(len(source_ids)):
        found = []
        for row in rec[int(off[q]): int(off[q + 1])].tolist():
            length, kinds = row[0], row[1] & 0xFFFFFFFF
            hops = [arr.ids[i] for i in row[2: 2 + length]]
            edges = [arr.kind_objs[(kinds >> (4 * h)) & 15] for h in range(length - 1)]
            found.append((hops, edges))
        out.append(found)
    return out, ms


def enrich_records(graph, arr: _Arrays, rec: np.ndarray, W: int, *, device: int = 0):
    """Device enrichment of search records: per path (kept items as ``category << 30 | label id``, offsets), execute counts,
    severity scores, flags, device ms."""
    lib = _lib.load()
    enc = arr.enrichment(graph)
    n_paths = int(rec.shape[0])
    rec = np.ascontiguousarray(rec, dtype=np.int32)
    off64 = np.ascontiguousarray(arr.off, dtype=np.int64)
    res = C.c_void_p()
    _lib.check(lib.abb_lateral_enrich_host(device, len(arr.ids), off64.ctypes.data, arr.nbr.ctypes.data, arr.ek.ctypes.data, enc.entry_name.ctypes.data,
                                           enc.code_ss, enc.code_sc, arr.nkind.ctypes.data, enc.node_label.ctypes.data, enc.node_value.ctypes.data,
                                           enc.node_surface.ctypes.data, len(enc.surface_off) - 1, enc.surface_off.ctypes.data, enc.surface_node.ctypes.data,
                                           n_paths, int(W), rec.ctypes.data, C.byref(res)))
    try:
        def take(fn, ctype, count, dtype):
            return np.ctypeslib.as_array(C.cast(fn(res), C.POINTER(ctype)), shape=(count,)).copy() if count else np.zeros(0, dtype)

        off = np.ctypeslib.as_array(C.cast(lib.abb_lateral_enrich_result_off(res), C.POINTER(C.c_int64)), shape=(n_paths + 1,)).copy()
        items = take(lib.abb_lateral_enrich_result_items, C.c_int32, int(off[-1]), np.int32)
        execute = take(lib.abb_lateral_enrich_result_exec, C.c_int32, n_paths, np.int32)
        severity = take(lib.abb_lateral_enrich_result_severity, C.c_float, n_paths, np.float32)
        flags = take(lib.abb_lateral_enrich_result_flags, C.c_int32, n_paths, np.int32)
        ms = float(lib.abb_lateral_enrich_result_ms(res))
    finally:
        lib.abb_lateral_enrich_result_free(res)
    return off, items, execute, severity, flags, ms


def find_lateral_paths_many(graph, source_ids: Iterable[str], max_depth: int = 4, *, device: int = 0, timings: dict | None = None) -> list[list[LateralPath]]:
    """``find_lateral_paths`` for many sources: one device search and one device enrichment for all of them; each list is
    sorted by composite risk, highest first.  ``timings``, when given, receives per-stage seconds (search, enrich, assemble;
    the first two include their device time, also given in ms as search_device_ms / enrich_device_ms) and the path count."""
    import time

    source_ids = list(source_ids)
    t0 = time.perf_counter()
    arr, off, rec, W, search_ms = _search_records(graph, source_ids, max_depth, device)
    t1 = time.perf_counter()
    e_off, items, execute, severity, flags, enrich_ms = enrich_records(graph, arr, rec, W, device=device)
    t2 = time.perf_counter()
    labels = arr.enrichment(graph).labels
    cats = (items.view(np.uint32) >> 30).tolist()
    lids = (items & 0x3FFFFFFF).tolist()
    e_off = e_off.tolist()
    execute, severity, bad = execute.tolist(), severity.tolist(), flags.tolist()
    nodes, ids, kind_objs = graph.nodes, arr.ids, arr.kind_objs
    out = []
    rows = rec.tolist()
    for q, sid in enumerate(source_ids):
        paths = []
        for k in range(int(off[q]), int(off[q + 1])):
            row = rows[k]
            length, kinds = row[0], row[1] & 0xFFFFFFFF
            hops = [ids[i] for i in row[2: 2 + length]]
            edges = [kind_objs[(kinds >> (4 * h)) & 15] for h in range(length - 1)]
            if bad[k]:                 # a first-added label's test raised in the encoding: let the host restatement raise it
                paths.append(build_lateral_path(graph, sid, hops[-1], hops, edges))
                continue
            lists: tuple[list, list, list] = ([], [], [])
            for j in range(e_off[k], e_off[k + 1]):
                c = cats[j]
                lists[c].append(labels[c][lids[j]])
            creds, tools, vulns = lists
            composite = min(severity[k] + len(creds) * 0.3 + execute[k] * 0.2, 10.0)
            summary = " → ".join(nodes[n].label for n in hops if nodes.get(n))
            paths.append(LateralPath(source=sid, target=hops[-1], hops=hops, edges=edges, composite_risk=round(composite, 1), summary=summary,
                                     credential_exposure=creds, tool_exposure=tools, vuln_ids=vulns))
        paths.sort(key=lambda p: p.composite_risk, reverse=True)
        out.append(paths[:MAX_PATHS])
    if timings is not None:
        timings.update(search=t1 - t0, enrich=t2 - t1, assemble=time.perf_counter() - t2, search_device_ms=search_ms, enrich_device_ms=enrich_ms, paths=len(rows))
    return out


def find_lateral_paths(graph, source_node_id: str, max_depth: int = 4, *, device: int = 0) -> list[LateralPath]:
    """Up to 100 lateral paths from one node, sorted by composite risk (drop-in for context_graph.py:397-477)."""
    if source_node_id not in graph.nodes:
        return []
    return find_lateral_paths_many(graph, [source_node_id], max_depth, device=device)[0]


__all__ = ["LateralPath", "LateralSearchOverflow", "build_lateral_path", "enrich_records", "find_lateral_paths", "find_lateral_paths_many", "search_many"]
