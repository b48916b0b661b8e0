"""ctypes binding of libabb200.so (the C ABI declared in include/abb200.h).

Loading fails loudly when the library is missing or cannot be built: there is
no CPU fallback for the traversal path.
"""

from __future__ import annotations

import ctypes as C
import os
import threading
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libabb200.so"

vp, i32, i64, u32, u8p = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_void_p


class EngineUnavailable(RuntimeError):
    """The CUDA engine library is missing / unloadable, or no CUDA device is present."""


class AbbError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"abb200 error {code}: {message}")
        self.code = code


class Csr(C.Structure):
    _fields_ = [
        ("n_nodes", i32), ("n_entries", i64),
        ("fwd_off", vp), ("fwd_nbr", vp), ("fwd_meta", vp), ("fwd_eid", vp),
        ("rev_off", vp), ("rev_nbr", vp), ("rev_meta", vp), ("rev_eid", vp),
        ("node_type", vp), ("node_rank", vp),
    ]


class WalkSpec(C.Structure):
    _fields_ = [
        ("direction", i32), ("max_depth", i32), ("rel_mask", u32), ("flags", u32),
        ("max_nodes", i64), ("max_edges", i64), ("emit_types", u32), ("reserved", u32),
    ]


class WalkIO(C.Structure):
    _fields_ = [
        ("n_queries", i64), ("roots", vp), ("root_off", vp), ("targets", vp),
        ("q_start", vp), ("q_count", vp), ("q_maxd", vp), ("q_flags", vp), ("q_estart", vp), ("q_ecount", vp), ("q_hist", vp),
        ("nodes", vp), ("parent", vp), ("depth", vp), ("node_cap", i64),
        ("edges", vp), ("edge_cap", i64), ("totals", vp),
    ]


class SearchSpec(C.Structure):
    _fields_ = [
        ("mode", i32), ("n_patterns", i32), ("patterns", vp), ("pattern_off", vp), ("type_ok", vp), ("cmp_ok", vp), ("src_ok", vp),
        ("n_types", i32), ("n_cmp", i32), ("n_src", i32), ("use_min_rank", i32), ("min_rank", i64), ("has_cursor", i32), ("cur_risk_null", i32),
        ("cur_sev", i64), ("cur_risk", C.c_double), ("cur_label_gt", i64), ("cur_label_eq", i64), ("cur_id_gt", i64), ("offset", i64), ("take", i64),
    ]


class PathsIO(C.Structure):
    _fields_ = [
        ("n_findings", i64), ("findings", vp), ("f_off", vp), ("hops", vp), ("rels", vp), ("ncred", vp), ("ntool", vp), ("row_cap", i64),
    ]


# walk flags (include/abb200.h)
WALK_TRAVERSABLE_ONLY, WALK_MARK_ROOTS, WALK_OMIT_ROOTS, WALK_PARENTS, WALK_DEPTHS = 0x1, 0x2, 0x4, 0x8, 0x10
WALK_EDGES, WALK_HIST, WALK_REAL_ROOTS, WALK_TARGET = 0x20, 0x40, 0x80, 0x100
QFLAG_TRUNCATED, QFLAG_NO_ROOT, QFLAG_TARGET_FOUND = 1, 2, 4
# focus bits of the fix-first ranking (include/abb200.h, table in csrc/paths.cuh)
FOCUS_CVE, FOCUS_CVE_FINDING, FOCUS_PACKAGE, FOCUS_AGENT = 0x1, 0x2, 0x4, 0x8
DIR_FORWARD, DIR_REVERSE, DIR_BOTH = 1, 2, 3
# source-list buckets of the finding context (include/abb200.h, csrc/context.cuh)
CTX_AGENT, CTX_SERVER, CTX_PACKAGE, CTX_CREDENTIAL, CTX_BUCKETS = 0, 1, 2, 3, 4

#: every symbol include/abb200.h declares (tests assert the .so exports all of them)
EXPORTS = {
    "abb_last_error": (C.c_char_p, []),
    "abb_version": (C.c_int, []),
    "abb_device_count": (C.c_int, []),
    "abb_csr_entries": (i64, [i64, vp]),
    "abb_csr_build_host": (C.c_int, [i32, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "abb_graph_upload": (C.c_int, [C.c_int, C.POINTER(Csr), C.POINTER(vp)]),
    "abb_graph_adopt": (C.c_int, [C.c_int, C.POINTER(Csr), C.POINTER(vp)]),
    "abb_graph_view": (C.c_int, [vp, C.POINTER(Csr)]),
    "abb_graph_bytes": (i64, [vp]),
    "abb_graph_set_dedup": (C.c_int, [vp, C.c_int]),
    "abb_graph_device": (C.c_int, [vp]),
    "abb_graph_set_option": (C.c_int, [vp, C.c_char_p, i64]),
    "abb_graph_get_option": (i64, [vp, C.c_char_p]),
    "abb_graph_free": (None, [vp]),
    "abb_spec_impact_of": (WalkSpec, [i32]),
    "abb_spec_bfs": (WalkSpec, [i32, i32]),
    "abb_spec_reachable_from": (WalkSpec, [i32, i32]),
    "abb_spec_shortest_path": (WalkSpec, []),
    "abb_spec_traverse_subgraph": (WalkSpec, [i32, i32, i64, i64, i32, u32, i32, i32, i32]),
    "abb_spec_distances_along": (WalkSpec, [u32, u32]),
    "abb_walk_launch": (C.c_int, [vp, C.POINTER(WalkSpec), C.POINTER(WalkIO), vp]),
    "abb_walk_signatures": (C.c_int, [vp, C.POINTER(WalkSpec), vp, i64, vp, vp]),
    "abb_launch_count": (i64, []),
    "abb_last_walk_ms": (C.c_float, [vp]),
    "abb_last_walk_stats": (C.c_int, [vp, vp]),
    "abb_last_walk_tier_counts": (C.c_int, [vp, vp]),
    "abb_last_paths_ms": (C.c_float, [vp]),
    "abb_walk_host": (C.c_int, [vp, C.POINTER(WalkSpec), vp, vp, vp, i64, C.POINTER(vp)]),
    "abb_walk_result_queries": (i64, [vp]),
    "abb_walk_result_total_nodes": (i64, [vp]),
    "abb_walk_result_total_edges": (i64, [vp]),
    "abb_walk_result_start": (vp, [vp]),
    "abb_walk_result_count": (vp, [vp]),
    "abb_walk_result_maxd": (vp, [vp]),
    "abb_walk_result_flags": (vp, [vp]),
    "abb_walk_result_estart": (vp, [vp]),
    "abb_walk_result_ecount": (vp, [vp]),
    "abb_walk_result_hist": (vp, [vp]),
    "abb_walk_result_hist_packed": (vp, [vp, vp, vp]),
    "abb_walk_result_nodes": (vp, [vp]),
    "abb_walk_result_parent": (vp, [vp]),
    "abb_walk_result_depth": (vp, [vp]),
    "abb_walk_result_edges": (vp, [vp]),
    "abb_walk_result_h2d_bytes": (i64, [vp]),
    "abb_walk_result_d2h_bytes": (i64, [vp]),
    "abb_walk_result_free": (None, [vp]),
    "abb_paths_count_launch": (C.c_int, [vp, C.POINTER(PathsIO), vp]),
    "abb_paths_fill_launch": (C.c_int, [vp, C.POINTER(PathsIO), vp]),
    "abb_paths_host": (C.c_int, [vp, vp, i64, C.POINTER(vp)]),
    "abb_paths_result_rows": (i64, [vp]),
    "abb_paths_result_links": (i64, [vp]),
    "abb_paths_result_template_rows": (i64, [vp]),
    "abb_paths_result_link_off": (vp, [vp]),
    "abb_paths_result_link_source": (vp, [vp]),
    "abb_paths_result_link_rel": (vp, [vp]),
    "abb_paths_result_link_row_off": (vp, [vp]),
    "abb_paths_result_link_template": (vp, [vp]),
    "abb_paths_result_template": (vp, [vp]),
    "abb_paths_result_template_rel": (vp, [vp]),
    "abb_paths_result_off": (vp, [vp]),
    "abb_paths_result_hops": (vp, [vp]),
    "abb_paths_result_rels": (vp, [vp]),
    "abb_paths_result_ncred": (vp, [vp]),
    "abb_paths_result_ntool": (vp, [vp]),
    "abb_paths_result_h2d_bytes": (i64, [vp]),
    "abb_paths_result_d2h_bytes": (i64, [vp]),
    "abb_paths_result_free": (None, [vp]),
    "abb_paths_rank_host": (C.c_int, [vp, vp, i64, vp, vp, i64, vp, vp, i64, i64, C.POINTER(vp)]),
    "abb_paths_rank_focus_host": (C.c_int, [vp, vp, i64, vp, vp, i64, vp, vp, vp, u32, i64, i64, C.POINTER(vp)]),
    "abb_rank_result_matched": (i64, [vp]),
    "abb_rank_result_total": (i64, [vp]),
    "abb_rank_result_count": (i64, [vp]),
    "abb_rank_result_hops": (vp, [vp]),
    "abb_rank_result_rels": (vp, [vp]),
    "abb_rank_result_ncred": (vp, [vp]),
    "abb_rank_result_ntool": (vp, [vp]),
    "abb_rank_result_risk_rank": (vp, [vp]),
    "abb_rank_result_row": (vp, [vp]),
    "abb_rank_result_free": (None, [vp]),
    "abb_exposure_host": (C.c_int, [vp, vp, i64, i32, C.POINTER(vp), C.POINTER(vp)]),
    "abb_finding_context_host": (C.c_int, [vp, i32, vp, i64, C.POINTER(vp)]),
    "abb_finding_context_result_queries": (i64, [vp]),
    "abb_finding_context_result_count": (vp, [vp]),
    "abb_finding_context_result_maxd": (vp, [vp]),
    "abb_finding_context_result_flags": (vp, [vp]),
    "abb_finding_context_result_hist_packed": (vp, [vp, vp, vp]),
    "abb_finding_context_result_hist": (vp, [vp]),
    "abb_finding_context_result_start": (vp, [vp]),
    "abb_finding_context_result_bucket_counts": (vp, [vp]),
    "abb_finding_context_result_total_sources": (i64, [vp]),
    "abb_finding_context_result_sources": (vp, [vp]),
    "abb_finding_context_result_h2d_bytes": (i64, [vp]),
    "abb_finding_context_result_d2h_bytes": (i64, [vp]),
    "abb_finding_context_result_walk_ms": (C.c_float, [vp]),
    "abb_finding_context_result_context_ms": (C.c_float, [vp]),
    "abb_finding_context_result_free": (None, [vp]),
    "abb_dependency_reach_host": (C.c_int, [vp, vp, i64, u32, u32, C.POINTER(vp)]),
    "abb_reach_n_packages": (i64, [vp]),
    "abb_reach_pkg_ids": (vp, [vp]),
    "abb_reach_pkg_off": (vp, [vp]),
    "abb_reach_pkg_agents": (vp, [vp]),
    "abb_reach_pkg_minhop": (vp, [vp]),
    "abb_reach_n_vulns": (i64, [vp]),
    "abb_reach_vuln_ids": (vp, [vp]),
    "abb_reach_vuln_poff": (vp, [vp]),
    "abb_reach_vuln_pkgs": (vp, [vp]),
    "abb_reach_vuln_aoff": (vp, [vp]),
    "abb_reach_vuln_agents": (vp, [vp]),
    "abb_reach_vuln_minhop": (vp, [vp]),
    "abb_reach_result_free": (None, [vp]),
    "abb_bottleneck_host": (C.c_int, [vp, vp, i64, vp]),
    "abb_pagerank_host": (C.c_int, [vp, vp, vp, vp]),
    "abb_betweenness_host": (C.c_int, [vp, vp]),
    "abb_bidir_paths_host": (C.c_int, [vp, vp, vp, i64, C.POINTER(vp)]),
    "abb_bidir_result_start": (vp, [vp]),
    "abb_bidir_result_length": (vp, [vp]),
    "abb_bidir_result_total": (i64, [vp]),
    "abb_bidir_result_nodes": (vp, [vp]),
    "abb_bidir_result_free": (None, [vp]),
    "abb_lateral_paths_host": (C.c_int, [C.c_int, i32, vp, vp, vp, vp, vp, i64, vp, vp, i32, i64, C.POINTER(vp)]),
    "abb_lateral_result_off": (vp, [vp]),
    "abb_lateral_result_records": (vp, [vp]),
    "abb_lateral_result_flags": (vp, [vp]),
    "abb_lateral_result_width": (i32, [vp]),
    "abb_lateral_result_ms": (C.c_double, [vp]),
    "abb_lateral_result_free": (None, [vp]),
    "abb_lateral_enrich_host": (C.c_int, [C.c_int, i32, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, i32, vp, vp, i64, i32, vp, C.POINTER(vp)]),
    "abb_lateral_enrich_result_off": (vp, [vp]),
    "abb_lateral_enrich_result_items": (vp, [vp]),
    "abb_lateral_enrich_result_exec": (vp, [vp]),
    "abb_lateral_enrich_result_severity": (vp, [vp]),
    "abb_lateral_enrich_result_flags": (vp, [vp]),
    "abb_lateral_enrich_result_ms": (C.c_double, [vp]),
    "abb_lateral_enrich_result_free": (None, [vp]),
    "abb_group_union_host": (C.c_int, [C.c_int, i64, vp, vp, i64, vp, vp, vp, vp, C.POINTER(vp)]),
    "abb_union_result_off": (vp, [vp]),
    "abb_union_result_items": (vp, [vp]),
    "abb_union_result_w0": (vp, [vp]),
    "abb_union_result_w1": (vp, [vp]),
    "abb_union_result_ms": (C.c_double, [vp]),
    "abb_union_result_free": (None, [vp]),
    "abb_clusters_build_host": (C.c_int, [vp, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "abb_clusters_fetch_host": (C.c_int, [vp, i64, vp, vp, vp, vp]),
    "abb_delta_table_host": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp]),
    "abb_delta_table_bytes": (i64, [vp]),
    "abb_delta_build_host": (C.c_int, [vp, vp, vp, vp, vp, vp]),
    "abb_delta_result_free": (None, [vp]),
    "abb_delta_fetch_host": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "abb_delta_shared_host": (C.c_int, [vp, vp]),
    "abb_delta_shared_fetch_host": (C.c_int, [vp, vp, vp]),
    "abb_lookup_table_host": (C.c_int, [vp, i32, vp, i64, vp, vp, vp, vp]),
    "abb_lookup_table_bytes": (i64, [vp]),
    "abb_lookup_edges_host": (C.c_int, [vp, i64, vp, vp, vp]),
    "abb_lookup_context_host": (C.c_int, [vp, i32, vp, vp]),
    "abb_lookup_fetch_host": (C.c_int, [vp, vp]),
    "abb_lookup_result_free": (None, [vp]),
    "abb_search_text_host": (C.c_int, [vp, i32, vp, vp, vp]),
    "abb_search_table_host": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32]),
    "abb_search_table_bytes": (i64, [vp]),
    "abb_search_host": (C.c_int, [vp, vp, vp, vp, vp, vp]),
    "abb_search_fetch_host": (C.c_int, [vp, vp]),
    "abb_search_result_free": (None, [vp]),
    "abb_compliance_table_host": (C.c_int, [vp, i32, vp, vp, vp, i32, vp, vp, i32, vp, i32, i32, i32, vp]),
    "abb_compliance_table_bytes": (i64, [vp]),
    "abb_compliance_fetch_host": (C.c_int, [vp, vp, vp, vp, vp, vp]),
    "abb_lifecycle_build_host": (C.c_int, [C.c_int, i64, vp, vp, vp, vp, vp, vp, i64, i64, i64, C.POINTER(vp), vp]),
    "abb_lifecycle_active_host": (C.c_int, [vp, i32, vp, vp, vp]),
    "abb_lifecycle_bytes": (i64, [vp]),
    "abb_lifecycle_free": (None, [vp]),
    "abb_hops_host": (C.c_int, [C.c_int, i32, i32, vp, vp, i32, vp, vp, vp, i32, vp, vp, i64, vp, vp, vp, vp, vp, vp, i64, C.POINTER(vp)]),
    "abb_hops_result_counts": (None, [vp, vp]),
    "abb_hops_result_times": (None, [vp, vp]),
    "abb_hops_result_disc_sig": (vp, [vp]),
    "abb_hops_result_disc_occ": (vp, [vp]),
    "abb_hops_result_disc_hop": (vp, [vp]),
    "abb_hops_result_disc_parent": (vp, [vp]),
    "abb_hops_result_entry_server": (vp, [vp]),
    "abb_hops_result_entry_parent": (vp, [vp]),
    "abb_hops_result_cred": (vp, [vp]),
    "abb_hops_result_free": (None, [vp]),
}

_lock = threading.Lock()
_lib = None


def load(build_if_missing: bool = True):
    """Return the loaded library, building it with nvcc first if it is absent."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            if not build_if_missing:
                raise EngineUnavailable(f"{LIB_PATH} is missing (run `python -m agent_bom_b200.build`); there is no CPU fallback")
            from . import build as _build

            try:
                _build.build()
            except Exception as exc:  # nvcc missing / compile error
                raise EngineUnavailable(f"cannot build {LIB_PATH.name}: {exc}") from exc
        path = LIB_PATH
        if os.environ.get("ABB_LIB"):      # experiment build (python -m agent_bom_b200.build <variant> <defines…>), A/B measurements only
            path = PKG / os.environ["ABB_LIB"]
            if not path.exists():
                raise EngineUnavailable(f"ABB_LIB={os.environ['ABB_LIB']}: {path} does not exist")
        try:
            lib = C.CDLL(str(path))
        except OSError as exc:
            raise EngineUnavailable(f"cannot load {LIB_PATH}: {exc}") from exc
        for name, (restype, argtypes) in EXPORTS.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().abb_last_error()
        raise AbbError(rc, msg.decode() if msg else "")


def require_device() -> int:
    n = load().abb_device_count()
    if n <= 0:
        raise EngineUnavailable("no CUDA device visible: the blast-radius engine has no CPU fallback")
    return n
