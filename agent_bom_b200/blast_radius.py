"""Multi-hop blast-radius expansion on the device: delegation chains, transitive agents and their credentials.

Reference: ``expand_blast_radius_hops`` (``scanners/blast_radius.py:16-97``), run at the end of every scan whose blast-radius
depth is above 1.  For each blast radius the reference runs a FIFO breadth-first search over agents and MCP server names: out
from the affected agents, through every server they use that is not one of the blast radius's own (direct) servers, to the
other agents of that server, and on.  Every agent it reaches adds a delegation chain, a transitive-agent record and its
credentials.  Here:

- host, once per call, in linear time (:func:`encode`): agent, server and credential names are interned; two CSRs are built,
  name -> servers (keyed by name, the last agent object of a name wins) and server -> agent occurrences (one per (agent object,
  server) pair, each with its object's credential set); blast radii are grouped by *signature* (ordered affected agent names,
  set of direct server names), and each signature's visited marks and first queue level are listed;
- device (``abb_hops_host``, ``csrc/hops.cuh``): every signature is searched once, level by level, with discovery order equal
  to the reference's FIFO order; each discovery comes back as (occurrence, hop, parent queue entry), and each signature's
  credential union as sorted unique ids;
- host (:func:`materialise`): each discovery's chain string extends its parent's, once per signature; each blast radius then
  gets fresh lists and dicts, and its hop-discounted risk score from its own ``risk_score``.

``transitive_credentials`` is returned in code-point order (the reference returns Python set order, which depends on the hash
seed).  There is no CPU fallback: without the library or a device the first call above depth 1 raises ``EngineUnavailable``.
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib

#: the reference's hop discount (``_HOP_RISK_FACTORS``), indexed by the deepest hop reached
HOP_RISK_FACTORS: dict[int, float] = {1: 1.0, 2: 0.7, 3: 0.5, 4: 0.35, 5: 0.25}

ARROW = "→"


def clamp_depth(max_depth: int) -> int:
    return max(1, min(max_depth, 5))


@dataclass
class Encoding:
    """Interned inputs of one call (see the module docstring).  Occurrence k is ``occ_obj[k]``'s use of server ``occ_server``."""

    names: list[str]
    servers: list[str]
    creds: list[str]                       # sorted: credential id order is code-point order
    name_srv_off: np.ndarray               # int64 [n_names + 1]
    name_srv: np.ndarray                   # int32 server ids
    srv_occ_off: np.ndarray                # int64 [n_servers + 1]
    occ_name: np.ndarray                   # int32 name id per occurrence
    occ_obj: np.ndarray                    # int32 agent object per occurrence (its type and credential set)
    obj_type: list[str]
    cset_off: np.ndarray                   # int64 [n_objects + 1]: per agent object its sorted unique credential ids
    cset_cred: np.ndarray                  # int32
    sig_members: list[list[int]]           # blast-radius indices per signature
    mark_agent_off: np.ndarray
    mark_agent: np.ndarray
    mark_srv_off: np.ndarray
    mark_srv: np.ndarray
    first_off: np.ndarray                  # per signature its first-level queue entries
    first_srv: np.ndarray
    first_root: list[str]                  # the affected agent name that starts each first-level entry's chain


def _csr(rows: list[list[int]]) -> tuple[np.ndarray, np.ndarray]:
    off = np.zeros(len(rows) + 1, np.int64)
    if rows:
        np.cumsum([len(r) for r in rows], out=off[1:])
    flat = np.fromiter((v for r in rows for v in r), np.int32, int(off[-1]))
    return off, flat


def encode(blast_radii, agents) -> Encoding:
    """Intern names, build both CSRs and group the blast radii by signature, in one pass over each input."""
    name_id: dict[str, int] = {}
    srv_id: dict[str, int] = {}
    name_srv_rows: list[list[int]] = []
    occ_rows: list[list[tuple[int, int]]] = []
    obj_type: list[str] = []
    obj_creds: list[set[str]] = []
    all_creds: set[str] = set()
    for a, agent in enumerate(agents):
        nid = name_id.setdefault(agent.name, len(name_id))
        if nid == len(name_srv_rows):
            name_srv_rows.append([])
        row: list[int] = []
        creds: set[str] = set()
        for server in agent.mcp_servers:
            sid = srv_id.get(server.name)
            if sid is None:
                sid = srv_id[server.name] = len(srv_id)
                occ_rows.append([])
            row.append(sid)
            occ_rows[sid].append((nid, a))
            creds.update(server.credential_names)
        name_srv_rows[nid] = row                # the last object of a name wins
        obj_type.append(agent.agent_type.value)
        obj_creds.append(creds)
        all_creds |= creds
    cred_list = sorted(all_creds)
    cred_id = {c: i for i, c in enumerate(cred_list)}
    name_srv_off, name_srv = _csr(name_srv_rows)
    srv_occ_off = np.zeros(len(occ_rows) + 1, np.int64)
    if occ_rows:
        np.cumsum([len(r) for r in occ_rows], out=srv_occ_off[1:])
    flat = [o for r in occ_rows for o in r]
    occ_name = np.fromiter((o[0] for o in flat), np.int32, len(flat))
    occ_obj = np.fromiter((o[1] for o in flat), np.int32, len(flat))
    cset_off, cset_cred = _csr([sorted(cred_id[c] for c in s) for s in obj_creds])

    sig_index: dict[tuple, int] = {}
    sig_members: list[list[int]] = []
    marks_a: list[list[int]] = []
    marks_s: list[list[int]] = []
    firsts: list[list[int]] = []
    first_root: list[str] = []
    for b, br in enumerate(blast_radii):
        affected = tuple(a.name for a in br.affected_agents)
        direct = frozenset(s.name for s in br.affected_servers)
        key = (affected, direct)
        s = sig_index.get(key)
        if s is not None:
            sig_members[s].append(b)
            continue
        sig_index[key] = len(sig_members)
        sig_members.append([b])
        marks_a.append([name_id[n] for n in dict.fromkeys(affected) if n in name_id])
        seen: set[int] = {srv_id[n] for n in direct if n in srv_id}
        first: list[int] = []
        for n in affected:
            nid = name_id.get(n)
            if nid is None:
                continue
            for sid in name_srv_rows[nid]:
                # a repeated queue entry discovers nothing new: its server's agents were all visited the first time
                if sid not in seen:
                    seen.add(sid)
                    first.append(sid)
                    first_root.append(n)
        marks_s.append(sorted(seen))
        firsts.append(first)
    mark_agent_off, mark_agent = _csr(marks_a)
    mark_srv_off, mark_srv = _csr(marks_s)
    first_off, first_srv = _csr(firsts)
    return Encoding(list(name_id), list(srv_id), cred_list, name_srv_off, name_srv, srv_occ_off, occ_name, occ_obj, obj_type, cset_off, cset_cred,
                    sig_members, mark_agent_off, mark_agent, mark_srv_off, mark_srv, first_off, first_srv, first_root)


@dataclass
class HopArrays:
    """Per-signature search results.  Discoveries of signature s are ``sig_off[s] .. sig_off[s + 1] - 1`` in discovery order;
    ``parent`` is a queue entry id: below ``n_first`` a first-level entry (``Encoding.first_srv``), otherwise entry
    ``parent - n_first`` of ``entry_srv`` / ``entry_parent`` (whose parent is a discovery index)."""

    sig_off: np.ndarray
    occ: np.ndarray
    hop: np.ndarray
    parent: np.ndarray
    n_first: int
    entry_srv: np.ndarray
    entry_parent: np.ndarray
    cred_off: np.ndarray
    cred: np.ndarray
    stats: dict = field(default_factory=dict)


def _take(ptr, n: int, ctype, dtype) -> np.ndarray:
    if n <= 0 or not ptr:
        return np.zeros(0, dtype)
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(n,)).astype(dtype, copy=True)


def search(enc: Encoding, max_depth: int, *, device: int = 0, batch: int = 0) -> HopArrays:
    """Search every signature of ``enc`` on the device (``abb_hops_host``) at a clamped depth of 2..5.  ``batch`` > 0 caps how
    many signatures run at once (tests use it to force many small batches)."""
    if not 2 <= max_depth <= 5:
        raise ValueError("search runs at a clamped depth of 2..5")
    lib = _lib.load()
    _lib.require_device()
    n_sigs = len(enc.sig_members)
    res = C.c_void_p()
    ptr = lambda a: a.ctypes.data  # noqa: E731
    _lib.check(lib.abb_hops_host(device, max_depth, len(enc.names), ptr(enc.name_srv_off), ptr(enc.name_srv), len(enc.servers), ptr(enc.srv_occ_off),
                                 ptr(enc.occ_name), ptr(enc.occ_obj), len(enc.obj_type), ptr(enc.cset_off), ptr(enc.cset_cred), n_sigs,
                                 ptr(enc.mark_agent_off), ptr(enc.mark_agent), ptr(enc.mark_srv_off), ptr(enc.mark_srv), ptr(enc.first_off),
                                 ptr(enc.first_srv), int(batch), C.byref(res)))
    try:
        counts = (C.c_int64 * 5)()
        lib.abb_hops_result_counts(res, counts)
        times = (C.c_double * 3)()
        lib.abb_hops_result_times(res, times)
        nd, ne, nc = int(counts[0]), int(counts[1]), int(counts[2])
        d_sig = _take(lib.abb_hops_result_disc_sig(res), nd, C.c_int32, np.int32)
        d_occ = _take(lib.abb_hops_result_disc_occ(res), nd, C.c_int32, np.int32)
        d_hop = _take(lib.abb_hops_result_disc_hop(res), nd, C.c_int32, np.int8)
        d_par = _take(lib.abb_hops_result_disc_parent(res), nd, C.c_int64, np.int64)
        e_srv = _take(lib.abb_hops_result_entry_server(res), ne, C.c_int32, np.int32)
        e_par = _take(lib.abb_hops_result_entry_parent(res), ne, C.c_int64, np.int64)
        keys = _take(lib.abb_hops_result_cred(res), nc, C.c_uint64, np.uint64)
        stats = {"discoveries": nd, "entries": ne, "cred_keys": nc, "batches": int(counts[3]), "batch_size": int(counts[4]),
                 "upload_ms": float(times[0]), "search_ms": float(times[1]), "readback_ms": float(times[2])}
    finally:
        lib.abb_hops_result_free(res)
    # the device returns (batch, level, signature) order; a stable sort by signature gives each signature's discovery order
    order = np.argsort(d_sig, kind="stable")
    inv = np.empty(nd, np.int64)
    inv[order] = np.arange(nd, dtype=np.int64)
    sig_off = np.zeros(n_sigs + 1, np.int64)
    np.cumsum(np.bincount(d_sig, minlength=n_sigs), out=sig_off[1:])
    key_sig = (keys >> np.uint64(32)).astype(np.int64)
    cred_off = np.zeros(n_sigs + 1, np.int64)
    np.cumsum(np.bincount(key_sig, minlength=n_sigs), out=cred_off[1:])
    return HopArrays(sig_off, d_occ[order], d_hop[order], d_par[order], len(enc.first_srv), e_srv, inv[e_par] if ne else np.zeros(0, np.int64),
                     cred_off, (keys & np.uint64(0xFFFFFFFF)).astype(np.int32), stats)


def materialise(enc: Encoding, arr: HopArrays) -> list[tuple[int, list[tuple[str, str, int, str]], list[str]] | None]:
    """Per signature: ``None`` when nothing was discovered, else ``(hop_depth, [(name, type, hop, chain)], credentials)``.
    Each chain string is built once, by extending its parent queue entry's chain."""
    names, servers, occ_name, occ_obj, obj_type = enc.names, enc.servers, enc.occ_name.tolist(), enc.occ_obj.tolist(), enc.obj_type
    occ = arr.occ.tolist()
    hop = arr.hop.tolist()
    parent = arr.parent.tolist()
    e_srv = arr.entry_srv.tolist()
    e_par = arr.entry_parent.tolist()
    n_first = arr.n_first
    first_chain = [root + ARROW + servers[s] for root, s in zip(enc.first_root, enc.first_srv.tolist())]
    entry_chain: list[str | None] = [None] * len(e_srv)
    disc_chain: list[str | None] = [None] * len(occ)
    disc_name = [names[occ_name[o]] for o in occ]
    # parents precede children by hop: level h's discoveries extend entries whose parents are at hop h - 1
    by_hop: dict[int, list[int]] = {}
    for i, h in enumerate(hop):
        by_hop.setdefault(h, []).append(i)
    ent_by_hop: dict[int, list[int]] = {}
    for k, p in enumerate(e_par):
        ent_by_hop.setdefault(hop[p], []).append(k)
    for h in sorted(by_hop):
        for i in by_hop[h]:
            p = parent[i]
            disc_chain[i] = (first_chain[p] if p < n_first else entry_chain[p - n_first]) + ARROW + disc_name[i]
        for k in ent_by_hop.get(h, ()):
            entry_chain[k] = disc_chain[e_par[k]] + ARROW + servers[e_srv[k]]
    creds = enc.creds
    cred = arr.cred.tolist()
    out: list = []
    sig_off, cred_off = arr.sig_off.tolist(), arr.cred_off.tolist()
    for s in range(len(sig_off) - 1):
        a, b = sig_off[s], sig_off[s + 1]
        if a == b:
            out.append(None)
            continue
        recs = [(disc_name[i], obj_type[occ_obj[occ[i]]], hop[i], disc_chain[i]) for i in range(a, b)]
        out.append((max(hop[a:b]), recs, [creds[c] for c in cred[cred_off[s]:cred_off[s + 1]]]))
    return out


def apply(blast_radii, enc: Encoding, per_sig) -> None:
    """Write each signature's result into its blast radii: fresh lists and dicts per blast radius, risk from its own score."""
    for members, res in zip(enc.sig_members, per_sig):
        if res is None:
            continue
        depth, recs, creds = res
        factor = HOP_RISK_FACTORS.get(depth, 0.25)
        for b in members:
            br = blast_radii[b]
            br.hop_depth = depth
            br.delegation_chain = [r[3] for r in recs]
            br.transitive_agents = [{"name": n, "type": t, "hop": h, "chain": c} for n, t, h, c in recs]
            br.transitive_credentials = list(creds)
            br.transitive_risk_score = round(br.risk_score * factor, 2)


def expand_blast_radius_hops(blast_radii, agents, max_depth: int = 1, *, device: int = 0, batch: int = 0) -> None:
    """Drop-in for the reference's ``expand_blast_radius_hops``: mutates ``blast_radii`` in place.  At a clamped depth of 1 it
    returns without touching anything (and without a device)."""
    depth = clamp_depth(max_depth)
    if depth <= 1:
        return
    blast_radii = list(blast_radii)
    enc = encode(blast_radii, agents)
    apply(blast_radii, enc, materialise(enc, search(enc, depth, device=device, batch=batch)))
