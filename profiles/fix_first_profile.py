#!/usr/bin/env python3
"""Cost of the fix-first view: the focused device ranking at L, and the whole view end to end at M2.

    python profiles/fix_first_profile.py [--out DIR] [--reps 7] [--skip-l]

L (bench estate, 215 K agents): the ranking inputs are built from the estate arrays, then for each case (unfocused top 8, the
heaviest agent, the finding on most rows, a package on few rows) the wall time of ``rank_exposure_paths_focused`` — a synchronous
call: count pass, key pass, compaction, sort, page gather and its copies — is the median of --reps calls after two warm-up calls;
one further call per case runs under torch.profiler and its device time is summed per kernel.  The focus nodes are picked from a
strided sample of the expanded rows; ``matched`` is what the device reports for the full estate.
M2 (20.7 K agents): ``fix_first_view`` on the labelled graph (``Estate.report_json()`` through the columnar builder): the first call
split into device upload, ranking-input build and label-index build, then warm calls per case.
Writes DIR/fix_first_profile.json and .md (DIR defaults to a directory under the system's temporary directory).
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from paths_profile import device_activities, gpu_info, kernel_name  # noqa: E402

AGENTS = {"M2": 20_700, "L": 215_000}


def median_s(fn, reps: int, warm: int = 2) -> float:
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def kernel_table(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out: dict[str, float] = {}
    for e in device_activities(prof):
        k = kernel_name(e)
        out[k] = out.get(k, 0.0) + e["dur"] / 1000.0
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def ranking_inputs_from_arrays(est, host):
    f = np.ascontiguousarray(est.findings)
    base_of_sev = np.asarray([100.0, 80.0, 60.0, 40.0])        # severity rank * 20 (risk_score is 0 in the estates)
    base_vals, base_id = np.unique(base_of_sev[est.node_sev[f]], return_inverse=True)
    scores = np.empty((len(base_vals), 5, 15))
    for bi, b in enumerate(base_vals.tolist()):
        for nc in range(5):
            for nt in range(15):
                risk = b
                risk += min(10.0, nc * 3.0)
                risk += min(10.0, nt * 0.75)
                scores[bi, nc, nt] = round(min(100.0, risk), 2)
    table = np.searchsorted(np.unique(scores), scores).astype(np.uint32)
    # labels are unique per node in the estates: distinct-label counts are the servers' credential / tool edge counts
    meta = host.fwd_meta
    keep = ((meta & 0x80) == 0) & (host.node_type[host.fwd_nbr] != 255)
    row = np.repeat(np.arange(host.n_nodes, dtype=np.int32), np.diff(host.fwd_off.astype(np.int64)))
    rel = meta & 0x1F
    ncu = np.bincount(row[keep & (rel == 4)], minlength=host.n_nodes).astype(np.int32)
    ntu = np.bincount(row[keep & (rel == 3)], minlength=host.n_nodes).astype(np.int32)
    return f, base_id.astype(np.int32), table, ncu, ntu


def profile_l(reps: int) -> dict:
    from agent_bom_b200 import _lib, estate
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.graph import csr as csrmod

    est = estate.generate(AGENTS["L"], 2145, estate.BENCH_KNOBS, exact_rank=False)
    host = csrmod.from_arrays(None, est.node_type, est.src, est.dst, est.rel, est.flags, node_rank=est.node_rank)
    dg = DeviceGraph.upload(host)
    try:
        args = ranking_inputs_from_arrays(est, host)
        sample = dg.exposure_paths_many(np.ascontiguousarray(est.findings[::64]))
        h, t = sample.hops, host.node_type
        ag, n_ag = np.unique(h[:, 0][t[h[:, 0]] == 0], return_counts=True)
        fi, n_fi = np.unique(h[:, 3], return_counts=True)
        vs = h[:, 2][h[:, 2] >= 0]
        pk, n_pk = np.unique(vs[t[vs] == 2], return_counts=True)
        picks = {"heavy_agent": (int(ag[np.argmax(n_ag)]), _lib.FOCUS_AGENT), "heavy_cve": (int(fi[np.argmax(n_fi)]), _lib.FOCUS_CVE),
                 "rare_package": (int(pk[np.argmin(n_pk)]), _lib.FOCUS_PACKAGE)}
        cases = {"unfocused_top8": (None, 0)}
        for name, (node, bit) in picks.items():
            focus = np.zeros(host.n_nodes, dtype=np.uint8)
            focus[node] = bit
            cases[name] = (focus, bit)
        out = {"nodes": host.n_nodes, "edges": int(est.src.shape[0]), "findings": int(args[0].shape[0]), "cases": {}}
        for name, (focus, need) in cases.items():
            def call():
                return dg.rank_exposure_paths_focused(*args, focus, need, 0, 8)
            _, _, total, matched = call()
            wall = median_s(call, reps)
            out["total_rows"] = total
            out["cases"][name] = {"matched": matched, "wall_ms_median": round(wall * 1000, 3), "reps": reps, "device_ms_by_kernel": kernel_table(call)}
            print(name, out["cases"][name], flush=True)
        return out
    finally:
        dg.close()


def profile_m2(reps: int) -> dict:
    from agent_bom_b200 import estate
    from agent_bom_b200.graph import build_unified_graph_from_report, fix_first_view
    from agent_bom_b200.graph.exposure import rank_inputs
    from agent_bom_b200.graph.fix_first import focus_index

    est = estate.generate(AGENTS["M2"], 2145, estate.BENCH_KNOBS, exact_rank=False)
    t0 = time.perf_counter()
    g = build_unified_graph_from_report(est.report_json(), columnar=True)
    out = {"nodes": len(g.nodes), "edges": len(g.edges), "build_graph_s": round(time.perf_counter() - t0, 3)}
    t0 = time.perf_counter(); g.device_graph; out["first_call_device_upload_s"] = round(time.perf_counter() - t0, 3)
    t0 = time.perf_counter(); rank_inputs(g); out["first_call_ranking_inputs_s"] = round(time.perf_counter() - t0, 3)
    t0 = time.perf_counter(); fix_first_view(g); out["first_call_unfocused_view_s"] = round(time.perf_counter() - t0, 3)
    top = fix_first_view(g, limit=25)
    t0 = time.perf_counter(); focus_index(g); out["first_focused_call_label_index_s"] = round(time.perf_counter() - t0, 3)
    cards = top["cards"]
    cases = {"unfocused_top8": {}, "top_card_agent": {"agent": cards[0]["affected"]["agents"][0]},
             "top_card_cve": {"cve": cards[0]["affected"]["findings"][0]},
             "package_of_last_card": {"package": next((c["affected"]["packages"][0] for c in reversed(cards) if c["affected"]["packages"]), "")}}
    out["total_paths"] = top["summary"]["total_paths"]
    out["cases"] = {}
    for name, focus in cases.items():
        view = fix_first_view(g, **focus)
        wall = median_s(lambda: fix_first_view(g, **focus), reps)
        out["cases"][name] = {"focus": focus, "matched": view["summary"]["matched_paths"], "warm_ms_median": round(wall * 1000, 3), "reps": reps}
        print(name, out["cases"][name], flush=True)
    return out


def markdown(rec: dict) -> str:
    gi = rec["gpu"]
    lines = [f"# fix-first view cost — {gi.get('gpu')} at a {gi.get('power_limit_w')} W power limit", ""]
    if rec.get("L"):
        L = rec["L"]
        lines += [f"## L: focused ranking ({L['nodes']:,} nodes, {L['total_rows']:,} exposure-path rows)", "",
                  "| case | matched rows | wall ms (median) | rank_keys_kernel ms | radix sort ms | select ms (count pass + focus compaction) | H2D copies ms |", "|---|---:|---:|---:|---:|---:|---:|"]
        for name, c in L["cases"].items():
            k = c["device_ms_by_kernel"]
            sort = sum(v for n, v in k.items() if "RadixSort" in n)
            comp = sum(v for n, v in k.items() if "Select" in n or "Compact" in n or "gather_keys" in n)
            h2d = sum(v for n, v in k.items() if n.startswith("Memcpy HtoD"))
            lines.append(f"| {name} | {c['matched']:,} | {c['wall_ms_median']} | {k.get('rank_keys_kernel', 'not measured')} | {round(sort, 3)} | {round(comp, 3)} | {round(h2d, 3)} |")
        lines.append("")
    if rec.get("M2"):
        M = rec["M2"]
        lines += [f"## M2: fix_first_view end to end ({M['nodes']:,} nodes, {M['edges']:,} edges, {M['total_paths']:,} paths)", "",
                  f"First call: device upload {M['first_call_device_upload_s']} s, ranking inputs {M['first_call_ranking_inputs_s']} s, "
                  f"unfocused view after those {M['first_call_unfocused_view_s']} s; the first focused call adds the label index, {M['first_focused_call_label_index_s']} s.", "",
                  "| case | matched paths | warm ms (median) |", "|---|---:|---:|"]
        for name, c in M["cases"].items():
            lines.append(f"| {name} | {c['matched']:,} | {c['warm_ms_median']} |")
        lines.append("")
    return "\n".join(lines)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--skip-l", action="store_true")
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "abb_fix_first_profile"), help="directory for the .json / .md tables")
    args = ap.parse_args()
    from agent_bom_b200 import _lib

    _lib.require_device()
    rec = {"gpu": gpu_info(), "command": " ".join(["python", "profiles/fix_first_profile.py", *sys.argv[1:]]),
           "M2": profile_m2(args.reps), "L": None if args.skip_l else profile_l(args.reps)}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "fix_first_profile.json").write_text(json.dumps(rec, indent=1) + "\n")
    (out / "fix_first_profile.md").write_text(markdown(rec))
    print(markdown(rec))


if __name__ == "__main__":
    main()
