#!/usr/bin/env python3
"""Kernel-by-kernel breakdown of the device-resident exposure-path pipeline (DevicePaths.count + fill) at one bench workload.

    python profiles/paths_profile.py [--workload L] [--seed 2145] [--out DIR]

Builds the bench estate, sizes the row buffers with one fitted pass, warms up, then times count + fill with CUDA events over
--steps passes and records ONE further pass under torch.profiler (CUDA activities).  Every device activity of that pass is
listed in stream order with its duration and the idle gap before it; the gaps in front of the two 8-byte device-to-host
copies are the count pass's host synchronisations.  Writes DIR/paths_profile_<workload>.json and .md (DIR defaults to a
directory under the system's temporary directory).  ABB_LIB selects an
experiment build of the engine (A/B runs).
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [p.strip() for p in out.split(",")]
        return {"gpu": name, "power_limit_w": float(pl), "sm_clock_max_mhz": int(float(clk))}
    except Exception as e:  # pragma: no cover
        return {"gpu": None, "error": str(e)}


def device_activities(prof) -> list:
    """Kernels, copies and memsets of a torch.profiler capture, in start order (read from its Chrome trace)."""
    with tempfile.TemporaryDirectory() as td:
        tp = Path(td) / "trace.json"
        prof.export_chrome_trace(str(tp))
        trace = json.loads(tp.read_text())
    return sorted((e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")),
                  key=lambda e: e["ts"])


def kernel_name(e: dict) -> str:
    name = e["name"]
    if e["cat"] != "kernel":
        return name
    name = name.split("(")[0].replace("void ", "").replace("abb::", "")
    if "cub::" in e["name"] or "DeviceScan" in name or "DeviceSelect" in name or "DeviceCompact" in name:
        return "cub " + name.split("<")[0].replace("cub::", "").split("::")[-1]
    # keep the template argument of count/fill kernels
    return name.replace("<(bool)0>", "<false>").replace("<(bool)1>", "<true>").replace("<0>", "<false>").replace("<1>", "<true>")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="L")
    ap.add_argument("--seed", type=int, default=2145)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "abb_paths_profile"), help="directory for the .json / .md tables")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from agent_bom_b200 import dist as abdist
    from agent_bom_b200.engine import DeviceGraph
    from agent_bom_b200.torch_api import DevicePaths

    info = abdist.init_from_env(None)
    device = torch.device("cuda", 0)
    est, _ = bench.generate_estate(args.workload, args.seed)
    host = bench.device_csr(est)
    tensors, n_nodes, n_entries = abdist.broadcast_csr(host, info, device)
    findings = abdist.broadcast_array(est.findings, info, device)
    dg = DeviceGraph.adopt(tensors, n_nodes, n_entries, 0)
    nf = int(findings.shape[0])

    paths = DevicePaths(dg, nf)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with profile(activities=[ProfilerActivity.CUDA]) as prof0:
        rows = paths.run_fitted(findings)      # the first call also builds the graph-constant server and exposure tables
        torch.cuda.synchronize()
    first_ms = 1000.0 * (time.perf_counter() - t0)
    one_time = {}
    for e in device_activities(prof0):
        name = kernel_name(e)
        if name.startswith(("server_", "node_links_kernel", "template_kernel")):
            one_time[name] = one_time.get(name, 0.0) + e["dur"] / 1000.0

    def one():
        paths.count(findings)
        paths.fill(findings)

    for _ in range(3):
        one()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    ev[0].record()
    for i in range(args.steps):
        one()
        ev[i + 1].record()
    torch.cuda.synchronize()
    per = [ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps)]

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        one()
        torch.cuda.synchronize()
    acts = device_activities(prof)
    timeline, prev_end = [], None
    for e in acts:
        name = kernel_name(e)
        gap = 0.0 if prev_end is None else max(0.0, e["ts"] - prev_end)
        timeline.append({"what": name, "kind": e["cat"], "us": float(e["dur"]), "gap_before_us": float(gap),
                         "bytes": (e.get("args") or {}).get("bytes")})
        prev_end = e["ts"] + e["dur"] if prev_end is None else max(prev_end, e["ts"] + e["dur"])
    span_us = (acts[-1]["ts"] + acts[-1]["dur"] - acts[0]["ts"]) if acts else 0.0
    by_kernel: dict = {}
    for t in timeline:
        by_kernel.setdefault(t["what"], 0.0)
        by_kernel[t["what"]] += t["us"]

    rec = {**gpu_info(), "workload": args.workload, "seed": args.seed, "findings": nf, "rows": rows,
           "row_bytes": rows * 28, "engine_lib": os.environ.get("ABB_LIB", "libabb200.so"),
           "first_call_ms": first_ms, "table_kernels_ms": one_time, "count_fill_ms": {"steps": args.steps, "per_step": per, "min": min(per), "median": sorted(per)[len(per) // 2]},
           "profiled_pass": {"span_ms": span_us / 1000.0, "busy_ms": sum(t["us"] for t in timeline) / 1000.0,
                             "idle_ms": sum(t["gap_before_us"] for t in timeline) / 1000.0, "timeline": timeline, "by_kernel_us": by_kernel}}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    tag = f"paths_profile_{args.workload}" + (f"_{os.environ['ABB_LIB'].replace('.so', '')}" if os.environ.get("ABB_LIB") else "")
    (out / f"{tag}.json").write_text(json.dumps(rec, indent=1))
    lines = [f"# {tag}: {rec.get('gpu')} at {rec.get('power_limit_w')} W power limit", "",
             f"{nf:,} findings, {rows:,} rows ({rows * 28 / 1e9:.2f} GB written). count+fill over {args.steps} passes (CUDA events): "
             f"median {rec['count_fill_ms']['median']:.3f} ms, min {rec['count_fill_ms']['min']:.3f} ms. Profiled pass: span "
             f"{span_us / 1000:.3f} ms, device busy {rec['profiled_pass']['busy_ms']:.3f} ms, idle {rec['profiled_pass']['idle_ms']:.3f} ms.", "",
             f"One-time graph-constant server and exposure tables (first call): {', '.join(f'`{k}` {v:.3f} ms' for k, v in one_time.items())}.", "",
             "| # | activity | kind | bytes | time (us) | idle before (us) |", "|---|---|---|---|---|---|"]
    for i, t in enumerate(timeline):
        lines.append(f"| {i} | `{t['what']}` | {t['kind']} | {t['bytes'] if t['bytes'] is not None else ''} | {t['us']:.1f} | {t['gap_before_us']:.1f} |")
    (out / f"{tag}.md").write_text("\n".join(lines) + "\n")
    print(json.dumps({k: rec[k] for k in ("gpu", "power_limit_w", "rows", "count_fill_ms", "table_kernels_ms")}))
    print("\n".join(lines))


if __name__ == "__main__":
    main()
