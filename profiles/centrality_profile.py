#!/usr/bin/env python3
"""Time the NetworkX analysis backend's centralities on the GPU (B200NetworkXBackend).

    python profiles/centrality_profile.py [--out FILE] [--estates 150,1000,M1]

Per estate (generator estates as DiGraphs, weights varied by relationship, seed 2145): ``centrality_scores`` (PageRank) and
``bottleneck_nodes`` (exact betweenness) timed with CUDA events after one warm-up call, the kernels of one call of each with
torch.profiler in a separate pass, and the work the oracle counts: forward adjacency entries scanned over all sources
(betweenness is reported as those entries per second).  PageRank is reported per power iteration, with the share of the
serial dangling-sum kernel.  The card's name and power limit are read in the same run.  A GPU is required.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power, clock = [x.strip() for x in out.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import nx_oracle
    from test_gpu_networkx_backend import estate_backend
    from agent_bom_b200 import estate

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "abb_centrality_profile" / "h100_centrality_profile.json"),
                    help="JSON file to write (profiles/h100_centrality_profile.json holds the committed run)")
    ap.add_argument("--estates", default="150,1000,M1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU only")
    shapes = {"150": (150, estate.Knobs()), "1000": (1000, estate.Knobs()), "M1": (2000, estate.BENCH_KNOBS)}
    result = {"card": card(), "estates": {}}

    def timed(fn, reps):
        fn()                                          # warm-up: upload, module load, scratch
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(reps):
            start.record()
            fn()
            end.record()
            end.synchronize()
            times.append(start.elapsed_time(end))
        return times

    for key in args.estates.split(","):
        agents, knobs = shapes[key]
        b, g = estate_backend(agents, knobs)
        dg = b.device_graph
        _, iters = dg.pagerank(b.weights)
        t0 = time.perf_counter()
        _, scanned = nx_oracle.betweenness(g)
        oracle_s = time.perf_counter() - t0
        reps_bc = 3 if key != "M1" else 1
        pr_ms = timed(b.centrality_scores, 10)
        bc_ms = timed(lambda: b.bottleneck_nodes(5), reps_bc)
        kern = {}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            b.centrality_scores()
            b.bottleneck_nodes(5)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                kern[ev.key] = {"calls": ev.count, "total_ms": ev.device_time_total / 1e3}
        dsum_ms = sum(v["total_ms"] for k, v in kern.items() if "pr_dangling_sum" in k)
        pr_kernel_ms = sum(v["total_ms"] for k, v in kern.items() if "nx" in k and "pr_" in k)
        bc_best = min(bc_ms)
        result["estates"][key] = {
            "agents": agents, "nodes": g.n, "adjacency_entries": int(g.foff[-1]),
            "pagerank": {"call_ms": pr_ms, "iterations": iters, "ms_per_iteration": min(pr_ms) / iters,
                         "kernel_ms": pr_kernel_ms, "dangling_sum_ms": dsum_ms, "dangling_sum_share_of_kernels": dsum_ms / pr_kernel_ms if pr_kernel_ms else None},
            "betweenness": {"call_ms": bc_ms, "entries_scanned": scanned, "entries_per_s": scanned / (bc_best / 1e3),
                            "oracle_cpu_s": oracle_s},
            "kernels": kern,
        }
        print(json.dumps({key: {k: v for k, v in result["estates"][key].items() if k != "kernels"}}), flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(result, indent=1, sort_keys=True))
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
