"""Profile the multi-hop blast-radius expansion (agent_bom_b200.blast_radius) on seeded clique fleets.

Fleets: ``oracle.hops_oracle.clique_fleet(n, seed=7)`` for n = 1 000 and 4 000 agents (cliques of 50 agents chained through
their first member, so hops 4 and 5 occur at depth 5), four blast radii per server name, at depths 2, 3 and 5.  Per fleet and
depth, medians over ``--reps`` warm calls of:

- encode: host interning, both CSRs and signature grouping;
- upload / search / readback: inside ``abb_hops_host`` (search is CUDA-event time of the batch's kernels and count readbacks);
- normalise: the signature sort of the returned arrays; materialise: chain strings and per-signature lists; apply: the
  per-blast-radius lists and dicts;
- end to end: the drop-in ``expand_blast_radius_hops`` on fresh objects.

The card's name and power limit are read in the same run.  Writes DIR/h100_blast_radius_hops_profile.json.
The reference's times on the same fleets (a CPU host) are in profiles/blast_radius_hops_reference.json; the two files are
not a like-for-like comparison.
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))
sys.path.insert(0, str(ROOT / "tests"))

from hops_golden import objects  # noqa: E402
from paths_profile import gpu_info  # noqa: E402

from agent_bom_b200 import blast_radius as hops  # noqa: E402
from oracle import hops_oracle  # noqa: E402


def profile(n: int, depth: int, reps: int) -> dict:
    data = hops_oracle.clique_fleet(n, 7)
    runs = []
    for _ in range(reps + 1):
        agents, radii = objects(data)
        t = {}
        t0 = time.perf_counter()
        enc = hops.encode(radii, agents)
        t1 = time.perf_counter()
        arr = hops.search(enc, depth)
        t2 = time.perf_counter()
        per_sig = hops.materialise(enc, arr)
        t3 = time.perf_counter()
        hops.apply(radii, enc, per_sig)
        t4 = time.perf_counter()
        t = {"encode_s": t1 - t0, "upload_s": arr.stats["upload_ms"] / 1e3, "search_s": arr.stats["search_ms"] / 1e3,
             "readback_s": arr.stats["readback_ms"] / 1e3,
             "normalise_s": (t2 - t1) - (arr.stats["upload_ms"] + arr.stats["search_ms"] + arr.stats["readback_ms"]) / 1e3,
             "materialise_s": t3 - t2, "apply_s": t4 - t3}
        agents, radii = objects(data)
        t0 = time.perf_counter()
        hops.expand_blast_radius_hops(radii, agents, max_depth=depth)
        t["end_to_end_s"] = time.perf_counter() - t0
        runs.append(t)
        stats = arr.stats
    runs = runs[1:]                                     # the first call loads the module and warms the allocator
    rec = {"agents": n, "depth": depth, "blast_radii": len(radii), "signatures": len(enc.sig_members), "discoveries": stats["discoveries"],
           "later_entries": stats["entries"], "credential_keys": stats["cred_keys"], "batches": stats["batches"], "batch_size": stats["batch_size"],
           "transitive_entries": sum(len(br.transitive_agents) for br in radii),
           "max_hop": max((br.hop_depth for br in radii if br.transitive_agents), default=1)}
    rec["median_s"] = {k: round(statistics.median(r[k] for r in runs), 4) for k in runs[0]}
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="1000,4000")
    ap.add_argument("--depths", default="2,3,5")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="hops_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    doc = {"device": gpu_info(), "fleet": "oracle.hops_oracle.clique_fleet(n, seed=7): cliques of 50, four blast radii per server name",
           "timing": "median of warm calls; search_s is CUDA-event time, the rest host clocks", "rows": []}
    for n in (int(x) for x in a.sizes.split(",")):
        for d in (int(x) for x in a.depths.split(",")):
            doc["rows"].append(profile(n, d, a.reps))
            print(json.dumps(doc["rows"][-1]), flush=True)
            (out / "h100_blast_radius_hops_profile.json").write_text(json.dumps(doc, indent=1) + "\n")
    print(f"-> {out / 'h100_blast_radius_hops_profile.json'}")


if __name__ == "__main__":
    main()
