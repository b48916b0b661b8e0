#!/usr/bin/env python3
"""Cost of the compliance posture (``graph/compliance.py``) through ``B200GraphStore`` on the M1 and M2 columnar estates saved to SQLite.

    python profiles/compliance_profile.py [--out DIR] [--sizes M1,M2] [--reps 5]
    python profiles/compliance_profile.py --reference [--out DIR] [--sizes M1] [--reps 3] [--timeout 300]
                                        # the same calls on the unmodified SQLite store (needs the reference)

The estate is written as search_profile.py writes it; then every finding node (entity type ``vulnerability``) gets a seeded
``compliance_tags`` list drawn from a vocabulary shaped like the reference builder's tag lists (OWASP LLM, ATLAS, ATT&CK, NIST AI
RMF, OWASP MCP / agentic, EU AI Act, NIST CSF, ISO 27001, SOC 2, CIS) plus ``skill_audit:`` tags.  Recorded: the first call's host
steps (the SQL read, the decode and interning, turning the table into the answer) and the device table build timed separately,
the first call end to end on a fresh store, the table's device bytes, and warm calls (median of --reps after one warm call)
unfiltered and filtered.  Kernel times of the table build are taken under torch.profiler in a separate build.  The card's name
and power limit are read in the same run.  Writes DIR/compliance_profile.json (``--reference``: DIR/compliance_reference.json).
"""

from __future__ import annotations

import argparse
import json
import random
import sqlite3
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "profiles"))

from search_profile import timed, write_db  # noqa: E402

VOCAB = [
    ["LLM01", "LLM02", "LLM05", "LLM06", "LLM08"], ["AML.T0010", "AML.T0051", "AML.T0054"], ["T1059", "T1195.002", "T1552"],
    ["GOVERN-1.1", "MAP-3.4", "MEASURE-2.7", "MANAGE-4.1"], ["MCP01", "MCP04", "MCP07"], ["ASI01", "ASI03", "ASI06"], ["ART-9", "ART-15"],
    ["ID.RA-01", "PR.DS-01", "DE.CM-08"], ["A.5.23", "A.8.8", "A.8.28"], ["CC6.1", "CC7.1", "CC8.1"], ["CIS-2.1", "CIS-7.4", "CIS-16.1"],
    ["skill_audit:credential_exposure", "skill_audit:shell_access"],
]
CALLS = {"all": "", "owasp_llm05": "llm05", "cis": "cis", "absent": "absent"}


def tag_db(size: str, work: Path) -> tuple[Path, dict]:
    db, rec = write_db(size, work)
    conn = sqlite3.connect(str(db))
    rng = random.Random(2145)
    ids = [r[0] for r in conn.execute("SELECT id FROM graph_nodes WHERE scan_id = 'old' AND entity_type = 'vulnerability'")]
    rows = []
    for nid in ids:
        tags = sorted({t for words in VOCAB if rng.random() < 0.5 for t in rng.sample(words, rng.randint(1, len(words)))})
        rows.append((json.dumps(tags), nid))
    conn.executemany("UPDATE graph_nodes SET compliance_tags = ? WHERE id = ? AND scan_id = 'old'", rows)
    conn.commit()
    conn.close()
    rec["tagged_nodes"] = sum(1 for t, _ in rows if t != "[]")
    rec["tag_pairs"] = sum(len(json.loads(t)) for t, _ in rows)
    return db, rec


def profile_size(size: str, reps: int, work: Path) -> dict:
    import torch
    from clusters_profile import kernel_table

    from agent_bom_b200.graph.compliance import ROWS_SQL, ComplianceInputs, summarize
    from agent_bom_b200.graph.lookup import connect
    from agent_bom_b200.store import B200GraphStore

    db, rec = tag_db(size, work)
    store = B200GraphStore(SimpleNamespace(_db_path=str(db), load_graph=lambda **_: None))
    g = store._graph("", "old")
    dg = g.device_graph
    torch.cuda.synchronize()
    # the first call's steps, one by one
    t0 = time.perf_counter()
    conn = connect(db)
    rows = conn.execute(ROWS_SQL, ("default", "old")).fetchall()
    conn.close()
    t1 = time.perf_counter()
    inputs = ComplianceInputs(rows)
    t2 = time.perf_counter()
    args = (inputs.row_text, inputs.row_sev, inputs.row_type, inputs.text_off, inputs.text_tags, inputs.tag_fw, len(inputs.frameworks),
            len(inputs.severities), len(inputs.types))
    table = dg.compliance_table(*args)                   # returns after the device is done and the table is copied back
    t3 = time.perf_counter()
    summarize(inputs, table)
    t4 = time.perf_counter()
    rec["first_call_steps_s"] = {"sql_read": round(t1 - t0, 4), "decode_intern": round(t2 - t1, 4), "device_table_and_fetch": round(t3 - t2, 4),
                                 "summarize": round(t4 - t3, 4)}
    rec["frameworks"], rec["distinct_tags"], rec["distinct_texts"] = len(inputs.frameworks), len(inputs.tags), len(inputs.text_off) - 1
    t0 = time.perf_counter()
    store.compliance_summary(scan_id="old")
    rec["first_call_store_s"] = round(time.perf_counter() - t0, 4)
    rec["compliance_table_bytes"] = dg.compliance_table_bytes()
    rec["warm"] = {name: timed(lambda f=flt: store.compliance_summary(scan_id="old", framework=f), reps) for name, flt in CALLS.items()}
    rec["table_build_kernels_ms"] = kernel_table(lambda: dg.compliance_table(*args))
    body = store.compliance_summary(scan_id="old")
    rec["answer"] = {"framework_count": body["framework_count"], "total_tagged_findings": body["total_tagged_findings"]}
    db.unlink(missing_ok=True)
    return rec


def _reference_call(db: str, flt: str, reps: int, out) -> None:
    import oracle.make_golden  # noqa: F401  (puts the reference on the path)
    from agent_bom.api.graph_store import SQLiteGraphStore

    store = SQLiteGraphStore(db)
    for _ in range(reps):
        t0 = time.perf_counter()
        store.compliance_summary(scan_id="old", framework=flt)
        out.put(time.perf_counter() - t0)


def reference_size(size: str, reps: int, work: Path, timeout_s: float) -> dict:
    """Each call in a child process of its own, ``reps`` times without a warm-up call, stopped after ``timeout_s``."""
    import multiprocessing as mp
    import statistics

    db, rec = tag_db(size, work)
    ctx = mp.get_context("fork")
    rec["wall"] = {}
    for name, flt in CALLS.items():
        q = ctx.Queue()
        p = ctx.Process(target=_reference_call, args=(str(db), flt, reps, q))
        p.start()
        p.join(timeout_s)
        done = []
        while not q.empty():
            done.append(q.get())
        if p.is_alive():
            p.terminate()
            p.join()
            rec["wall"][name] = {"did_not_finish_within_s": timeout_s, "finished_reps": len(done)}
        else:
            rec["wall"][name] = {"median_ms": round(statistics.median(done) * 1e3, 2), "min_ms": round(min(done) * 1e3, 2), "reps": len(done)}
        print(name, rec["wall"][name], flush=True)
    db.unlink(missing_ok=True)
    return rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="M1,M2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--timeout", type=float, default=300.0, help="--reference: seconds allowed per call")
    a = ap.parse_args()
    out = Path(a.out) if a.out else Path(tempfile.mkdtemp(prefix="compliance_profile_"))
    out.mkdir(parents=True, exist_ok=True)
    work = Path(tempfile.mkdtemp(prefix="compliance_db_"))
    if a.reference:
        import os
        import platform

        doc = {"store": "unmodified reference SQLiteGraphStore, one CPU process per call; a CPU-only host, not a like-for-like comparison "
                        "with the GPU numbers", "host": {"machine": platform.machine(), "cpu_count": os.cpu_count()}, "sizes": {}}
        name = "compliance_reference.json"
    else:
        from paths_profile import gpu_info

        doc = {"device": gpu_info(), "sizes": {}}
        name = "compliance_profile.json"
    for size in a.sizes.split(","):
        doc["sizes"][size] = reference_size(size, a.reps, work, a.timeout) if a.reference else profile_size(size, a.reps, work)
        (out / name).write_text(json.dumps(doc, indent=1))
        print(size, json.dumps(doc["sizes"][size]), flush=True)
    print(f"-> {out / name}")


if __name__ == "__main__":
    main()
