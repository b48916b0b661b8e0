"""CPU restatement of the snapshot diff's device part (csrc/delta.cuh) with Python string sorts and set operations.

``DeltaOracle(csr)`` answers ``build_delta_table`` / ``diff`` like ``engine.DeviceGraph`` does, so the host pipeline in
``agent_bom_b200/graph/delta.py`` runs without a GPU (tests/test_delta.py checks it against the reference's goldens) and the device
can be checked against it on seeded random graph pairs (tests/test_gpu_delta.py).
"""

from __future__ import annotations

import numpy as np

CODE_OTHER = 255
TYPE_OTHER = 254


class DeltaOracle:
    def __init__(self, csr):
        self.csr = csr
        self.n_nodes = csr.n_nodes
        self.t = None

    def build_delta_table(self, n_real, ids, id_off, perm, labels, label_off, status, severity, risk, erel, eflag, weight=None) -> None:
        def unpack(buf, off):
            return [bytes(buf[off[i]: off[i + 1]]) for i in range(len(off) - 1)]

        self.t = {"n_real": n_real, "ids": unpack(ids, id_off), "labels": unpack(labels, label_off), "status": np.asarray(status), "severity": np.asarray(severity),
                  "risk": np.asarray(risk, np.float64), "erel": np.asarray(erel), "eflag": np.asarray(eflag),
                  "weight": None if weight is None else np.asarray(weight, np.float64)}

    def diff(self, old: "DeltaOracle", relmap_old, relmap_new) -> dict[str, np.ndarray]:
        a, b = self.t, old.t
        ca, cb = self.csr, old.csr
        pos_a = {s: i for i, s in enumerate(a["ids"])}
        pos_b = {s: i for i, s in enumerate(b["ids"])}
        union = sorted(set(a["ids"]) | set(b["ids"]))
        urank = {s: i for i, s in enumerate(union)}
        order_a = sorted(range(len(a["ids"])), key=lambda i: a["ids"][i])
        order_b = sorted(range(len(b["ids"])), key=lambda i: b["ids"][i])
        na_real, nb_real = a["n_real"], b["n_real"]

        def real_partner(s, pos, n_real):
            p = pos.get(s, -1)
            return p if 0 <= p < n_real else -1

        added = [i for i in order_a if i < na_real and real_partner(a["ids"][i], pos_b, nb_real) < 0]
        removed = [i for i in order_b if i < nb_real and real_partner(b["ids"][i], pos_a, na_real) < 0]
        ch_new, ch_old, ch_flag = [], [], []
        for i in order_a:
            if i >= na_real:
                continue
            p = real_partner(a["ids"][i], pos_b, nb_real)
            if p < 0:
                continue
            ta, tb = int(ca.node_type[i]), int(cb.node_type[p])
            sa, sb, va, vb = int(a["status"][i]), int(b["status"][p]), int(a["severity"][i]), int(b["severity"][p])
            differ = ta != tb or sa != sb or va != vb or not (a["risk"][i] == b["risk"][p]) or a["labels"][i] != b["labels"][p]
            f = 1 if differ else (2 if TYPE_OTHER == ta or CODE_OTHER in (sa, va) else 0)
            if f:
                ch_new.append(i), ch_old.append(p), ch_flag.append(f)

        def keys(t, c, relmap):
            return {(urank[t["ids"][int(s)]], urank[t["ids"][int(d)]], int(relmap[int(r)])): e
                    for e, (s, d, r) in enumerate(zip(c.src.tolist(), c.dst.tolist(), t["erel"].tolist()))}

        ka, kb = keys(a, ca, relmap_new), keys(b, cb, relmap_old)
        e_add = [ka[k] for k in sorted(set(ka) - set(kb))]
        e_rem = [kb[k] for k in sorted(set(kb) - set(ka))]
        ec_new, ec_old = [], []
        weights = a["weight"] is not None and b["weight"] is not None
        for k in sorted(set(ka) & set(kb)):
            x, y = ka[k], kb[k]
            if a["eflag"][x] != b["eflag"][y] or (weights and not (a["weight"][x] == b["weight"][y])):
                ec_new.append(x), ec_old.append(y)
        i32 = lambda v: np.asarray(v, np.int32)
        return {"nodes_added": i32(added), "nodes_removed": i32(removed), "changed_new": i32(ch_new), "changed_old": i32(ch_old),
                "changed_flag": np.asarray(ch_flag, np.uint8), "edges_added": i32(e_add), "edges_removed": i32(e_rem), "echanged_new": i32(ec_new),
                "echanged_old": i32(ec_old)}
