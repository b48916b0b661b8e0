"""Semantic clusters on the host: the key table against the reference's per-node keys, risks and severities, the columnar key
table against the record one, the whole pipeline (with the numpy oracle standing in for the device) against the reference's
clusters and route bodies, argument validation, and refusal without a device.

The hand-made ``kat_clusters`` graph (oracle/make_clusters_golden.py) covers dimensions set and unset, every attribute key the
rules read, empty and multiple data sources, ``name@1.0`` / ``@scope/pkg@1.0`` / empty labels, CVE in the id, the label, only
an attribute, lower case, CWE only and neither, credential providers and label tokens, tool label words, risk scores at the
rounding and threshold edges, upper-case / ``info`` / ``unknown`` severities, a label tie between two keys, relationships
outside the enum, bidirectional, intra-cluster and self-loop edges, and ghost endpoints.
"""

from __future__ import annotations

import numpy as np
import pytest

from clusters_golden import NAMES, case, graph, light_graph, roundtrip
from oracle.clusters_oracle import ClusterOracle

from agent_bom_b200.graph import clusters as cl


def with_oracle(g):
    g._dg = ClusterOracle(g.csr)        # the device graph's cluster calls, answered by the numpy restatement
    return g


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dims_form", ["dict", "object"])
def test_key_table_matches_reference_keys(name, dims_form):
    if dims_form == "object" and "nodes" not in case(name):
        pytest.skip("rebuilt graph")
    c = case(name)
    g = graph(name, dims_form=dims_form)
    t = cl.cluster_table(g)
    n = len(g.nodes)
    got = [[[t.kind[k], t.layer[k], t.key[k], t.label[k]] for k in t.codes[i].tolist() if k >= 0] for i in range(n)]
    assert got == c["keys"]
    assert t.risk[:n].tolist() == c["risk"]
    assert [cl.LEVELS[v] for v in t.level[:n].tolist()] == c["severity"]
    assert (t.codes[n:] == -1).all()


def test_key_table_without_dimensions_attribute():
    """Records without ``dimensions`` (this package's own) count as empty dimensions."""
    g = graph("kat_clusters", dims_form="none")
    t = cl.cluster_table(g)
    ref = case("kat_clusters")
    plain = [i for i, n in enumerate(ref["nodes"]) if not n["dimensions"]]
    got = [[[t.kind[k], t.layer[k], t.key[k], t.label[k]] for k in t.codes[i].tolist() if k >= 0] for i in plain]
    assert got == [ref["keys"][i] for i in plain]
    assert len(plain) < len(ref["nodes"])


def test_columnar_key_table_equals_record_key_table():
    a = cl.cluster_table(light_graph())
    b = cl.cluster_table(light_graph(columnar=True))
    for f in ("codes", "level", "risk"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    for f in ("kind", "layer", "key", "label", "type_names"):
        assert getattr(a, f) == getattr(b, f), f
    assert np.array_equal(np.asarray(a.type_names)[a.etype[: len(a.etype)]], np.asarray(b.type_names)[b.etype])


def test_columnar_key_table_builds_no_node_record():
    g = light_graph(columnar=True)
    cl.cluster_table(g)
    assert not g.nodes._cache


@pytest.mark.parametrize("value, severity, risk, level", [
    (8.99995, "", 89.999, "high"), (8.99996, "", 90.0, "critical"), (89.9996, "", 90.0, "critical"), (89.9994, "", 89.999, "high"),
    (10.0, "", 100.0, "critical"), (10.5, "", 10.5, "low"), (150, "", 100.0, "critical"), (-3.0, "medium", 60.0, "medium"),
    (-1.0, "", 0.0, "none"), (0.0, "info", 20.0, "low"), (0.0999, "", 0.999, "none"), (0.1, "", 1.0, "low"), (3.99996, "", 40.0, "medium"),
    (6.99995, "", 69.999, "medium"), (None, "CRITICAL", 100.0, "critical"), (0.0, "unknown", 0.0, "none"), (95.0, "Low", 95.0, "low"),
])
def test_cluster_risk_and_level_at_boundaries(value, severity, risk, level):
    r = cl.cluster_risk(value, severity)
    assert r == risk
    assert cl.LEVELS[cl.cluster_level(severity, r)] == level


@pytest.mark.parametrize("name", NAMES)
def test_oracle_pipeline_matches_reference_clusters(name):
    c = case(name)
    g = with_oracle(graph(name))
    for m in ("1", "2", "3"):
        got = cl.semantic_clusters(g, min_members=int(m))
        assert roundtrip([x.to_dict() for x in got]) == c["clusters"][m]["clusters"], f"min_members={m}"
        assert cl.semantic_cluster_stats(got) == c["clusters"][m]["stats"]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_pipeline_matches_reference_route_bodies(name):
    g = with_oracle(graph(name))
    for v in case(name)["views"]:
        assert roundtrip(cl.semantic_clusters_view(g, **v["params"])) == v["body"], v["params"]


def test_validation_errors():
    g = with_oracle(graph("kat_clusters"))
    with pytest.raises(ValueError, match=r"Unknown semantic cluster kind\(s\): bogus, zzz"):
        cl.semantic_clusters_view(g, kinds="zzz, package_family,bogus")
    with pytest.raises(ValueError, match="Unknown semantic cluster kind"):
        cl.semantic_clusters_view(g, kinds=["nope"])
    for bad in (0, 101):
        with pytest.raises(ValueError, match="min_members"):
            cl.semantic_clusters_view(g, min_members=bad)
    for bad in (0, 1001):
        with pytest.raises(ValueError, match="limit"):
            cl.semantic_clusters_view(g, limit=bad)
    assert cl.semantic_clusters_view(g, kinds=["cve_family"], min_members=1)["stats"]["cve_family_count"] > 0


def test_empty_graph_view_needs_no_device():
    from agent_bom_b200.graph import UnifiedGraph

    body = cl.semantic_clusters_view(UnifiedGraph(scan_id="s", tenant_id="t", created_at="c"))
    assert body == {"scan_id": "s", "tenant_id": "t", "created_at": "c", "clusters": [],
                    "stats": {"cluster_count": 0, "member_count": 0, **{f"{k}_count": 0 for k in cl.SEMANTIC_CLUSTER_KINDS}},
                    "available_kinds": list(cl.SEMANTIC_CLUSTER_KINDS)}
    assert cl.semantic_clusters(UnifiedGraph()) == []


def test_node_merge_drops_the_key_table():
    from agent_bom_b200.graph import UnifiedGraph, UnifiedNode

    g = UnifiedGraph()
    g.add_node(UnifiedNode(id="a", entity_type="agent", label="a"))
    first = cl.cluster_table(g)
    g.add_node(UnifiedNode(id="a", entity_type="agent", label="a", attributes={"fleet": "ops"}))
    assert cl.cluster_table(g) is not first
    assert cl.cluster_table(g).key == ["ops"]


def test_refuses_without_a_device():
    from agent_bom_b200 import _lib

    if _lib.load().abb_device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(_lib.EngineUnavailable):
        cl.semantic_clusters_view(graph("kat_clusters"))
