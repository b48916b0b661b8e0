"""Scan-time graph-delta alerts (reference ``graph/webhooks.py:75-261`` ``compute_delta_alerts``) with the node part on the device.

After a scan the new graph is compared with the tenant's previous snapshot.  The reference takes Python set differences over
every node id; here the device diff (``graph/delta.py``, ``csrc/delta.cuh``) returns the new and the removed real nodes in id
order, and their entity-type and severity codes pick the candidates without touching a record.  Attribute reads, the
attack-path and interaction-risk key differences and the event relationships are small and stay on the host.

Order: the reference walks ``new_node_ids - old_node_ids`` and builds the ``agent_removed`` node list in Python *set* order,
which changes from run to run.  Here both are in id order; every other list is in the reference's order.

The canonical event references of ``agent_bom/event_normalization.py:27-93`` and the redaction rules they apply
(``agent_bom/security.py``) are restated below.
"""

from __future__ import annotations

import base64
import binascii
import math
import re
from collections import Counter
from typing import Any
from urllib.parse import urlsplit, urlunsplit

import numpy as np

from .schema import ENTITY_CODE, SEVERITY_RANK, enum_value

# ── redaction rules (reference security.py), restated ──
_ANSI_ESCAPE_RE = re.compile(r"\x1b\[[0-?]*[ -/]*[@-~]")
_SENSITIVE_PATTERNS = [r"token", r"password", r"secret", r"api[_-]?key", r"auth", r"credential", r"bearer", r"jwt"]
_VALUE_CREDENTIAL_PATTERNS = [
    re.compile(r"(?:sk|pk|rk)[-_](?:live|test|prod)[-_]\w{10,}", re.I),
    re.compile(r"(?:ghp|gho|ghu|ghs|ghr)_[A-Za-z0-9_]{30,}"),
    re.compile(r"(?:AKIA|ASIA)[A-Z0-9]{16}"),
    re.compile(r"-----BEGIN (?:RSA |EC |DSA )?PRIVATE KEY-----"),
    re.compile(r"eyJ[A-Za-z0-9_-]{20,}\.eyJ[A-Za-z0-9_-]{20,}"),
    re.compile(r"xox[bpsar]-[A-Za-z0-9-]{10,}"),
    re.compile(r"\w+://[^:]+:[^@]+@"),
]
_B64_RE = re.compile(r"^[A-Za-z0-9+/\-_]+=*$")
_CLOUD_IDENTITY_KEYS = {"account_id", "arn", "cloud_principal", "endpoint_id", "location", "principal_arn", "project_id", "region", "resource_group",
                        "resource_id", "resource_name", "service", "subscription_id", "tenant_id"}
REDACTED = "***REDACTED***"


def _log_label(value: object, max_len: int = 500) -> str:
    text = _ANSI_ESCAPE_RE.sub("", str(value))
    text = text.replace("\r", " ").replace("\n", " ").replace("\t", " ")
    text = "".join(ch for ch in text if ch >= " " and ch != "\x7f")
    return re.sub(r" {2,}", " ", text).strip()[:max_len]


def _entropy(s: str) -> float:
    if not s:
        return 0.0
    n = len(s)
    return -sum((c / n) * math.log2(c / n) for c in Counter(s).values())


def _obfuscated_credential(value: str) -> bool:
    stripped = value.strip()
    if len(stripped) >= 28 and _B64_RE.match(stripped):
        try:
            decoded = base64.b64decode(stripped + "==").decode("utf-8", errors="strict")
            if any(re.search(p, decoded.lower()) for p in _SENSITIVE_PATTERNS) or any(p.search(decoded) for p in _VALUE_CREDENTIAL_PATTERNS):
                return True
        except (ValueError, UnicodeDecodeError, binascii.Error):
            pass
    n = len(stripped)
    if n >= 24 and " " not in stripped and "://" not in stripped:
        return _entropy(stripped) > (5.0 if n < 40 else 4.5)
    return False


def _sensitive_value(value: str) -> bool:
    return any(p.search(value) for p in _VALUE_CREDENTIAL_PATTERNS) or _obfuscated_credential(value)


def _sanitize_url(value: str | None) -> str | None:
    if value is None:
        return None
    try:
        parsed = urlsplit(value)
    except ValueError:
        return "<redacted-url>"
    if not parsed.scheme or not parsed.netloc:
        return value
    host = parsed.hostname or parsed.netloc.rsplit("@", 1)[-1]
    if parsed.port:
        host = f"{host}:{parsed.port}"
    return urlunsplit((parsed.scheme, host, parsed.path, "", ""))


def _sanitize_text(value: object, max_len: int = 1000) -> str:
    text = _log_label(value, max_len=max_len)
    text = re.sub(r"https?://[^\s\"'<>]+", lambda m: str(_sanitize_url(m.group(0)) or ""), text)
    for pattern in _VALUE_CREDENTIAL_PATTERNS:
        text = pattern.sub("<redacted>", text)
    return text[:max_len]


def _key_sensitive(key: object) -> bool:
    return any(re.search(p, str(key).lower()) for p in _SENSITIVE_PATTERNS)


def _key_url(key: object) -> bool:
    k = str(key).lower()
    return k in {"url", "uri", "endpoint", "webhook"} or k.endswith(("_url", "_uri", "_endpoint", "_webhook"))


def _key_path(key: object) -> bool:
    k = str(key).lower()
    return any(t in k for t in ("path", "file", "dir", "directory", "cwd", "workspace", "config_path", "source_path"))


def _path_value(value: str) -> bool:
    if not value or "://" in value:
        return False
    return value.startswith("/") or value.startswith("~/") or bool(re.match(r"^[A-Za-z]:[\\/]", value))


def _key_cloud_identity(key: object) -> bool:
    k = str(key or "").strip().lower().replace("-", "_")
    return k in _CLOUD_IDENTITY_KEYS or k.endswith("_arn") or k.endswith("_resource_id")


def _path_label(value: object) -> str:
    text = _log_label(value, max_len=1000)
    if re.fullmatch(r"<path:[^<>]+>", text):
        return text
    base = re.split(r"[\\/]+", text.rstrip("/\\"))[-1] if text else ""
    base = _sanitize_text(base or "path", max_len=80)
    if not base or _key_sensitive(base) or _sensitive_value(base):
        base = "path"
    return f"<path:{base}>"


def sanitize_payload(value: object, *, key: object | None = None, max_str_len: int = 1000, depth: int = 0) -> object:
    """``sanitize_sensitive_payload`` (reference security.py:438-470)."""
    if depth >= 8:
        return "[truncated]"
    if value is None or isinstance(value, bool | int | float):
        return value
    if isinstance(value, str):
        if key is not None and _key_sensitive(key):
            return REDACTED
        if key is not None and _key_url(key):
            return _sanitize_url(value)
        if key is not None and _key_cloud_identity(key):
            return REDACTED if _sensitive_value(value) else _sanitize_text(value, max_len=max_str_len)
        if "://" in value:
            return _sanitize_text(value, max_len=max_str_len)
        if key is not None and _key_path(key) and _path_value(value):
            return _path_label(value)
        if _path_value(value):
            return _path_label(value)
        if _sensitive_value(value):
            return REDACTED
        return _sanitize_text(value, max_len=max_str_len)
    if isinstance(value, dict):
        out: dict[str, object] = {}
        for k, v in value.items():
            ck = _sanitize_text(k, max_len=200)
            out[ck] = sanitize_payload(v, key=ck, max_str_len=max_str_len, depth=depth + 1)
        return out
    if isinstance(value, list | tuple | set):
        return [sanitize_payload(v, key=key, max_str_len=max_str_len, depth=depth + 1) for v in list(value)]
    return _sanitize_text(value, max_len=max_str_len)


# ── canonical event references (reference event_normalization.py:27-93), restated ──
def event_ref(*, ref_type: str, ref_id: str, name: str | None = None, role: str | None = None, attributes=None) -> dict[str, Any] | None:
    safe_id = sanitize_payload(ref_id, key=ref_type)
    safe_name = sanitize_payload(name, key=ref_type) if name else None
    if not safe_id:
        return None
    ref: dict[str, Any] = {"type": ref_type, "id": str(safe_id)}
    if safe_name:
        ref["name"] = str(safe_name)
    if role:
        ref["role"] = role
    scalars = {_sanitize_text(k, max_len=200): sanitize_payload(v, key=k) for k, v in (attributes or {}).items()
               if isinstance(v, (str, int, float, bool)) and v not in ("", None)}
    if scalars:
        ref["attributes"] = scalars
    return ref


def event_relationships(*, source: str, targets: list) -> dict[str, Any] | None:
    clean = [t for t in targets if t]
    if not clean:
        return None
    return {"normalization_version": "1", "source": source, "targets": clean}


def _node_ref(graph, node_id: str, role: str):
    if graph is None:
        return None
    node = graph.nodes.get(node_id)
    if node is None:
        return None
    return event_ref(ref_type=enum_value(node.entity_type), ref_id=node.id, name=node.label, role=role,
                     attributes={"severity": node.severity, "status": enum_value(node.status), "risk_score": node.risk_score})


def _relationships(graph, targets) -> dict[str, Any] | None:
    return event_relationships(source="graph_delta", targets=[_node_ref(graph, nid, role) for nid, role in targets])


# ── the alerts ──
_HIGH_SEVERITIES = [s for s, r in SEVERITY_RANK.items() if r >= 4]


def _new_and_removed(old_graph, new_graph) -> tuple[list[str], list[str], list[str]]:
    """New vulnerability, new misconfiguration and removed agent ids, in id order, from the device diff's node part."""
    from .container import UnifiedGraph
    from .delta import SEVERITY_CODES, delta_table, device_diff

    old = old_graph if old_graph is not None else UnifiedGraph(scan_id="", tenant_id=getattr(new_graph, "tenant_id", ""))
    d = device_diff(old, new_graph)
    added, removed = d["nodes_added"].astype(np.int64), d["nodes_removed"].astype(np.int64)
    t_new = new_graph.csr.node_type[added]
    high = np.isin(delta_table(new_graph).severity[added], [SEVERITY_CODES[s] for s in _HIGH_SEVERITIES])
    ids_new, ids_old = new_graph.csr.node_ids, old.csr.node_ids
    vulns = [ids_new[i] for i in added[(t_new == ENTITY_CODE["vulnerability"]) & high].tolist()]
    misconf = [ids_new[i] for i in added[(t_new == ENTITY_CODE["misconfiguration"]) & high].tolist()]
    agents = [ids_old[i] for i in removed[old.csr.node_type[removed] == ENTITY_CODE["agent"]].tolist()] if old_graph is not None else []
    return vulns, misconf, agents


def compute_delta_alerts(old_graph, new_graph) -> list[dict[str, Any]]:
    """Alert dicts for the critical changes from ``old_graph`` (or ``None``) to ``new_graph``, as the reference's
    ``compute_delta_alerts``; graphs of other packages (e.g. the reference's) are adopted without copying records."""
    from .container import UnifiedGraph

    if new_graph is not None and not isinstance(new_graph, UnifiedGraph):
        new_graph = UnifiedGraph.from_graph(new_graph)
    if old_graph is not None and not isinstance(old_graph, UnifiedGraph):
        old_graph = UnifiedGraph.from_graph(old_graph)
    scan = new_graph.scan_id
    vulns, misconf, agents_removed = _new_and_removed(old_graph, new_graph)
    alerts: list[dict[str, Any]] = []
    for nid in vulns:
        node = new_graph.nodes[nid]
        attrs = node.attributes
        details = {"node_ids": [nid], "scan_id": scan, "delta_type": "new_vulnerability", "risk_score": node.risk_score,
                   "cvss_score": attrs.get("cvss_score"), "is_kev": attrs.get("is_kev", False), "affected_agent_count": attrs.get("affected_agent_count", 0)}
        alerts.append({
            "type": "new_vulnerability", "detector": "graph_new_vulnerability", "severity": node.severity,
            "message": f"New {node.severity} vulnerability: {node.label}", "title": f"New {node.severity} vulnerability: {node.label}",
            "description": f"Vulnerability {node.label} appeared in scan {scan}", "node_ids": [nid], "scan_id": scan, "details": details,
            "event_relationships": _relationships(new_graph, [(nid, "affected_finding")]),
            "attributes": {"cvss_score": attrs.get("cvss_score"), "is_kev": attrs.get("is_kev", False), "affected_agent_count": attrs.get("affected_agent_count", 0)},
        })
    for nid in misconf:
        node = new_graph.nodes[nid]
        details = {"node_ids": [nid], "scan_id": scan, "delta_type": "new_misconfiguration", "risk_score": node.risk_score}
        alerts.append({
            "type": "new_misconfiguration", "detector": "graph_new_misconfiguration", "severity": node.severity,
            "message": f"New {node.severity} misconfiguration: {node.label}", "title": f"New {node.severity} misconfiguration: {node.label}",
            "description": f"CIS/SAST finding appeared in scan {scan}", "node_ids": [nid], "scan_id": scan, "details": details,
            "event_relationships": _relationships(new_graph, [(nid, "affected_finding")]),
        })
    old_paths = {(p.source, p.target) for p in old_graph.attack_paths} if old_graph else set()
    for path in new_graph.attack_paths:
        if (path.source, path.target) in old_paths or path.composite_risk < 7.0:
            continue
        details = {"node_ids": path.hops, "scan_id": scan, "delta_type": "new_attack_path", "risk_score": path.composite_risk,
                   "composite_risk": path.composite_risk, "credential_exposure": path.credential_exposure, "vuln_ids": path.vuln_ids}
        title = f"New high-risk attack path: {path.summary or f'{path.source} → {path.target}'}"
        alerts.append({
            "type": "new_attack_path", "detector": "graph_new_attack_path", "severity": "critical" if path.composite_risk >= 9.0 else "high",
            "message": title, "title": title, "description": f"Composite risk {path.composite_risk}/10, {len(path.hops)} hops", "node_ids": path.hops,
            "scan_id": scan, "details": details,
            "event_relationships": _relationships(new_graph, [(path.source, "path_source"), (path.target, "path_target")]),
            "attributes": {"composite_risk": path.composite_risk, "credential_exposure": path.credential_exposure, "vuln_ids": path.vuln_ids},
        })
    old_risks = {(r.pattern, tuple(sorted(r.agents))) for r in old_graph.interaction_risks} if old_graph else set()
    for risk in new_graph.interaction_risks:
        if (risk.pattern, tuple(sorted(risk.agents))) in old_risks or risk.risk_score < 7.0:
            continue
        node_ids = [f"agent:{a}" for a in risk.agents]
        details = {"node_ids": node_ids, "scan_id": scan, "delta_type": "new_interaction_risk", "risk_score": risk.risk_score, "pattern": risk.pattern,
                   "owasp_agentic_tag": risk.owasp_agentic_tag}
        alerts.append({
            "type": "new_interaction_risk", "detector": "graph_new_interaction_risk", "severity": "critical" if risk.risk_score >= 9.0 else "high",
            "message": f"New interaction risk: {risk.pattern}", "title": f"New interaction risk: {risk.pattern}", "description": risk.description,
            "node_ids": node_ids, "scan_id": scan, "details": details,
            "event_relationships": _relationships(new_graph, [(nid, "affected_agent") for nid in node_ids]),
            "attributes": {"risk_score": risk.risk_score, "pattern": risk.pattern, "owasp_agentic_tag": risk.owasp_agentic_tag},
        })
    if agents_removed:
        details = {"node_ids": agents_removed, "scan_id": scan, "delta_type": "agent_removed"}
        alerts.append({
            "type": "agent_removed", "detector": "graph_agent_removed", "severity": "medium",
            "message": f"{len(agents_removed)} agent(s) no longer detected", "title": f"{len(agents_removed)} agent(s) no longer detected",
            "description": f"Agents removed: {', '.join(sorted(agents_removed))}", "node_ids": agents_removed, "scan_id": scan, "details": details,
            "event_relationships": _relationships(old_graph, [(nid, "removed_agent") for nid in agents_removed]),
        })
    return alerts
