"""Payload -> flat POD tables: the IN side of the drop-in boundary.

Takes what the reference's ``SimulationRunner`` takes -- a validated
``SimulationPayload`` (reference ``schemas/payload.py:12-18``) or the YAML-shaped
``dict`` it is validated from (``runtime/simulation_runner.py:396-398``) -- and
produces the ``AfScenario`` the C ABI uploads (``include/asyncflow_b200.h``).

The Pydantic schemas are *reused*, not re-implemented: when the reference
package is importable the payload arrives validated and ``model_dump`` supplies
every default.  On a box without the reference (the GPU box) a plain dict is
accepted and only the schema DEFAULTS are restated here
(``config/constants.py:23-40,113-137,222-230``); structural validation is then
limited to what the engine itself needs (``af_host_common.h: validate``).

What the flattening resolves once, on the host, instead of per event:

* node ids -> indices, each edge's target inbox (``simulation_runner.py:205-260``);
* RAM steps are summed into ``total_ram`` and dropped from the step list
  (``runtime/actors/server.py:106-110``: reserved up front, no-ops in the loop);
* the two injection timelines are sorted with the reference's key
  ``(t, mark == start, event_id, target_id)`` and their f64 FIRE times are
  accumulated exactly like ``dt = t - last_t; yield timeout(dt)`` does
  (``runtime/events/injection.py:142-151,185-188``).
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Any

import numpy as np

from . import _capi as K

CPU_KINDS = {"initial_parsing", "cpu_bound_operation"}
IO_KINDS = {"io_task_spawn", "io_llm", "io_wait", "io_db", "io_cache"}
RAM_KINDS = {"ram"}
ALL_SAMPLED = ("ready_queue_len", "event_loop_io_sleep", "ram_in_use",
               "edge_concurrent_connection")


def _s(x: Any) -> str:
    """Enum members and plain strings alike -> their string value."""
    return str(getattr(x, "value", x))


def _as_dict(payload: Any) -> dict:
    if isinstance(payload, dict):
        return payload
    if hasattr(payload, "model_dump"):  # a reference SimulationPayload
        return payload.model_dump()
    msg = f"unsupported payload type {type(payload)!r}"
    raise TypeError(msg)


def _rv(d: dict) -> tuple[str, float, float]:
    dist = _s(d.get("distribution") or "poisson")
    var = d.get("variance")
    if var is None and dist in ("normal", "log_normal"):
        var = d["mean"]          # RVConfig.default_variance (schemas/common/random_variables.py)
    return dist, float(d["mean"]), 0.0 if var is None else float(var)


@dataclass
class FlatScenario:
    """The POD plus the names needed to map results back to ids."""

    pod: K.AfScenario
    edge_ids: list[str]
    server_ids: list[str]
    client_id: str
    generator_id: str
    lb_id: str | None
    endpoint_names: list[str]
    step_index: dict[tuple[str, int, int], int]        # (server, endpoint, original step idx) -> AfStep
    endpoint_index: dict[tuple[str, int], int]
    spike_mark_events: list[tuple[str, str]]           # (event_id, start|end) per AfSpikeMark
    horizon_s: int
    sample_period: float
    enabled_metrics: list[str]
    _keep: list = field(default_factory=list, repr=False)

    @property
    def n_edges(self) -> int:
        return len(self.edge_ids)

    @property
    def n_servers(self) -> int:
        return len(self.server_ids)

    @property
    def n_series(self) -> int:
        return 3 * self.n_servers + self.n_edges


def _timeline(marks: list[tuple[float, str, str, str]]) -> list[float]:
    """Fire times of a sorted timeline: injection.py:178-188 in f64."""
    now = 0.0
    last_t = 0.0
    out = []
    for t, *_ in marks:
        dt = t - last_t
        if dt > 0.0:
            now = now + dt
        last_t = t
        out.append(now)
    return out


def flatten(payload: Any) -> FlatScenario:
    p = _as_dict(payload)
    gen = p["rqs_input"]
    topo = p["topology_graph"]
    nodes = topo["nodes"]
    ss = p.get("sim_settings") or {}
    events = p.get("events") or []

    udist, umean, usigma = _rv(gen["avg_active_users"])
    if udist not in ("poisson", "normal"):
        msg = "avg_active_users must be poisson or normal (schemas/workload/rqs_generator.py)"
        raise ValueError(msg)
    _, rpm, _ = _rv(gen["avg_request_per_minute_per_user"])
    window = int(gen.get("user_sampling_window") or 60)
    horizon = int(ss.get("total_simulation_time") or 3600)
    period = float(ss.get("sample_period_s") or 0.01)
    esm = ss.get("enabled_sample_metrics")
    enabled = [_s(m) for m in (ALL_SAMPLED if esm is None else esm)]   # an explicit empty set disables sampling
    mask = 0
    for m in enabled:
        mask |= K.METRIC_BITS.get(m, 0)

    servers = nodes["servers"]
    server_ids = [s["id"] for s in servers]
    sidx = {sid: i for i, sid in enumerate(server_ids)}
    client_id = nodes["client"]["id"]
    lb = nodes.get("load_balancer")
    lb_id = lb["id"] if lb else None
    gen_id = gen["id"]

    edges = topo["edges"]
    edge_ids = [e["id"] for e in edges]
    eidx = {eid: i for i, eid in enumerate(edge_ids)}

    def out_edge_of(node_id: str) -> int:
        for i, e in enumerate(edges):
            if e["source"] == node_id:
                return i
        msg = f"node {node_id!r} has no outgoing edge"
        raise ValueError(msg)

    c_edges = (K.AfEdge * len(edges))()
    for i, e in enumerate(edges):
        dist, mean, sigma = _rv(e["latency"])
        tgt = e["target"]
        if tgt == client_id:
            kind, tix = K.TARGET_CLIENT, 0
        elif lb_id is not None and tgt == lb_id:
            kind, tix = K.TARGET_LB, 0
        elif tgt in sidx:
            kind, tix = K.TARGET_SERVER, sidx[tgt]
        else:
            msg = f"Unknown runtime for {tgt!r}"       # simulation_runner.py:229-230
            raise TypeError(msg)
        dr = e.get("dropout_rate")
        c_edges[i] = K.AfEdge(mean, sigma, 0.01 if dr is None else float(dr), K.DIST[dist], kind, tix, 0)

    c_servers = (K.AfServer * len(servers))()
    eps: list[K.AfEndpoint] = []
    steps: list[K.AfStep] = []
    ep_names: list[str] = []
    step_index: dict[tuple[str, int, int], int] = {}
    endpoint_index: dict[tuple[str, int], int] = {}
    for i, s in enumerate(servers):
        res = s.get("server_resources") or {}
        ep_begin = len(eps)
        for j, ep in enumerate(s["endpoints"]):
            sb = len(steps)
            total_ram = 0
            for k, st in enumerate(ep["steps"]):
                kind = _s(st["kind"])
                (op, val), = st["step_operation"].items()
                if kind in RAM_KINDS:
                    total_ram += int(val)
                    continue
                if kind in CPU_KINDS:
                    code = K.STEP_CPU
                elif kind in IO_KINDS:
                    code = K.STEP_IO
                else:
                    msg = f"unknown step kind {kind!r}"
                    raise ValueError(msg)
                step_index[(s["id"], j, k)] = len(steps)
                steps.append(K.AfStep(float(val), code, 0))
            endpoint_index[(s["id"], j)] = len(eps)
            eps.append(K.AfEndpoint(sb, len(steps) - sb, total_ram, 0))
            ep_names.append(f'{s["id"]}:{str(ep["endpoint_name"]).lower()}')
        c_servers[i] = K.AfServer(int(res.get("cpu_cores") or 1), int(res.get("ram_mb") or 1024),
                                  out_edge_of(s["id"]), ep_begin, len(eps) - ep_begin, 0)
    c_eps = (K.AfEndpoint * max(1, len(eps)))(*eps)
    c_steps = (K.AfStep * max(1, len(steps)))(*steps)

    lb_edges = [i for i, e in enumerate(edges) if lb_id is not None and e["source"] == lb_id]
    c_lb = (C.c_int32 * max(1, len(lb_edges)))(*lb_edges)
    lb_algo = K.LB_NONE
    if lb is not None:
        algo = _s(lb.get("algorithms") or "round_robin")
        lb_algo = K.LB_ROUND_ROBIN if algo == "round_robin" else K.LB_LEAST_CONNECTIONS

    # ---- event injection (runtime/events/injection.py:112-164) ---------------
    e_tl: list[tuple[float, str, str, str]] = []
    s_tl: list[tuple[float, str, str, str]] = []
    spike_of: dict[tuple[str, str], float] = {}
    for ev in events:
        st, en = ev["start"], ev["end"]
        a = (float(st["t_start"]), ev["event_id"], ev["target_id"], "start")
        b = (float(en["t_end"]), ev["event_id"], ev["target_id"], "end")
        if ev["target_id"] in eidx:
            spike_of[(ev["event_id"], ev["target_id"])] = float(st["spike_s"])
            e_tl += [a, b]
        elif ev["target_id"] in sidx:
            s_tl += [a, b]
    key = lambda m: (m[0], m[3] == "start", m[1], m[2])  # noqa: E731
    e_tl.sort(key=key)
    s_tl.sort(key=key)
    edge_by_server: dict[str, int] = {}
    for i in lb_edges:                                  # injection.py:158-164
        edge_by_server[edges[i]["target"]] = i
    c_spikes = (K.AfSpikeMark * max(1, len(e_tl)))()
    for i, (m, fire) in enumerate(zip(e_tl, _timeline(e_tl))):
        amp = spike_of[(m[1], m[2])]
        c_spikes[i] = K.AfSpikeMark(fire, amp if m[3] == "start" else -amp, eidx[m[2]], 0)
    c_out = (K.AfOutageMark * max(1, len(s_tl)))()
    pool = set(lb_edges)                                # replay of the outage marks over the LB's edge set
    for i, (m, fire) in enumerate(zip(s_tl, _timeline(s_tl))):
        le = edge_by_server.get(m[2], -1)
        c_out[i] = K.AfOutageMark(fire, le, 1 if m[3] == "start" else 0)
        if le >= 0:
            pool.discard(le) if m[3] == "start" else pool.add(le)
            if lb_edges and not pool and fire < horizon:
                # The reference only rejects "all servers down" (schemas/payload.py:145-252); servers chained BEHIND a
                # covered one keep that check quiet while the LB's own dict runs empty, and the first request that
                # then reaches the LB dies in round_robin (routing/lb_algorithms.py:22-36).  Say so up front.
                msg = (f"event injection: at t={fire:g}s every server behind the load balancer is down "
                       f"(mark {m[1]!r} on {m[2]!r}); the reference's load balancer raises on an empty edge set")
                raise ValueError(msg)

    pod = K.AfScenario()
    pod.users_dist = K.DIST[udist]
    pod.window_s = window
    pod.users_mean = umean
    pod.users_sigma = usigma
    pod.rate_per_user = rpm / 60               # float(mean) / TimeDefaults.MIN_TO_SEC
    pod.horizon_s = horizon
    pod.metrics_mask = mask
    pod.sample_period = period
    pod.n_edges, pod.n_servers = len(edges), len(servers)
    pod.n_endpoints, pod.n_steps = len(eps), len(steps)
    pod.n_lb_edges, pod.lb_algo = len(lb_edges), lb_algo
    pod.gen_edge, pod.client_edge = out_edge_of(gen_id), out_edge_of(client_id)
    pod.n_spike_marks, pod.n_outage_marks = len(e_tl), len(s_tl)
    pod.edges = C.cast(c_edges, C.POINTER(K.AfEdge))
    pod.servers = C.cast(c_servers, C.POINTER(K.AfServer))
    pod.endpoints = C.cast(c_eps, C.POINTER(K.AfEndpoint))
    pod.steps = C.cast(c_steps, C.POINTER(K.AfStep))
    pod.lb_edges = C.cast(c_lb, C.POINTER(C.c_int32))
    pod.spike_marks = C.cast(c_spikes, C.POINTER(K.AfSpikeMark))
    pod.outage_marks = C.cast(c_out, C.POINTER(K.AfOutageMark))

    return FlatScenario(
        pod=pod, edge_ids=edge_ids, server_ids=server_ids, client_id=client_id,
        generator_id=gen_id, lb_id=lb_id, endpoint_names=ep_names, step_index=step_index,
        endpoint_index=endpoint_index,
        spike_mark_events=[(m[1], m[3]) for m in e_tl], horizon_s=horizon, sample_period=period,
        enabled_metrics=enabled,
        _keep=[c_edges, c_servers, c_eps, c_steps, c_lb, c_spikes, c_out],
    )


# --------------------------------------------------------------------------- #
# sweeps                                                                      #
# --------------------------------------------------------------------------- #
def balanced_order(cost: Any, deal: int = 1) -> np.ndarray:
    """Launch order for a skewed sweep: ``order[p]`` = the sweep row that runs at position ``p``
    (= gets replica id ``p``).

    Within one launch the engine already hands replicas to its lanes heaviest first, by each
    replica's own predicted work (DESIGN.md §3.3), whatever their ids.  What it cannot do is move
    work between GPU ranks, which run contiguous replica ranges (``distributed.shard_bounds``): a
    sweep sorted by load gives the last rank the heaviest rows.  ``deal`` > 1 deals the rows, sorted
    heaviest first (LPT), round-robin into ``deal`` consecutive blocks, so that the ranges of
    ``deal`` ranks each get the same mix (SURVEY.md 8e).  The permutation changes which replica id,
    and hence which random numbers, each row gets.  Stable: equal costs keep their row order, a
    flat sweep comes back unchanged.
    """
    c = np.asarray(cost, dtype=np.float64).ravel()
    by_cost = np.argsort(-c, kind="stable")
    deal = max(1, int(deal))
    if deal == 1:
        return by_cost.astype(np.int64)
    return np.concatenate([by_cost[b::deal] for b in range(deal)]).astype(np.int64)


class SweepSpec:
    """Per-replica overrides of scenario fields (the Monte-Carlo sweep).

    ``columns`` maps a field selector to an array of one value per replica::

        SweepSpec(flat, n, {("users_mean",): np.linspace(10, 1000, n),
                            ("edge_mean", "client-lb"): rtt})

    Selectors: ``("users_mean",)``, ``("users_sigma",)``, ``("rate_per_user",)``
    (requests per second per user), ``("edge_mean"|"edge_sigma"|"edge_dropout", edge_id)``,
    ``("server_cpu_cores"|"server_ram_mb", server_id)``,
    ``("step_duration", server_id, endpoint_idx, step_idx)``,
    ``("endpoint_ram", server_id, endpoint_idx)``, ``("spike_delta", event_id)``.
    """

    def __init__(self, flat: FlatScenario, n_replicas: int, columns: dict[tuple, Any]) -> None:
        self.n_replicas = int(n_replicas)
        self.selectors: list[tuple[tuple, np.ndarray]] = []
        cols: list[tuple[int, int]] = []
        vals: list[np.ndarray] = []
        for sel, v in columns.items():
            sel = tuple(sel) if not isinstance(sel, str) else (sel,)
            name = sel[0]
            arr = np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (self.n_replicas,)))
            if name in ("users_mean", "users_sigma", "rate_per_user"):
                targets = [0]
            elif name.startswith("edge_"):
                targets = [flat.edge_ids.index(sel[1])]
            elif name.startswith("server_"):
                targets = [flat.server_ids.index(sel[1])]
            elif name == "step_duration":
                targets = [flat.step_index[(sel[1], int(sel[2]), int(sel[3]))]]
            elif name == "endpoint_ram":
                targets = [flat.endpoint_index[(sel[1], int(sel[2]))]]
            elif name == "spike_delta":
                targets = [i for i, (eid, _) in enumerate(flat.spike_mark_events) if eid == sel[1]]
                if not targets:
                    msg = f"no spike event {sel[1]!r}"
                    raise KeyError(msg)
            else:
                msg = f"unknown sweep field {name!r}"
                raise KeyError(msg)
            self.selectors.append((sel, arr))
            for t in targets:
                cols.append((K.FIELDS[name], t))
                vals.append(arr)
        self.n_columns = len(cols)
        self.values = (np.ascontiguousarray(np.stack(vals, axis=1)) if vals
                       else np.zeros((self.n_replicas, 0)))
        self._cols = (K.AfSweepColumn * max(1, len(cols)))(*[K.AfSweepColumn(f, i) for f, i in cols])
        self.columns = cols

    def estimated_cost(self, flat: FlatScenario) -> np.ndarray:
        """Expected arrivals per row (users x rate x horizon): the load proxy ``balanced_order`` sorts by."""
        users = np.full(self.n_replicas, float(flat.pod.users_mean))
        rate = np.full(self.n_replicas, float(flat.pod.rate_per_user))
        for sel, arr in self.selectors:
            if sel[0] == "users_mean":
                users = arr
            elif sel[0] == "rate_per_user":
                rate = arr
        return np.maximum(users, 0.0) * np.maximum(rate, 0.0) * float(flat.horizon_s)

    def permuted(self, flat: FlatScenario, order: np.ndarray) -> "SweepSpec":
        """The same sweep with row ``order[p]`` at position ``p``."""
        order = np.asarray(order, dtype=np.int64)
        return SweepSpec(flat, self.n_replicas, {sel: arr[order] for sel, arr in self.selectors})

    def payload_for(self, payload: Any, replica: int) -> dict:
        """The scenario of ONE replica of the sweep as a plain YAML-shaped dict.

        Feeding the result to the reference's ``SimulationRunner`` (or to a one-replica
        ``GpuSimulationRunner``) simulates exactly what row ``replica`` of the sweep simulates;
        it is how a sweep point is handed back to the reference for inspection, and how the parity
        tests build the oracle's input.  ``payload`` is the base scenario the sweep was made from.
        """
        import copy  # noqa: PLC0415

        p = copy.deepcopy(_as_dict(payload))
        topo = p["topology_graph"]
        edges = {e["id"]: e for e in topo["edges"]}
        servers = {s["id"]: s for s in topo["nodes"]["servers"]}
        # endpoint_ram rewrites the step list, so it goes last (step selectors use original indices)
        for sel, arr in sorted(self.selectors, key=lambda sa: sa[0][0] == "endpoint_ram"):
            name, v = sel[0], float(arr[replica])
            if name == "users_mean":
                p["rqs_input"]["avg_active_users"]["mean"] = v
            elif name == "users_sigma":
                p["rqs_input"]["avg_active_users"]["variance"] = v
            elif name == "rate_per_user":
                p["rqs_input"]["avg_request_per_minute_per_user"]["mean"] = v * 60.0
            elif name == "edge_mean":
                edges[sel[1]]["latency"]["mean"] = v
            elif name == "edge_sigma":
                edges[sel[1]]["latency"]["variance"] = v
            elif name == "edge_dropout":
                edges[sel[1]]["dropout_rate"] = v
            elif name == "server_cpu_cores":
                servers[sel[1]].setdefault("server_resources", {})["cpu_cores"] = int(v)
            elif name == "server_ram_mb":
                servers[sel[1]].setdefault("server_resources", {})["ram_mb"] = int(v)
            elif name == "step_duration":
                op = servers[sel[1]]["endpoints"][int(sel[2])]["steps"][int(sel[3])]["step_operation"]
                (k, _), = op.items()
                op[k] = v
            elif name == "endpoint_ram":
                ep = servers[sel[1]]["endpoints"][int(sel[2])]
                rest = [st for st in ep["steps"] if _s(st["kind"]) not in RAM_KINDS]
                if int(v) > 0:      # total RAM is reserved up front, so one RAM step says it all
                    rest.append({"kind": "ram", "step_operation": {"necessary_ram": int(v)}})
                ep["steps"] = rest
            elif name == "spike_delta":
                for ev in p.get("events") or []:
                    if ev["event_id"] == sel[1]:
                        ev["start"]["spike_s"] = v
        return p

    def pin(self) -> None:
        """Move the value table into page-locked host memory (needs torch + a CUDA device)."""
        try:
            import torch  # noqa: PLC0415  (plumbing only)
        except ImportError:
            return
        if not torch.cuda.is_available() or self.values.size == 0:
            return
        t = torch.empty(self.values.shape, dtype=torch.float64, pin_memory=True)
        arr = t.numpy()
        arr[...] = self.values
        self.values = arr
        self._pin_keep = t

    def pod(self, first: int = 0, count: int | None = None) -> tuple[K.AfSweep, np.ndarray]:
        """AfSweep over rows ``[first, first+count)``; keep the returned array alive."""
        count = self.n_replicas - first if count is None else count
        rows = np.ascontiguousarray(self.values[first:first + count])
        sw = K.AfSweep()
        sw.n_columns = self.n_columns
        sw.n_rows = count
        sw.columns = C.cast(self._cols, C.POINTER(K.AfSweepColumn))
        sw.values = rows.ctypes.data_as(C.POINTER(C.c_double))
        return sw, rows
