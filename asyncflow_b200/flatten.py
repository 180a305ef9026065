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
  (``runtime/events/injection.py:142-151,185-188``) -- :func:`build_timelines`, which
  also builds the per-row timelines of a sweep over event times.
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


#: numpy mirrors of AfSpikeMark / AfOutageMark: one row of mark tables per sweep row (af_timeline_upload)
SPIKE_MARK_DTYPE = np.dtype([("fire_time", "<f8"), ("delta", "<f8"), ("edge", "<i4"), ("reserved", "<i4")])
OUTAGE_MARK_DTYPE = np.dtype([("fire_time", "<f8"), ("lb_edge", "<i4"), ("down", "<i4")])
assert SPIKE_MARK_DTYPE.itemsize == C.sizeof(K.AfSpikeMark) and OUTAGE_MARK_DTYPE.itemsize == C.sizeof(K.AfOutageMark)


#: ``lb_algorithm`` sweep values: ``K.LB_*`` code -> the reference's name (routing/lb_algorithms.py)
LB_ALGORITHMS = {K.LB_ROUND_ROBIN: "round_robin", K.LB_LEAST_CONNECTIONS: "least_connection"}


def _lb_position(flat: "FlatScenario", server_id: str) -> int:
    """Position in ``flat.lb_edges`` of the load balancer's edge to ``server_id`` (``KeyError`` when it covers none)."""
    for k, e in enumerate(flat.lb_edges):
        if flat.server_ids[flat.pod.edges[e].target_index] == server_id:
            return k
    msg = f"sweep column ('lb_covered', {server_id!r}): the scenario's load balancer does not cover that server"
    raise KeyError(msg)


def _limit(x: Any) -> float:
    """An admission limit as a float, NaN unless it is an integer in [0, 2**31) (bools refused)."""
    if isinstance(x, (bool, np.bool_)):
        return np.nan
    try:
        v = float(x)
    except (TypeError, ValueError):
        return np.nan
    return v if v == v and 0.0 <= v < 2.0 ** 31 and v == int(v) else np.nan


def set_admission(flat: "FlatScenario", admission: dict[str, int] | None) -> None:
    """The scenario's admission limits (DESIGN.md §3.12): ``admission[server_id]`` requests in service at once, 0 = no
    limit; servers left out keep theirs.  ``KeyError`` for an unknown server, ``ValueError`` for a limit that is not an
    integer in [0, 2**31)."""
    for sid, v in (admission or {}).items():
        if sid not in flat.server_ids:
            msg = f"admission: no server {sid!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        lim = _limit(v)
        if lim != lim:
            msg = f"admission: server {sid!r}: limit {v!r} is not an integer in [0, 2**31)"
            raise ValueError(msg)
        flat.pod.servers[flat.server_ids.index(sid)].max_in_service = int(lim)


def _seconds(x: Any) -> float:
    """A deadline or a timeout as a float, NaN unless it is a finite number of seconds >= 0 (bools refused)."""
    if isinstance(x, (bool, np.bool_)):
        return np.nan
    try:
        v = float(x)
    except (TypeError, ValueError):
        return np.nan
    return v if np.isfinite(v) and v >= 0.0 else np.nan


def set_deadlines(flat: "FlatScenario", deadlines: dict[str, float] | None, *, client_timeout: float | None = None) -> None:
    """The scenario's request deadlines and client timeout (DESIGN.md §3.13), in seconds, 0 = none:
    ``deadlines[server_id]`` (servers left out keep theirs) and ``client_timeout`` (``None``: kept).  ``KeyError`` for
    an unknown server, ``ValueError`` for a value that is not a finite number >= 0."""
    for sid, v in (deadlines or {}).items():
        if sid not in flat.server_ids:
            msg = f"deadlines: no server {sid!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        d = _seconds(v)
        if d != d:
            msg = f"deadlines: server {sid!r}: deadline {v!r} is not a finite number of seconds >= 0"
            raise ValueError(msg)
        flat.pod.servers[flat.server_ids.index(sid)].deadline = d
    if client_timeout is not None:
        t = _seconds(client_timeout)
        if t != t:
            msg = f"client_timeout {client_timeout!r} is not a finite number of seconds >= 0"
            raise ValueError(msg)
        flat.pod.client_timeout = t


def _rate(x: Any) -> float:
    """A rate limit in requests per second as a float, NaN unless it is finite and >= 0 (bools refused)."""
    return _seconds(x)


def _burst(x: Any, lo: int = 1) -> float:
    """A burst as a float, NaN unless it is an integer in [lo, 2**31) (bools refused)."""
    v = _limit(x)
    return v if v >= lo else np.nan


def set_rate_limits(flat: "FlatScenario", limits: dict[str, tuple[float, int]] | None, *,
                    lb: tuple[float, int] | None = None) -> None:
    """The scenario's rate limits (DESIGN.md §3.14): ``limits[server_id] = (rate, burst)`` (servers left out keep
    theirs) and the load balancer's ``lb = (rate, burst)`` (``None``: kept), a rate in requests per second (0 = none)
    and a burst, an integer >= 0 (0 reads as 1).  ``KeyError`` for an unknown server, ``ValueError`` for a bad value or
    an LB limit on a scenario without a load balancer."""
    def pair(what: str, v: Any) -> tuple[float, int]:
        try:
            r, b = v
        except (TypeError, ValueError):
            msg = f"{what}: {v!r} is not a (rate, burst) pair"
            raise ValueError(msg) from None
        rr, bb = _rate(r), _burst(b, lo=0)
        if rr != rr:
            msg = f"{what}: rate {r!r} is not a finite number of requests per second >= 0"
            raise ValueError(msg)
        if bb != bb:
            msg = f"{what}: burst {b!r} is not an integer in [0, 2**31)"
            raise ValueError(msg)
        return rr, int(bb)
    for sid, v in (limits or {}).items():
        if sid not in flat.server_ids:
            msg = f"rate limits: no server {sid!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        srv = flat.pod.servers[flat.server_ids.index(sid)]
        srv.rate_limit, srv.burst = pair(f"rate limits: server {sid!r}", v)
    if lb is not None:
        if flat.lb_id is None:
            msg = "rate limits: the scenario has no load balancer to limit"
            raise ValueError(msg)
        flat.pod.lb_rate_limit, flat.pod.lb_burst = pair("rate limits: load balancer", lb)


def _rv(d: dict) -> tuple[str, float, float]:
    dist = _s(d.get("distribution") or "poisson")
    var = d.get("variance")
    if var is None and dist in ("normal", "log_normal"):
        var = d["mean"]          # RVConfig.default_variance (schemas/common/random_variables.py)
    return dist, float(d["mean"]), 0.0 if var is None else float(var)


@dataclass(frozen=True)
class FlatEvent:
    """One injected event, as :func:`build_timelines` needs it."""

    event_id: str
    target_id: str
    spike: bool          # a network spike on an edge; else a server outage
    target: int          # spike: the edge; outage: the load balancer's edge to the server, -1 when it covers none
    server: int          # outage: the server; spike: -1
    t_start: float
    t_end: float
    spike_s: float       # the spike's amplitude (0 for an outage)


@dataclass
class Timelines:
    """Spike and outage mark tables of R rows (the layout of ``AfTimeline``), and which mark each entry is:
    ``*_mark[r, j]`` = 2 k for the start of the k-th event of its kind (in payload order), 2 k + 1 for its end."""

    spikes: np.ndarray          # [R, n_spike_marks] SPIKE_MARK_DTYPE
    outages: np.ndarray         # [R, n_outage_marks] OUTAGE_MARK_DTYPE
    spike_mark: np.ndarray      # [R, n_spike_marks] int64
    outage_mark: np.ndarray     # [R, n_outage_marks] int64


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
    events: list[FlatEvent]                            # the spikes and outages, in payload order
    lb_edges: list[int]
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


def _sorted_fold(events: list[FlatEvent], t_start: np.ndarray, t_end: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The marks of ``events`` (one kind) in every row, sorted with the reference's key ``(t, mark == start, event_id,
    target_id)`` (a stable sort: equal keys keep payload order), and their FIRE times: injection.py:178-188 in f64,
    ``dt = t - last_t; now += dt`` only when ``dt > 0``.  ``t_start`` / ``t_end``: [R, len(events)].
    Returns (mark [R, 2k] as in :class:`Timelines`, fire [R, 2k])."""
    R, k = t_start.shape[0], len(events)
    t = np.empty((R, 2 * k))
    t[:, 0::2], t[:, 1::2] = t_start, t_end
    ids = [(e.event_id, e.target_id) for e in events]
    rank = {key: i for i, key in enumerate(sorted(set(ids)))}
    ev_rank = np.broadcast_to(np.repeat([rank[key] for key in ids], 2), t.shape)
    is_start = np.broadcast_to(np.tile([True, False], k), t.shape)
    mark = np.lexsort((ev_rank, is_start, t), axis=1) if k else np.zeros((R, 0), dtype=np.int64)
    ts = np.take_along_axis(t, mark, axis=1)
    fire = np.empty_like(ts)
    now, last = np.zeros(R), np.zeros(R)
    for j in range(2 * k):
        dt = ts[:, j] - last
        now = np.where(dt > 0.0, now + dt, now)
        last = ts[:, j]
        fire[:, j] = now
    return mark.astype(np.int64), fire


def build_timelines(events: list[FlatEvent], lb_edges: list[int], horizon: float, t_start: np.ndarray,
                    t_end: np.ndarray, spike_s: np.ndarray, label=lambda r: "", covered: np.ndarray | None = None) -> Timelines:
    """The spike and outage mark tables of R rows of event times (``t_start`` / ``t_end`` / ``spike_s``: [R, n_events],
    columns in the order of ``events``): what ``flatten`` uploads for one row and ``SweepSpec`` for each of its rows.
    ``covered`` ([R, len(lb_edges)] bool, default all): which LB edges each row keeps; an outage mark of a server whose
    edge a row leaves out gets ``lb_edge = -1`` there (the reference's no-op for a server not behind the LB), its fire
    time unchanged.  Refuses (``ValueError``, prefixed by ``label(row)``) a row whose load balancer runs out of servers
    before the horizon."""
    sp = [i for i, e in enumerate(events) if e.spike]
    out = [i for i, e in enumerate(events) if not e.spike]
    R = t_start.shape[0]
    s_mark, s_fire = _sorted_fold([events[i] for i in sp], t_start[:, sp], t_end[:, sp])
    spikes = np.zeros(s_mark.shape, dtype=SPIKE_MARK_DTYPE)
    if sp:
        ev = np.asarray(sp)[s_mark // 2]
        amp = np.take_along_axis(spike_s, ev, axis=1)
        spikes["fire_time"] = s_fire
        spikes["delta"] = np.where(s_mark % 2 == 0, amp, -amp)
        spikes["edge"] = np.asarray([e.target for e in events])[ev]
    o_mark, o_fire = _sorted_fold([events[i] for i in out], t_start[:, out], t_end[:, out])
    outages = np.zeros(o_mark.shape, dtype=OUTAGE_MARK_DTYPE)
    if out:
        ev = np.asarray(out)[o_mark // 2]
        outages["fire_time"] = o_fire
        outages["lb_edge"] = np.asarray([e.target for e in events])[ev]
        outages["down"] = o_mark % 2 == 0
    if lb_edges and out:                                # replay of the outage marks over the LB's edge set
        pos = np.zeros(max(lb_edges) + 1, dtype=np.int64)      # LB edge -> its column of `up`
        pos[lb_edges] = np.arange(len(lb_edges))
        up = np.ones((R, len(lb_edges)), dtype=bool) if covered is None else np.array(covered, dtype=bool)
        rows = np.arange(R)
        if covered is not None:
            for j in range(o_mark.shape[1]):
                le = outages["lb_edge"][:, j]
                hit = le >= 0
                cut = np.zeros(R, dtype=bool)
                cut[hit] = ~up[rows[hit], pos[le[hit]]]
                outages["lb_edge"][cut, j] = -1
        for j in range(o_mark.shape[1]):
            le, down = outages["lb_edge"][:, j], outages["down"][:, j] != 0
            hit = le >= 0
            up[rows[hit], pos[le[hit]]] = ~down[hit]
            bad = np.flatnonzero(hit & ~up.any(axis=1) & (o_fire[:, j] < horizon))
            if bad.size:
                # The reference only rejects "all servers down" (schemas/payload.py:145-252); servers chained BEHIND a
                # covered one keep that check quiet while the LB's own dict runs empty, and the first request that
                # then reaches the LB dies in round_robin (routing/lb_algorithms.py:22-36).  Say so up front.
                r = int(bad[0])
                e = events[out[int(o_mark[r, j]) // 2]]
                msg = (f"{label(r)}event injection: at t={o_fire[r, j]:g}s every server behind the load balancer is down "
                       f"(mark {e.event_id!r} on {e.target_id!r}); the reference's load balancer raises on an empty edge set")
                raise ValueError(msg)
    return Timelines(spikes, outages, s_mark, o_mark)


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
    edge_by_server: dict[str, int] = {}
    for i in lb_edges:                                  # injection.py:158-164
        edge_by_server[edges[i]["target"]] = i
    flat_events: list[FlatEvent] = []
    for ev in events:
        st, en = ev["start"], ev["end"]
        tgt = ev["target_id"]
        if tgt in eidx:
            flat_events.append(FlatEvent(ev["event_id"], tgt, True, eidx[tgt], -1, float(st["t_start"]),
                                         float(en["t_end"]), float(st["spike_s"])))
        elif tgt in sidx:
            flat_events.append(FlatEvent(ev["event_id"], tgt, False, edge_by_server.get(tgt, -1), sidx[tgt],
                                         float(st["t_start"]), float(en["t_end"]), 0.0))
    tl = build_timelines(flat_events, lb_edges, horizon, np.array([[e.t_start for e in flat_events]]),
                         np.array([[e.t_end for e in flat_events]]), np.array([[e.spike_s for e in flat_events]]))
    c_spikes = (K.AfSpikeMark * max(1, tl.spikes.shape[1]))()
    C.memmove(c_spikes, tl.spikes.tobytes(), tl.spikes.nbytes)
    c_out = (K.AfOutageMark * max(1, tl.outages.shape[1]))()
    C.memmove(c_out, tl.outages.tobytes(), tl.outages.nbytes)
    spike_events = [e for e in flat_events if e.spike]
    spike_mark_events = [(spike_events[m // 2].event_id, "start" if m % 2 == 0 else "end") for m in tl.spike_mark[0]]

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
    pod.n_spike_marks, pod.n_outage_marks = tl.spikes.shape[1], tl.outages.shape[1]
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
        spike_mark_events=spike_mark_events, events=flat_events, lb_edges=lb_edges, horizon_s=horizon,
        sample_period=period,
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
    ``("endpoint_ram", server_id, endpoint_idx)``, ``("spike_delta", event_id)``,
    ``("event_start"|"event_end", event_id)`` (the ``t_start`` / ``t_end`` of a spike or an outage),
    ``("lb_covered", server_id)`` (1: behind the load balancer as in the scenario, 0: not; bools accepted) and
    ``("lb_algorithm",)`` (``"round_robin"`` or ``"least_connection"``, enum members or ``K.LB_*`` codes accepted) and
    ``("server_max_in_service", server_id)`` (the server's admission limit, an integer >= 0, 0 = none; DESIGN.md §3.12),
    ``("server_deadline", server_id)`` and ``("client_timeout",)`` (seconds >= 0, 0 = none; DESIGN.md §3.13),
    ``("server_rate"|"server_burst", server_id)`` and ``("lb_rate",)`` / ``("lb_burst",)`` (a rate limit in requests per
    second, finite and >= 0, 0 = none, and its burst, an integer in [1, 2**31); DESIGN.md §3.14).

    A row that uncovers a server simulates the scenario without the load balancer's edge to it (:meth:`payload_for`):
    its round-robin order is the scenario's with that edge left out, and an outage of that server is a no-op.  The
    scenario's load balancer covers the largest fleet: only servers it covers can be swept.  A row that covers no
    server, uncovers a server whose LB edge a spike targets, or whose covered servers are all down at once is refused
    with a ``ValueError`` naming the row.

    A spec that sweeps an event time gives every row its own spike and outage timelines (:attr:`timelines`, uploaded
    with the sweep): the marks sorted and their fire times folded as ``flatten`` does for the scenario, a row's
    ``spike_delta`` folded into its marks' amplitudes.  Each row must pass the reference's payload rules --
    ``0 <= t_start < t_end <= horizon``, no two outages of one server overlapping, not every server down at once --
    and keep a server behind the load balancer up until the horizon; a row that does not is refused with a
    ``ValueError`` naming the row, the event and the rule.
    """

    def __init__(self, flat: FlatScenario, n_replicas: int, columns: dict[tuple, Any]) -> None:
        self.n_replicas = int(n_replicas)
        self.selectors: list[tuple[tuple, np.ndarray]] = []
        self.timelines: Timelines | None = None
        cols: list[tuple[int, int]] = []
        vals: list[np.ndarray] = []
        keys = [tuple(sel) if not isinstance(sel, str) else (sel,) for sel in columns]
        arrays = [self._lb_values(flat, sel, v) if sel[0] in ("lb_covered", "lb_algorithm")
                  else self._limits(flat, sel, v) if sel[0] in K.ADMISSION_FIELDS
                  else self._seconds(flat, sel, v) if sel[0] in K.DEADLINE_FIELDS
                  else self._rates(flat, sel, v) if sel[0] in K.RATE_FIELDS
                  else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (self.n_replicas,)))
                  for sel, v in zip(keys, columns.values())]
        self.covered = self._covered(flat, keys, arrays)
        # the scenario's rate limits (set_rate_limits), which a row's rate or burst column overrides
        self._rl_base = ({sid: (float(flat.pod.servers[i].rate_limit), int(flat.pod.servers[i].burst))
                          for i, sid in enumerate(flat.server_ids)},
                         (float(flat.pod.lb_rate_limit), int(flat.pod.lb_burst)) if flat.lb_id is not None else None)
        # rows need their own timelines when event times are swept or when a row drops a server that has outage marks
        times = any(k[0] in ("event_start", "event_end") for k in keys) or (
            self.covered is not None and any((~self.covered[:, flat.lb_edges.index(e.target)]).any()
                                             for e in flat.events if not e.spike and e.target >= 0))
        event_of = {e.event_id: i for i, e in enumerate(flat.events)}
        for sel, arr in zip(keys, arrays):
            name = sel[0]
            if name in ("event_start", "event_end") or (times and name == "spike_delta"):
                if sel[1] not in event_of or (name == "spike_delta" and not flat.events[event_of[sel[1]]].spike):
                    msg = f"no {'spike ' if name == 'spike_delta' else ''}event {sel[1]!r}"
                    raise KeyError(msg)
                self.selectors.append((sel, arr))       # carried by the rows' timelines, not by a column
                continue
            if name in ("users_mean", "users_sigma", "rate_per_user", "client_timeout", "lb_rate", "lb_burst"):
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
            elif name == "lb_covered":
                targets = [_lb_position(flat, sel[1])]
            elif name == "lb_algorithm":
                targets = [0]
            else:
                msg = f"unknown sweep field {name!r}"
                raise KeyError(msg)
            self.selectors.append((sel, arr))
            for t in targets:
                cols.append(({**K.FIELDS, **K.LB_FIELDS, **K.ADMISSION_FIELDS, **K.DEADLINE_FIELDS, **K.RATE_FIELDS}[name], t))
                vals.append(arr)
        self.n_columns = len(cols)
        self.values = (np.ascontiguousarray(np.stack(vals, axis=1)) if vals
                       else np.zeros((self.n_replicas, 0)))
        self._cols = (K.AfSweepColumn * max(1, len(cols)))(*[K.AfSweepColumn(f, i) for f, i in cols])
        self.columns = cols
        if times:
            self.timelines = self._timelines(flat)
        elif self.covered is not None and any(not e.spike for e in flat.events):
            self._timelines(flat)               # the fleet-down check alone: every row runs the scenario's marks

    def _lb_values(self, flat: FlatScenario, sel: tuple, v: Any) -> np.ndarray:
        """A load-balancer column as float codes: 0 / 1 for ``lb_covered``, ``K.LB_*`` for ``lb_algorithm``."""
        if flat.lb_id is None:
            msg = f"sweep column {sel!r}: the scenario has no load balancer to sweep"
            raise ValueError(msg)
        raw = np.broadcast_to(np.asarray(v, dtype=object), (self.n_replicas,))
        if sel[0] == "lb_algorithm":
            code = {name: float(c) for c, name in LB_ALGORITHMS.items()}

            def one(x: Any) -> float:
                if isinstance(x, (int, float, np.integer, np.floating)) and not isinstance(x, (bool, np.bool_)):
                    return float(x) if x in LB_ALGORITHMS else np.nan
                return code.get(_s(x), np.nan)
            out = np.array([one(x) for x in raw], dtype=np.float64)
            bad = np.isnan(out)
            if bad.any():
                r = int(np.flatnonzero(bad)[0])
                msg = (f"sweep row {r}: {sel!r} = {raw[r]!r}: the algorithm is 'round_robin' or 'least_connection' "
                       "(or K.LB_ROUND_ROBIN / K.LB_LEAST_CONNECTIONS)")
                raise ValueError(msg)
            return out
        try:
            out = np.asarray(raw.astype(np.float64))
        except (TypeError, ValueError):
            out = np.full(self.n_replicas, np.nan)
        bad = ~((out == 0.0) | (out == 1.0))
        if bad.any():
            r = int(np.flatnonzero(bad)[0])
            msg = f"sweep row {r}: {sel!r} = {raw[r]!r}: a server is covered (1) or not (0)"
            raise ValueError(msg)
        return np.ascontiguousarray(out)

    def _limits(self, flat: FlatScenario, sel: tuple, v: Any) -> np.ndarray:
        """An admission-limit column: integers in [0, 2**31) as floats (``KeyError`` / ``ValueError`` naming the row)."""
        if len(sel) != 2 or sel[1] not in flat.server_ids:
            msg = f"sweep column {sel!r}: no server {sel[1] if len(sel) > 1 else None!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        raw = np.broadcast_to(np.asarray(v, dtype=object), (self.n_replicas,))
        out = np.array([_limit(x) for x in raw], dtype=np.float64)
        bad = np.isnan(out)
        if bad.any():
            r = int(np.flatnonzero(bad)[0])
            msg = f"sweep row {r}: {sel!r} = {raw[r]!r}: an admission limit is an integer in [0, 2**31) (0: none)"
            raise ValueError(msg)
        return out

    def _seconds(self, flat: FlatScenario, sel: tuple, v: Any) -> np.ndarray:
        """A deadline or client-timeout column: finite seconds >= 0 (``KeyError`` / ``ValueError`` naming the row)."""
        if sel[0] == "server_deadline" and (len(sel) != 2 or sel[1] not in flat.server_ids):
            msg = f"sweep column {sel!r}: no server {sel[1] if len(sel) > 1 else None!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        if sel[0] == "client_timeout" and len(sel) != 1:
            msg = f"sweep column {sel!r}: the client timeout takes no index (('client_timeout',))"
            raise KeyError(msg)
        raw = np.broadcast_to(np.asarray(v, dtype=object), (self.n_replicas,))
        out = np.array([_seconds(x) for x in raw], dtype=np.float64)
        bad = np.isnan(out)
        if bad.any():
            r = int(np.flatnonzero(bad)[0])
            msg = f"sweep row {r}: {sel!r} = {raw[r]!r}: a deadline or timeout is a finite number of seconds >= 0 (0: none)"
            raise ValueError(msg)
        return out

    def _rates(self, flat: FlatScenario, sel: tuple, v: Any) -> np.ndarray:
        """A rate-limit column: a rate finite and >= 0, or a burst, an integer in [1, 2**31) (``KeyError`` /
        ``ValueError`` naming the row)."""
        if sel[0] in ("server_rate", "server_burst") and (len(sel) != 2 or sel[1] not in flat.server_ids):
            msg = f"sweep column {sel!r}: no server {sel[1] if len(sel) > 1 else None!r} (servers: {list(flat.server_ids)})"
            raise KeyError(msg)
        if sel[0] in ("lb_rate", "lb_burst"):
            if flat.lb_id is None:
                msg = f"sweep column {sel!r}: the scenario has no load balancer to limit"
                raise ValueError(msg)
            if len(sel) != 1:
                msg = f"sweep column {sel!r}: the load balancer's limit takes no index (({sel[0]!r},))"
                raise KeyError(msg)
        raw = np.broadcast_to(np.asarray(v, dtype=object), (self.n_replicas,))
        rate = sel[0].endswith("_rate")
        out = np.array([_rate(x) if rate else _burst(x) for x in raw], dtype=np.float64)
        bad = np.isnan(out)
        if bad.any():
            r = int(np.flatnonzero(bad)[0])
            what = ("a rate limit is a finite number of requests per second >= 0 (0: none)" if rate
                    else "a burst is an integer in [1, 2**31)")
            msg = f"sweep row {r}: {sel!r} = {raw[r]!r}: {what}"
            raise ValueError(msg)
        return out

    def rate_limits_for(self, replica: int) -> tuple[dict[str, tuple[float, int]], tuple[float, int] | None]:
        """Row ``replica``'s rate limits: ``{server_id: (rate, burst)}`` for every server with a scenario limit or a
        column, and the load balancer's ``(rate, burst)`` (``None`` without either), from the scenario's limits and this
        spec's columns (zeros included; a burst of 0 reads as 1)."""
        base, lb_base = self._rl_base
        srv = {sid: list(rb) for sid, rb in base.items() if rb[0] > 0.0}
        lb = list(lb_base) if lb_base is not None and lb_base[0] > 0.0 else None
        for sel, arr in self.selectors:
            if sel[0] not in K.RATE_FIELDS:
                continue
            k = 0 if sel[0].endswith("_rate") else 1
            if sel[0].startswith("server_"):
                srv.setdefault(sel[1], list(base[sel[1]]))[k] = float(arr[replica])
            else:
                if lb is None:
                    lb = list(lb_base)
                lb[k] = float(arr[replica])
        pair = lambda rb: (float(rb[0]), max(1, int(rb[1])))  # noqa: E731
        return {sid: pair(rb) for sid, rb in srv.items()}, (pair(lb) if lb is not None else None)

    def _refuse_rates(self, replica: int, what: str) -> None:
        srv, lb = self.rate_limits_for(replica)
        set_ = {**{sid: rb for sid, rb in srv.items() if rb[0] > 0.0}, **({"load_balancer": lb} if lb and lb[0] > 0.0 else {})}
        if set_:
            msg = (f"sweep row {replica} sets rate limits {set_}, which {what} cannot express; "
                   "payload_and_overload() returns the payload with the rate limits, the deadlines and the limits")
            raise ValueError(msg)

    def deadlines_for(self, replica: int) -> tuple[dict[str, float], float | None]:
        """Row ``replica``'s deadlines ``{server_id: seconds}`` and client timeout (``None`` without such a column) from
        this spec's columns (zeros included)."""
        dl = {sel[1]: float(arr[replica]) for sel, arr in self.selectors if sel[0] == "server_deadline"}
        to = [float(arr[replica]) for sel, arr in self.selectors if sel[0] == "client_timeout"]
        return dl, (to[-1] if to else None)

    def _refuse_deadlines(self, replica: int, what: str) -> None:
        dl, to = self.deadlines_for(replica)
        set_ = {**{sid: v for sid, v in dl.items() if v}, **({"client_timeout": to} if to else {})}
        if set_:
            msg = (f"sweep row {replica} sets deadlines {set_}, which {what} cannot express; "
                   "payload_and_overload() returns the payload with the deadlines, the timeout and the limits")
            raise ValueError(msg)

    def payload_and_overload(self, payload: Any, replica: int) -> tuple[dict, dict]:
        """Row ``replica`` as the oracle takes it: the row's payload (:meth:`payload_for` without the overload columns)
        and ``{"admission": {server_id: limit}, "deadline": {server_id: seconds}, "client_timeout": seconds | None}``
        (0: none; ``None``: the scenario's).  When the sweep has a rate limit (a column, or the scenario's), also
        ``"rate_limit": {server_id: (rate, burst)}`` and ``"lb_rate_limit": (rate, burst) | None``
        (:meth:`rate_limits_for`).  The reference can express none of them."""
        dl, to = self.deadlines_for(replica)
        ov = {"admission": self.admission_for(replica), "deadline": dl, "client_timeout": to}
        if self.has_rate_limits:
            ov["rate_limit"], ov["lb_rate_limit"] = self.rate_limits_for(replica)
        return self._payload(payload, replica), ov

    @property
    def has_rate_limits(self) -> bool:
        """Does the sweep have a rate limit somewhere: a rate-limit column (zeros included) or a scenario rate?"""
        base, lb = self._rl_base
        return (any(sel[0] in K.RATE_FIELDS for sel, _ in self.selectors) or any(r > 0.0 for r, _ in base.values())
                or (lb is not None and lb[0] > 0.0))

    def admission_for(self, replica: int) -> dict[str, int]:
        """Row ``replica``'s admission limits ``{server_id: limit}`` from this spec's columns (zeros included)."""
        return {sel[1]: int(arr[replica]) for sel, arr in self.selectors if sel[0] in K.ADMISSION_FIELDS}

    def payload_and_admission(self, payload: Any, replica: int) -> tuple[dict, dict[str, int]]:
        """Row ``replica`` as the oracle takes it: the row's payload (:meth:`payload_for` without the admission
        columns) and its admission limits, ``{server_id: limit}`` (0: none).  The reference cannot express a limit, so a
        capped row has no payload of its own.  A row with a deadline or a client timeout is refused (``ValueError``):
        use :meth:`payload_and_overload`."""
        self._refuse_deadlines(replica, "payload_and_admission()")
        self._refuse_rates(replica, "payload_and_admission()")
        return self._payload(payload, replica), self.admission_for(replica)

    def _covered(self, flat: FlatScenario, keys: list[tuple], arrays: list[np.ndarray]) -> np.ndarray | None:
        """[R, len(flat.lb_edges)] bool: the LB edges each row keeps (``None`` without ``lb_covered`` columns), checked
        against the rules that need no timeline: a covered server in every row, no uncovered edge a spike targets."""
        sel_arr = [(sel, arr) for sel, arr in zip(keys, arrays) if sel[0] == "lb_covered"]
        if not sel_arr:
            return None
        cov = np.ones((self.n_replicas, len(flat.lb_edges)), dtype=bool)
        for sel, arr in sel_arr:
            cov[:, _lb_position(flat, sel[1])] = arr != 0.0
        none = ~cov.any(axis=1)
        if none.any():
            r = int(np.flatnonzero(none)[0])
            msg = f"sweep row {r}: ('lb_covered', ...): the row covers no server; the load balancer needs one"
            raise ValueError(msg)
        for e in flat.events:
            if e.spike and e.target in flat.lb_edges:
                k = flat.lb_edges.index(e.target)
                if not cov[:, k].all():
                    r = int(np.flatnonzero(~cov[:, k])[0])
                    msg = (f"sweep row {r}: ('lb_covered', {flat.server_ids[flat.pod.edges[e.target].target_index]!r}) = 0: "
                           f"the spike {e.event_id!r} targets the load balancer's edge to that server; a server whose LB "
                           "edge is spiked cannot be uncovered")
                    raise ValueError(msg)
        return cov

    def _timelines(self, flat: FlatScenario) -> Timelines:
        """Every row's event times and amplitudes, checked against the payload rules, then its mark tables."""
        ev = flat.events
        R, E = self.n_replicas, len(ev)
        field = {"event_start": "t_start", "event_end": "t_end", "spike_delta": "spike_s"}
        cols = {f: np.tile(np.array([getattr(e, f) for e in ev], dtype=np.float64), (R, 1)) for f in field.values()}
        index = {e.event_id: i for i, e in enumerate(ev)}
        for sel, arr in self.selectors:
            if sel[0] in field:
                cols[field[sel[0]]][:, index[sel[1]]] = arr
        ts, te, amp = cols["t_start"], cols["t_end"], cols["spike_s"]
        H = float(flat.horizon_s)

        def refuse(bad: np.ndarray, e: int, rule: str) -> None:
            r = int(np.flatnonzero(bad)[0])
            msg = (f"sweep row {r}: event {ev[e].event_id!r} (t_start={float(ts[r, e])!r}, t_end={float(te[r, e])!r}"
                   f"{f', spike_s={float(amp[r, e])!r}' if ev[e].spike else ''}): {rule}")
            raise ValueError(msg)

        for e in range(E):                      # schemas/events/injection.py:88, schemas/payload.py:64-104
            ok = (ts[:, e] >= 0.0) & (ts[:, e] < te[:, e]) & (te[:, e] <= H)
            if not ok.all():
                refuse(~ok, e, f"an event needs 0 <= t_start < t_end <= the horizon ({H:g} s)")
            if ev[e].spike and not (np.isfinite(amp[:, e]) & (amp[:, e] >= 0.0)).all():
                refuse(~(np.isfinite(amp[:, e]) & (amp[:, e] >= 0.0)), e, "a spike's spike_s is finite and >= 0")
        by_server: dict[int, list[int]] = {}
        for e, x in enumerate(ev):
            if not x.spike:
                by_server.setdefault(x.server, []).append(e)
        for evs in by_server.values():           # payload.py:203-252 (back to back is fine: END sorts before START)
            for i, a in enumerate(evs):
                for b in evs[i + 1:]:
                    both = (ts[:, a] < te[:, b]) & (ts[:, b] < te[:, a])
                    if both.any():
                        refuse(both, b, f"overlaps the outage {ev[a].event_id!r} of the same server")
        if len(by_server) == flat.n_servers:     # payload.py:145-200: at some outage's start every server is down
            for e0 in (e for evs in by_server.values() for e in evs):
                t = ts[:, e0]
                down = np.ones(R, dtype=bool)
                for evs in by_server.values():
                    down &= np.any([(ts[:, e] <= t) & (t < te[:, e]) for e in evs], axis=0)
                if down.any():
                    refuse(down, e0, "every server is down once it starts; keep at least one up")
        return build_timelines(ev, flat.lb_edges, H, ts, te, amp, label=lambda r: f"sweep row {r}: ", covered=self.covered)

    def timeline_pod(self, first: int = 0, count: int | None = None) -> tuple[K.AfTimeline | None, Any]:
        """AfTimeline over rows ``[first, first+count)`` (``None`` when the spec sweeps no event time); keep the returned
        arrays alive."""
        if self.timelines is None:
            return None, None
        count = self.n_replicas - first if count is None else count
        sp = np.ascontiguousarray(self.timelines.spikes[first:first + count])
        ou = np.ascontiguousarray(self.timelines.outages[first:first + count])
        tl = K.AfTimeline(count, sp.ctypes.data_as(C.POINTER(K.AfSpikeMark)), ou.ctypes.data_as(C.POINTER(K.AfOutageMark)))
        return tl, (sp, ou)

    @property
    def timeline_row_bytes(self) -> int:
        """Bytes of one row's timelines (0 without)."""
        tl = self.timelines
        return 0 if tl is None else tl.spikes.shape[1] * tl.spikes.itemsize + tl.outages.shape[1] * tl.outages.itemsize

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
        A row with an admission limit, a deadline, a client timeout or a rate limit has no such payload (the reference
        has none of them): ``ValueError``; use :meth:`payload_and_overload`.
        """
        self._refuse_deadlines(replica, "a payload")
        self._refuse_rates(replica, "a payload")
        capped = {sid: v for sid, v in self.admission_for(replica).items() if v}
        if capped:
            msg = (f"sweep row {replica} sets admission limits {capped}, which a payload cannot express; "
                   "payload_and_admission() returns the payload and the limits")
            raise ValueError(msg)
        return self._payload(payload, replica)

    def _payload(self, payload: Any, replica: int) -> dict:
        import copy  # noqa: PLC0415

        p = copy.deepcopy(_as_dict(payload))
        topo = p["topology_graph"]
        edges = {e["id"]: e for e in topo["edges"]}
        servers = {s["id"]: s for s in topo["nodes"]["servers"]}
        uncovered: set[str] = set()
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
            elif name in ("event_start", "event_end"):
                for ev in p.get("events") or []:
                    if ev["event_id"] == sel[1]:
                        if name == "event_start":
                            ev["start"]["t_start"] = v
                        else:
                            ev["end"]["t_end"] = v
            elif name == "lb_covered":
                if v == 0.0:
                    uncovered.add(sel[1])
                else:
                    uncovered.discard(sel[1])
            elif name == "lb_algorithm":
                topo["nodes"]["load_balancer"]["algorithms"] = LB_ALGORITHMS[int(v)]
        if uncovered:           # the reduced payload: the server stays, the LB neither covers it nor has an edge to it
            lb = topo["nodes"]["load_balancer"]
            lb["server_covered"] = [sid for sid in lb.get("server_covered") or [] if sid not in uncovered]
            topo["edges"] = [e for e in topo["edges"] if not (e["source"] == lb["id"] and e["target"] in uncovered)]
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
