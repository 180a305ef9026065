"""The oracle with rate limits (DESIGN.md §3.14) -- TEST INFRASTRUCTURE ONLY.

The reference has no rate limit, so this is the specification of the behaviour the engine adds, written on
``tests/des_deadline.py``'s server (admission limits, deadlines and rate limits compose) and on ``oracle/des_port.py``'s
load balancer, leaving ``des_port.py``, ``des_admission.py`` and ``des_deadline.py`` unchanged.  A site -- a server, or
the load balancer -- with a rate ``r > 0`` requests per second and a burst ``B >= 1`` runs a GCRA token bucket: one f64,
its theoretical arrival time ``tat``, 0.0 at the start.  Where the site's process takes a request from its inbox::

    tau = 1.0 / r
    L = (B - 1) * tau
    if tat - now > L:
        throttled += 1                    # the request is gone
    else:
        tat = max(tat, now) + tau

A server checks in its dispatcher right after it takes the request, before the admission limit: a throttled request is
gone as a shed one is (no hop, no endpoint, no handler; the in-edge counted it as sent).  The load balancer checks after
it takes the request and records its hop, before the pick: a throttled request moves no round-robin order and no
connection count.  Both loop back to ``get()``.  No random number is drawn.

``simulate(payload, ..., admission=, deadline=, client_timeout=, rate_limit={server_id: (r, B)}, lb_rate_limit=(r, B))``
is ``des_deadline.simulate`` plus ``server_throttled`` per server and ``lb_throttled``; ``r = 0`` or a missing server:
no limit, a burst of 0 reads as 1.  Without a rate anywhere every other output is ``des_deadline.simulate``'s.
``checks=[]`` collects ``(site, rid, now, tat, tau, L, passed)`` at every check of a limited site, ``tat`` as it was
before the check."""

from __future__ import annotations

import math

import des_deadline
from des_admission import des_port


def _pair(what: str, v) -> tuple[float, int]:
    try:
        r, b = v
    except (TypeError, ValueError):
        raise ValueError(f"{what}: {v!r} is not a (rate, burst) pair") from None
    if isinstance(r, bool) or not isinstance(r, (int, float)) or not math.isfinite(r) or r < 0:
        raise ValueError(f"{what}: rate {r!r} is not a finite number of requests per second >= 0")
    if isinstance(b, bool) or int(b) != b or not 0 <= b < 2 ** 31:
        raise ValueError(f"{what}: burst {b!r} is not an integer in [0, 2**31)")
    return float(r), max(1, int(b))


class _Bucket:
    """One site's GCRA bucket; ``take(now)``: does the request pass?"""

    def __init__(self, site: str, rate: float, burst: int, checks: list | None) -> None:
        self.site = site
        self.tau = 1.0 / rate
        self.lim = (burst - 1) * self.tau
        self.tat = 0.0
        self.checks = checks

    def take(self, rid: int, now: float) -> bool:
        tat = self.tat
        passed = not (tat - now > self.lim)
        if passed:
            self.tat = max(tat, now) + self.tau
        if self.checks is not None:
            self.checks.append((self.site, rid, now, tat, self.tau, self.lim, passed))
        return passed


def _server_class(base, limits: dict, made: list, checks: list | None):
    class _RateLimitedServer(base):
        def __init__(self, sim, cfg: dict) -> None:
            super().__init__(sim, cfg)
            r, b = limits.get(self.id, (0.0, 1))
            self.bucket = _Bucket(self.id, r, b, checks) if r > 0.0 else None
            self.throttled = 0
            made.append(self)

        def dispatch(self):
            env = self.sim.env
            while True:
                req = yield self.box.get()
                if self.bucket is not None and not self.bucket.take(req.rid, env.now):
                    self.throttled += 1          # before the admission limit: the cap never sees it
                    continue
                if self.limit and self.in_service >= self.limit:
                    self.rejected += 1
                    continue
                self.in_service += 1
                env.process(self.handle(req))

    return _RateLimitedServer


def _lb_class(limit: tuple[float, int] | None, made: list, checks: list | None):
    class _RateLimitedLoadBalancer(des_port._LoadBalancer):
        def __init__(self, sim, cfg: dict) -> None:
            super().__init__(sim, cfg)
            r, b = limit if limit is not None else (0.0, 1)
            self.bucket = _Bucket(self.id, r, b, checks) if r > 0.0 else None
            self.throttled = 0
            made.append(self)

        def run(self):
            env = self.sim.env
            while True:
                req = yield self.box.get()
                req.hops += 1
                if self.bucket is not None and not self.bucket.take(req.rid, env.now):
                    self.throttled += 1          # before the pick: no order moves, no connection counts
                    continue
                edges = self.out_edges
                if self.algo == "round_robin":
                    key, edge = next(iter(edges.items()))
                    edges.move_to_end(key)
                else:
                    key = min(edges, key=lambda k: edges[k].conn)
                    edge = edges[key]
                edge.transport(req)

    return _RateLimitedLoadBalancer


def simulate(payload: dict, *, seed: int, replica: int, backend: str = "auto", normalised: bool = False,
             admission: dict[str, int] | None = None, deadline: dict[str, float] | None = None,
             client_timeout: float | None = None, rate_limit: dict[str, tuple[float, int]] | None = None,
             lb_rate_limit: tuple[float, int] | None = None, checks: list | None = None,
             ages: list | None = None) -> dict:
    """One replica as ``des_deadline.simulate``, its servers and load balancer throttling requests beyond their token
    buckets' rate and burst."""
    limits = {sid: _pair(f"rate_limit: server {sid!r}", v) for sid, v in (rate_limit or {}).items()}
    lb = _pair("lb_rate_limit", lb_rate_limit) if lb_rate_limit is not None else None
    p = payload if normalised else des_port.normalise_payload(payload)
    unknown = set(limits) - {s["id"] for s in p["servers"]}
    if unknown:
        raise KeyError(f"rate_limit: no server {sorted(unknown)}")
    if lb is not None and lb[0] > 0.0 and not p["load_balancer"]:
        raise ValueError("lb_rate_limit: the scenario has no load balancer")
    servers: list = []
    lbs: list = []
    base_factory = des_deadline._server_class

    def factory(lim, dls, made, ages_):
        return _server_class(base_factory(lim, dls, made, ages_), limits, servers, checks)

    saved_lb = des_port._LoadBalancer
    des_deadline._server_class = factory       # des_deadline.simulate builds its server class through this name
    des_port._LoadBalancer = _lb_class(lb, lbs, checks)
    try:
        out = des_deadline.simulate(p, seed=seed, replica=replica, backend=backend, normalised=True,
                                    admission=admission, deadline=deadline, client_timeout=client_timeout, ages=ages)
    finally:
        des_deadline._server_class = base_factory
        des_port._LoadBalancer = saved_lb
    out["server_throttled"] = {s.id: s.throttled for s in servers}
    out["lb_throttled"] = lbs[0].throttled if lbs else 0
    return out
