"""The oracle with request deadlines and a client timeout (DESIGN.md §3.13) -- TEST INFRASTRUCTURE ONLY.

The reference has no deadline, so this is the specification of the behaviour the engine adds, written on
``tests/des_admission.py``'s server (admission limits and deadlines compose) and leaving ``oracle/des_port.py`` and
``des_admission.py`` unchanged.  A request's age is ``now - t0``, ``t0`` the time the generator created it.  A server
with a deadline D checks the age before each CPU step's timeout, once the request holds a core (a core just granted
or one kept from the previous CPU step); past it, the request abandons::

    if self.deadline and env.now - req.t0 > self.deadline:
        yield from self._release(core_locked, in_io, waiting, total_ram)   # the handler's tail, as it stands
        self.expired += 1
        return                                                            # no out_edge.transport(req)

The abandon path yields what a finished handler yields, in the same order, so SimPy's event order is that of a
request whose remaining steps took no time.  A request that never runs a CPU step there is never checked, nor is one
waiting for RAM before its first CPU step.  With an admission limit the request leaves service there.

The client timeout T counts a completion with ``finish - start > T`` in ``late`` (the completion still counts
everywhere else).  ``simulate(payload, ..., admission=, deadline={server_id: D}, client_timeout=T)`` is
``des_admission.simulate`` plus ``server_expired`` per server and ``late``; 0 or a missing server: none.  Without
deadlines and a timeout every other output is ``des_admission.simulate``'s.  ``ages=[]`` collects
``(server_id, rid, now - t0)`` at every check, deadline or not."""

from __future__ import annotations

import math

import des_admission
from des_admission import des_port

CPU_KINDS, IO_KINDS, RAM_KINDS = des_port.CPU_KINDS, des_port.IO_KINDS, des_port.RAM_KINDS


def _seconds(what: str, v) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
        raise ValueError(f"{what}: {v!r} is not a finite number of seconds >= 0")
    return float(v)


def _server_class(limits: dict, deadlines: dict, made: list, ages: list | None):
    base = des_admission._server_class(limits, made)

    class _DeadlineServer(base):
        def __init__(self, sim, cfg: dict) -> None:
            super().__init__(sim, cfg)
            self.deadline = float(deadlines.get(self.id, 0.0))
            self.expired = 0

        def _release(self, core_locked: bool, in_io: bool, waiting: bool, total_ram: int):
            """The tail of des_port's handler (its lines after the step loop), up to the forward."""
            if core_locked:
                yield self.cpu.put(1)
            if in_io:
                self.io_q -= 1
            if waiting:
                self.ready_q -= 1
            if total_ram:
                self.ram_in_use -= total_ram
                yield self.ram.put(total_ram)

        def _handle(self, req):
            """des_port._Server.handle with the deadline check after a CPU step's core is held."""
            env = self.sim.env
            req.hops += 1
            ep = self.endpoints[self.sim.rng.endpoint(req.rid, req.hops, len(self.endpoints))]
            steps = ep["steps"]
            total_ram = sum(s["value"] for s in steps if s["kind"] in RAM_KINDS)
            if total_ram:
                yield self.ram.get(total_ram)
                self.ram_in_use += total_ram
            core_locked = False
            in_io = False
            waiting = False
            for s in steps:
                kind = s["kind"]
                if kind in CPU_KINDS:
                    if in_io:
                        in_io = False
                        self.io_q -= 1
                    if not core_locked:
                        cpu_req = self.cpu.get(1)
                        if not cpu_req.triggered:
                            waiting = True
                            self.ready_q += 1
                        yield cpu_req
                        if waiting:
                            waiting = False
                            self.ready_q -= 1
                        core_locked = True
                    if ages is not None:
                        ages.append((self.id, req.rid, env.now - req.t0))
                    if self.deadline and env.now - req.t0 > self.deadline:
                        yield from self._release(core_locked, in_io, waiting, total_ram)
                        self.expired += 1
                        return
                    yield env.timeout(s["value"])
                elif kind in IO_KINDS:
                    if core_locked:
                        yield self.cpu.put(1)
                        core_locked = False
                        if not in_io:
                            in_io = True
                            self.io_q += 1
                    elif not in_io:
                        in_io = True
                        self.io_q += 1
                    yield env.timeout(s["value"])
            yield from self._release(core_locked, in_io, waiting, total_ram)
            self.out_edge.transport(req)

        def handle(self, req):
            # the request leaves service (admission limit) when it is handed to the out-edge or abandons
            yield from self._handle(req)
            self.in_service -= 1

    return _DeadlineServer


def simulate(payload: dict, *, seed: int, replica: int, backend: str = "auto", normalised: bool = False,
             admission: dict[str, int] | None = None, deadline: dict[str, float] | None = None,
             client_timeout: float | None = None, ages: list | None = None) -> dict:
    """One replica as ``des_admission.simulate``, its servers dropping requests older than ``deadline[server_id]``
    at a CPU step and its client counting completions later than ``client_timeout`` in ``late``."""
    limits = dict(admission or {})
    dls = {sid: _seconds(f"deadline: server {sid!r}", v) for sid, v in (deadline or {}).items()}
    timeout = _seconds("client_timeout", client_timeout) if client_timeout is not None else 0.0
    p = payload if normalised else des_port.normalise_payload(payload)
    ids = {s["id"] for s in p["servers"]}
    unknown = (set(limits) | set(dls)) - ids
    if unknown:
        raise KeyError(f"no server {sorted(unknown)}")
    for sid, v in limits.items():
        if int(v) != v or v < 0:
            raise ValueError(f"admission: server {sid!r}: limit {v!r} is not an integer >= 0")
    made: list = []
    saved = des_port._Server
    des_port._Server = _server_class(limits, dls, made, ages)
    try:
        out = des_port.simulate(p, seed=seed, replica=replica, backend=backend, normalised=True)
    finally:
        des_port._Server = saved
    out["server_rejected"] = {s.id: s.rejected for s in made}
    out["server_expired"] = {s.id: s.expired for s in made}
    out["late"] = sum(1 for t0, t1 in out["clocks"] if t1 - t0 > timeout) if timeout > 0.0 else 0
    return out
