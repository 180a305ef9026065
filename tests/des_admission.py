"""The oracle with per-server admission limits (DESIGN.md §3.12) -- TEST INFRASTRUCTURE ONLY.

The reference has no admission limit (its ``ServerResources`` schema forbids extra keys), so this is the specification
of the behaviour the engine adds, written on ``oracle/des_port.py``'s actors and left unchanged there: a server with a
limit L sheds a request its dispatcher takes while L requests are in service, counting from admission until the
handler hands the request to the out-edge (RAM and core waits included)::

    def dispatch(self):
        while True:
            req = yield self.box.get()
            if self.limit and self.in_service >= self.limit:
                self.rejected += 1       # shed at the door: no hop recorded, no endpoint drawn, no handler started
                continue
            self.in_service += 1
            env.process(self.handle(req))

``simulate(payload, ..., admission={server_id: limit})`` is ``des_port.simulate`` with these servers (0 or a missing
server: no limit) plus ``server_rejected`` per server.  Without limits every output is ``des_port.simulate``'s."""

from __future__ import annotations

import sys
from pathlib import Path

_ORACLE = Path(__file__).resolve().parent.parent / "oracle"
if str(_ORACLE) not in sys.path:
    sys.path.insert(0, str(_ORACLE))

import des_port  # noqa: E402


def _server_class(limits: dict, made: list):
    class _AdmissionServer(des_port._Server):
        def __init__(self, sim, cfg: dict) -> None:
            super().__init__(sim, cfg)
            self.limit = int(limits.get(self.id, 0))
            self.in_service = 0
            self.rejected = 0
            made.append(self)

        def dispatch(self):
            env = self.sim.env
            while True:
                req = yield self.box.get()
                if self.limit and self.in_service >= self.limit:
                    self.rejected += 1
                    continue
                self.in_service += 1
                env.process(self.handle(req))

        def handle(self, req):
            # des_port's handler ends with out_edge.transport(req) and no yield after it: the request leaves service
            # in the same step, before any other process runs
            yield from super().handle(req)
            self.in_service -= 1

    return _AdmissionServer


def simulate(payload: dict, *, seed: int, replica: int, backend: str = "auto", normalised: bool = False,
             admission: dict[str, int] | None = None) -> dict:
    """One replica as ``des_port.simulate``, its servers shedding at ``admission[server_id]`` requests in service."""
    limits = dict(admission or {})
    p = payload if normalised else des_port.normalise_payload(payload)
    unknown = set(limits) - {s["id"] for s in p["servers"]}
    if unknown:
        raise KeyError(f"admission: no server {sorted(unknown)}")
    for sid, v in limits.items():
        if int(v) != v or v < 0:
            raise ValueError(f"admission: server {sid!r}: limit {v!r} is not an integer >= 0")
    made: list = []
    saved = des_port._Server
    des_port._Server = _server_class(limits, made)      # simulate() builds its servers from the module's class
    try:
        out = des_port.simulate(p, seed=seed, replica=replica, backend=backend, normalised=True)
    finally:
        des_port._Server = saved
    out["server_rejected"] = {s.id: s.rejected for s in made}
    return out
