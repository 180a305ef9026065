"""The oracle side of the band and occupancy tests -- TEST INFRASTRUCTURE ONLY.

Definitions restated in Python, independently of the engines' code: the prefix scans that turn difference rows into
per-tick values, the latency-band binning of a replica's clocks, the occupancy fixed point, and the oracle's ledger of
the state changes the occupancy columns integrate."""

from __future__ import annotations

import math

import des_port
import numpy as np
import simpy
from twin import ticks

from asyncflow_b200 import _capi as K

MASK64 = (1 << 64) - 1


# ---- per-tick and distribution bands ---------------------------------------------------------------------------------
def scan(flat, rows: np.ndarray, n_groups: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Difference rows -> (count [G, T] u32, sum [G, S, T] u64, sumsq [G, S, T] u64), as af_run's scan kernel."""
    T, S = ticks(flat), flat.n_series
    v = np.cumsum(rows[:n_groups, :, :T], axis=2, dtype=np.uint64)      # u64 wraps: the device's modular arithmetic
    return v[:, 0, :].astype(np.uint32), v[:, 1:1 + S, :], v[:, 1 + S:, :]


def dist_scan(rows: np.ndarray, n_groups: int, T: int) -> np.ndarray:
    """Difference rows -> [G, n_dist, T, n_bins] u32, as af_dist_scan_kernel (u32 modular sums)."""
    return np.cumsum(rows[:n_groups, :, :T], axis=2, dtype=np.uint32)


# ---- latency bands ---------------------------------------------------------------------------------------------------
def hist_bin(lat: float) -> int:
    bits = int(np.array([lat], dtype=np.float64).view(np.uint64)[0])
    idx = (bits >> (52 - K.AF_HIST_SUB_BITS)) - ((1023 + K.AF_HIST_MIN_EXP) << K.AF_HIST_SUB_BITS)
    return min(max(idx, 0), K.AF_HIST_BINS - 1)


def bin_clocks(rows: np.ndarray, g: int, clocks: np.ndarray, w: int, horizon_s: int) -> None:
    """Add one replica's completions ``clocks[i] = (start, finish)`` to group ``g`` of ``rows``: window
    ``(ceil(finish) - 1) // w`` (bucket clamped at 0), latency bin, ``round(lat * 2^32)`` split into two words."""
    for start, finish in clocks:
        lat = float(finish) - float(start)
        b = max(math.ceil(float(finish)) - 1, 0)
        if b >= horizon_s:
            continue
        k = b // w
        u = round(lat * 4294967296.0)                 # exact scaling; Python rounds half to even
        rows[g, k, hist_bin(lat)] += np.uint64(1)
        rows[g, k, K.AF_HIST_BINS] += np.uint64(u >> 32)
        rows[g, k, K.AF_HIST_BINS + 1] += np.uint64(u & 0xFFFFFFFF)


# ---- occupancy ---------------------------------------------------------------------------------------------------------
def fixed(rest: float, f: int) -> int:
    """``afr::occ_fixed`` restated: round-to-nearest-even(rest * 2^f) (Python's round() of a float ties to even)."""
    return round(math.ldexp(rest, f))


def oracle_ledger(payload: dict, flat, *, seed: int, replica: int) -> tuple[dict, list, list]:
    """One oracle replica (``des_port.simulate``, unchanged) with every change of a count the occupancy columns
    integrate recorded as ``(t, column, delta)``: the servers' ready / I/O queues and RAM in use, the edges' connections
    (the sampled gauges, whether sampled or not), the cores held (capacity minus the CPU container's level) and the
    requests waiting in the RAM container's get queue (a get served at once enters and leaves at the same instant).
    Returns (the oracle's result, the ledger, every generated request as (start, end) -- end = finish or drop time,
    None while in flight at the horizon)."""
    sid = {s: i for i, s in enumerate(flat.server_ids)}
    eid = {e: i for i, e in enumerate(flat.edge_ids)}
    ns = flat.n_servers
    ledger: list = []
    requests: list = []
    env_of: dict = {}

    def log(owner, col, delta):
        if delta:
            ledger.append((env_of["env"].now, col, delta))

    def gauge(attr, col_of):
        hidden = "_occ_" + attr

        def get(self):
            return getattr(self, hidden)

        def put(self, v):
            old = getattr(self, hidden, None)
            if old is not None:
                log(self, col_of(self), v - old)
            setattr(self, hidden, v)
        return property(get, put)

    class CpuContainer(simpy.Container):
        col = 0

        @property
        def _level(self):
            return self._occ_level

        @_level.setter
        def _level(self, v):
            old = getattr(self, "_occ_level", None)
            if old is not None:
                log(self, self.col, old - v)                  # a core taken lowers the level
            self._occ_level = v

    class RamQueue(list):
        def __init__(self, col):
            super().__init__()
            self.col = col

        def append(self, x):
            super().append(x)
            log(self, self.col, 1)

        def pop(self, i=-1):
            x = super().pop(i)
            log(self, self.col, -1)
            return x

    class Server(des_port._Server):
        ready_q = gauge("ready_q", lambda s: 5 * sid[s.id] + 1)
        io_q = gauge("io_q", lambda s: 5 * sid[s.id] + 3)
        ram_in_use = gauge("ram_in_use", lambda s: 5 * sid[s.id] + 4)

        def __init__(self, sim, cfg):
            env_of["env"] = sim.env
            super().__init__(sim, cfg)
            cpu = CpuContainer(sim.env, capacity=cfg["cpu_cores"], init=cfg["cpu_cores"])
            cpu.col = 5 * sid[self.id] + 2
            self.cpu = cpu
            self.ram.get_queue = RamQueue(5 * sid[self.id])

    class Edge(des_port._Edge):
        conn = gauge("conn", lambda e: 5 * ns + eid[e.id])

    class Request(des_port._Request):
        __slots__ = ()

        def __init__(self, rid, t0):
            super().__init__(rid, t0)
            requests.append(self)

    saved = des_port._Server, des_port._Edge, des_port._Request
    des_port._Server, des_port._Edge, des_port._Request = Server, Edge, Request
    try:
        o = des_port.simulate(payload, seed=seed, replica=replica)
    finally:
        des_port._Server, des_port._Edge, des_port._Request = saved
    return o, ledger, [(r.t0, r.finish) for r in requests]


def ledger_rows(ledger: list, n: int, horizon: float, f: int) -> np.ndarray:
    """[n] u64: sum of delta * fixed(H - t) over the ledger, in u64 modular arithmetic."""
    acc = [0] * n
    for t, c, d in ledger:
        acc[c] = (acc[c] + d * fixed(horizon - t, f)) & MASK64
    return np.array(acc, dtype=np.uint64)
