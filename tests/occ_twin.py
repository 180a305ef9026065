"""Python face of tests/host_twin/af_occ_twin.cpp: both state machines with occupancy integrals, and the oracle's ledger
of the same state changes -- TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a private temporary directory (``AF_OCC_TWIN_SO`` points at a build made by
hand instead).  Never imported by the product package."""

from __future__ import annotations

import atexit
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import band_twin as BT
import des_port
import dist_twin as DT
import latency_twin as LT
import numpy as np
import simpy

from asyncflow_b200 import _capi as K

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_occ_twin.cpp"
_lib = None
MASK64 = (1 << 64) - 1
#: the occupancy states of a server, in column order (afl::OC_*)
SERVER_STATES = ("ram_wait", "cpu_wait", "cpu", "io", "ram_mb")


def build() -> Path:
    if os.environ.get("AF_OCC_TWIN_SO"):
        return Path(os.environ["AF_OCC_TWIN_SO"])
    d = Path(tempfile.mkdtemp(prefix="af_occ_twin_"))
    atexit.register(shutil.rmtree, d, True)
    so = d / "libaf_occ_twin.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                    str(_SRC)], check=True)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
        L.af_occ_twin_error.restype = C.c_char_p
        L.af_occ_twin_frac_bits.argtypes = [u64, i32]
        L.af_occ_twin_frac_bits.restype = i32
        L.af_occ_twin_fixed.argtypes = [C.c_double, i32]
        L.af_occ_twin_fixed.restype = u64
        L.af_occ_twin_fits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), i32,
                                       C.c_char_p, C.c_int]
        L.af_occ_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), i32, u64, u64, u64, i32, i32, vp,
            i32, i32, vp, u64, u64, u32, vp, vp, vp, vp, vp, i32, vp, vp] + [vp] * 10
        L.af_occ_twin_run_warp.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), u64, u64, u64, vp, u64, i32, vp,
            i32, i32, vp, u64, u64, u32, vp, vp, vp, vp, vp, i32, vp, vp] + [vp] * 10
        _lib = L
    return _lib


def n_cols(flat) -> int:
    return 5 * flat.n_servers + flat.n_edges


def frac_bits(bound: int, horizon_s: int) -> int:
    """``afh::occ_frac_bits``: the f af_run's users pick for a bound and a horizon."""
    return int(lib().af_occ_twin_frac_bits(int(bound), int(horizon_s)))


def fixed_c(rest: float, f: int) -> int:
    """``afr::occ_fixed`` on the host."""
    return int(lib().af_occ_twin_fixed(float(rest), int(f)))


def fits(flat, f: int, *, request_capacity: int = 0, sweep=None) -> tuple[bool, str]:
    """The check ``af_run`` applies to a launch with f fraction bits: (fits, why not)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    sw_p, keep = LT._sweep(sweep)
    why = C.create_string_buffer(400)
    ok = lib().af_occ_twin_fits(C.byref(flat.pod), sw_p, C.byref(opt), int(f), why, 400)
    del keep
    return bool(ok), why.value.decode()


def _bands(flat, n, groups, n_groups, series, window, request_capacity, sweep):
    s = np.ascontiguousarray(series, dtype=np.int32)
    rows = {
        "band_rows": BT.new_rows(flat, n_groups),
        "band_from": np.full(n, 0xFFFFFFFF, dtype=np.uint32),
        "lat_rows": LT.new_rows(flat, n_groups, max(window, 1)),
        "lat_from": np.full(n, 0xFFFFFFFF, dtype=np.uint32),
        "dist_rows": (DT.new_rows(flat, s, n_groups, request_capacity, sweep) if s.size else np.zeros(1, dtype=np.uint32)),
    }
    return s, BT._groups(groups, n_groups), rows


def run_lane(flat, *, seed: int, n: int, f: int = 0, replica_begin: int = 0, sweep=None, lean: bool = False,
             groups=None, n_groups: int = 1, band_first: int = 0, sampled: bool = False, window: int = 0, series=(),
             trace: int = 0, clock_cap: int = 0, event_capacity: int = 2048, request_capacity: int = 16384,
             lane_bytes: int = 1816) -> dict:
    """The thread-per-replica engine over replicas ``[replica_begin, replica_begin + n)`` with occupancy integrals of
    ``f`` fraction bits (0: off) and optionally every kind of band.  Returns its outputs plus ``occ`` ([n, C] u64) and
    the band rows."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = BT._outputs(flat, n, trace, clock_cap)
    s, g, rows = _bands(flat, n, groups, n_groups, series, window, request_capacity, sweep)
    out.update(rows)
    out["occ"] = np.zeros((n, n_cols(flat)), dtype=np.uint64)
    slot = np.zeros(flat.n_series, dtype=np.int32)
    sw_p, keep = LT._sweep(sweep)
    rc = L.af_occ_twin_run_lane(C.byref(flat.pod), sw_p, C.byref(opt), lane_bytes, seed, replica_begin, n, int(lean),
                                int(f), out["occ"].ctypes.data, int(sampled), int(window), g.ctypes.data, band_first,
                                g.size, n_groups, out["band_rows"].ctypes.data, out["band_from"].ctypes.data,
                                out["lat_rows"].ctypes.data, out["lat_from"].ctypes.data, s.ctypes.data, s.size,
                                slot.ctypes.data, out["dist_rows"].ctypes.data, *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_occ_twin_error().decode())
    del keep
    return out


def run_warp(flat, *, seed: int, n: int, f: int = 0, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, sampled: bool = False, window: int = 0, series=(), trace: int = 0, clock_cap: int = 0,
             event_capacity: int = 0, request_capacity: int = 0, redo=None, into: dict | None = None) -> dict:
    """The warp-per-replica engine.  First-hand (``redo=None``) or, as af_run's second pass, a re-run of the local
    indices ``redo`` over ``into`` (the thread-per-replica pass's outputs): their bands continue from ``into``'s stop
    ticks, their other outputs and occupancy rows are overwritten."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = into if into is not None else BT._outputs(flat, n, trace, clock_cap)
    s, g, rows = _bands(flat, n, groups, n_groups, series, window, request_capacity or 16384, sweep)
    for k, v in rows.items():
        out.setdefault(k, v)
    out.setdefault("occ", np.zeros((n, n_cols(flat)), dtype=np.uint64))
    lst = None if redo is None else np.ascontiguousarray(redo, dtype=np.uint32)
    slot = np.zeros(flat.n_series, dtype=np.int32)
    sw_p, keep = LT._sweep(sweep)
    rc = L.af_occ_twin_run_warp(C.byref(flat.pod), sw_p, C.byref(opt), seed, replica_begin, n,
                                None if lst is None else lst.ctypes.data, 0 if lst is None else lst.size, int(f),
                                out["occ"].ctypes.data, int(sampled), int(window), g.ctypes.data, band_first, g.size,
                                n_groups, out["band_rows"].ctypes.data,
                                None if lst is None else out["band_from"].ctypes.data, out["lat_rows"].ctypes.data,
                                None if lst is None else out["lat_from"].ctypes.data, s.ctypes.data, s.size,
                                slot.ctypes.data, out["dist_rows"].ctypes.data, *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_occ_twin_error().decode())
    del keep
    return out


# ---- the oracle's ledger ---------------------------------------------------------------------------------------------
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
