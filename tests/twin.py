"""Python face of the CPU debugging twin (tests/host_twin) -- TEST INFRASTRUCTURE ONLY.

Runs the engine's state machine (asyncflow_b200/csrc/af_core.cuh compiled for the
host, one-lane warp) so CPU-only tests can check event semantics against the
oracle.  Never imported by the product package.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_host_twin.so"
_SRC = [_DIR / "af_host_twin.cpp"] + sorted((_DIR.parent.parent / "asyncflow_b200" / "csrc").glob("*.*h")) \
    + [_DIR.parent.parent / "include" / "asyncflow_b200.h"]


def build() -> Path:
    if os.environ.get("AF_TWIN_SO"):          # experiments: a twin built by hand (e.g. with a -D of a kernel variant)
        return Path(os.environ["AF_TWIN_SO"])
    so = _SO
    newest = max(p.stat().st_mtime for p in _SRC)
    if not so.exists() or so.stat().st_mtime < newest:
        so.parent.mkdir(exist_ok=True)
        subprocess.run(
            ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
             "-o", str(so), str(_DIR / "af_host_twin.cpp")], check=True)
    return so


_libs: dict = {}


def lib() -> C.CDLL:
    if None not in _libs:
        L = C.CDLL(str(build()))
        L.af_twin_error.restype = C.c_char_p
        L.af_twin_hist_percentile.restype = C.c_double
        L.af_twin_hist_percentile.argtypes = [C.c_void_p, C.c_uint64, C.c_double, C.c_double, C.c_double]
        L.af_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_twin_run.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_uint64, C.POINTER(K.AfOptions),
            C.c_uint64, C.c_uint64, C.c_uint64] + [C.c_void_p] * 10
        L.af_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_uint64, C.POINTER(K.AfOptions), C.c_int32,
            C.c_uint64, C.c_uint64, C.c_uint64] + [C.c_void_p] * 10
        _libs[None] = L
    return _libs[None]


#: which state machine run() drives when the caller does not say: "lane" = af_lane.cuh (thread per replica, the
#: product's first pass), "warp" = af_core.cuh (warp per replica, the product's pass for flagged replicas)
DEFAULT_ENGINE = os.environ.get("AF_TWIN_ENGINE", "lane")
#: the lane's share of shared memory in the twin (the CUDA engine derives it from the occupancy it picks)
DEFAULT_LANE_BYTES = int(os.environ.get("AF_TWIN_LANE_BYTES", "1816"))


def run(flat, *, seed: int, replica_begin: int = 0, n: int = 1, sweep=None, sweep_first: int = 0, trace: int = 0,
        clock_cap: int = 0, event_capacity: int = 0, request_capacity: int = 0,
        engine: str | None = None, lane_bytes: int | None = None, ev_need: int = 0) -> dict:
    """``ev_need``: the pending-events estimate the lane engine splits its shared memory by (af_run computes it from the
    scenario and the sweep; 0 = the even split)."""
    L = lib()
    engine = engine or DEFAULT_ENGINE
    if engine == "lane":      # same default capacities as the warp engine (the CUDA lane pass has smaller ones and escalates)
        event_capacity = event_capacity or 2048
        request_capacity = request_capacity or 16384
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    T = flat.horizon_s
    ne, nser = flat.n_edges, flat.n_series
    tick_cap = L.af_twin_trace_tick_capacity(C.byref(flat.pod))
    out = {
        "stats": np.zeros(n, dtype=K.STATS_DTYPE),
        "sent": np.zeros((n, ne), dtype=np.uint32),
        "dropped": np.zeros((n, ne), dtype=np.uint32),
        "hist": np.zeros((n, K.AF_HIST_BINS), dtype=np.uint32),
        "thr": np.zeros((n, T), dtype=np.uint32),
        "samp_sum": np.zeros((n, nser), dtype=np.uint64),
        "samp_max": np.zeros((n, nser), dtype=np.uint32),
        "trace_clocks": np.zeros((max(trace, 1), max(clock_cap, 1), 2), dtype=np.float64),
        "trace_series": np.zeros((max(trace, 1), nser, tick_cap), dtype=np.uint32),
        "trace_counts": np.zeros((max(n, 1), 2), dtype=np.uint32),
    }
    sw_p, keep = None, None
    if sweep is not None:
        # rows [sweep_first, end) of the table describe replicas sweep_first, sweep_first+1, ...
        sw, keep = sweep.pod(sweep_first, None)
        sw_p = C.byref(sw)
    bufs = [out[k].ctypes.data for k in ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max",
                                         "trace_clocks", "trace_series", "trace_counts")]
    if engine == "lane":
        L.af_twin_set_ev_need(int(ev_need))
        rc = L.af_twin_run_lane(C.byref(flat.pod), sw_p, sweep_first, C.byref(opt), lane_bytes or DEFAULT_LANE_BYTES,
                                seed, replica_begin, n, *bufs)
    else:
        rc = L.af_twin_run(C.byref(flat.pod), sw_p, sweep_first, C.byref(opt), seed, replica_begin, n, *bufs)
    if rc != 0:
        raise RuntimeError(L.af_twin_error().decode())
    del keep
    return out
