"""Python face of tests/host_twin/af_split_twin.cpp: the thread-per-replica state machine with its shared-memory pool
split per replica (by each sweep row's own estimate, as af_run does, or at random) -- TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a private temporary directory (``AF_SPLIT_TWIN_SO`` points at a build made by
hand instead, e.g. under a sanitizer).  Never imported by the product package."""

from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from asyncflow_b200 import _capi as K

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_split_twin.cpp"
_lib = None

MODES = {"rows": 1, "random": 2}


def build() -> Path:
    if os.environ.get("AF_SPLIT_TWIN_SO"):
        return Path(os.environ["AF_SPLIT_TWIN_SO"])
    d = Path(tempfile.mkdtemp(prefix="af_split_twin_"))
    atexit.register(shutil.rmtree, d, True)
    so = d / "libaf_split_twin.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                    str(_SRC)], check=True)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.af_split_twin_error.restype = C.c_char_p
        L.af_split_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_split_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_uint64, C.POINTER(K.AfOptions), C.c_int32, C.c_int32,
            C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64] + [C.c_void_p] * 10
        L.af_split_twin_row_splits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_int32, C.c_void_p]
        _lib = L
    return _lib


def run(flat, *, split: str, seed: int, split_seed: int = 0, replica_begin: int = 0, n: int = 1, sweep=None,
        sweep_first: int = 0, trace: int = 0, clock_cap: int = 0, event_capacity: int = 2048,
        request_capacity: int = 16384, lane_bytes: int = 1816) -> dict:
    """Like tests/twin.py ``run(engine="lane")``, with every replica on its own split of the pool: ``split="rows"``
    (each replica with a sweep row by the row's estimate) or ``"random"`` (drawn from ``split_seed`` and the replica)."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    T = flat.horizon_s
    ne, nser = flat.n_edges, flat.n_series
    tick_cap = L.af_split_twin_trace_tick_capacity(C.byref(flat.pod))
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
        sw, keep = sweep.pod(sweep_first, None)
        sw_p = C.byref(sw)
    bufs = [out[k].ctypes.data for k in ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max",
                                         "trace_clocks", "trace_series", "trace_counts")]
    rc = L.af_split_twin_run_lane(C.byref(flat.pod), sw_p, sweep_first, C.byref(opt), lane_bytes, MODES[split],
                                  split_seed, seed, replica_begin, n, *bufs)
    if rc != 0:
        raise RuntimeError(L.af_split_twin_error().decode())
    del keep
    return out


def row_splits(flat, spec, lane_bytes: int):
    """(pool, reported (ev_s, rq_s), [(estimate, ev_s, rq_s) per row]) as af_run splits lanes of `lane_bytes`."""
    L = lib()
    sw, keep = spec.pod(0, None)
    out = (C.c_int32 * (3 + 3 * sw.n_rows))()
    assert L.af_split_twin_row_splits(C.byref(flat.pod), C.byref(sw), lane_bytes, out) == 0
    rows = [tuple(out[3 + 3 * r: 6 + 3 * r]) for r in range(sw.n_rows)]
    del keep
    return out[0], (out[1], out[2]), rows
