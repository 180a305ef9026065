"""Python face of tests/host_twin/af_band_twin.cpp: both state machines with per-tick bands -- TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a private temporary directory (``AF_BAND_TWIN_SO`` points at a build made by
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

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_band_twin.cpp"
_lib = None
OUTPUTS = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "trace_clocks", "trace_series",
           "trace_counts")


def build() -> Path:
    if os.environ.get("AF_BAND_TWIN_SO"):
        return Path(os.environ["AF_BAND_TWIN_SO"])
    d = Path(tempfile.mkdtemp(prefix="af_band_twin_"))
    atexit.register(shutil.rmtree, d, True)
    so = d / "libaf_band_twin.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                    str(_SRC)], check=True)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
        L.af_band_twin_error.restype = C.c_char_p
        L.af_band_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_band_twin_ticks.argtypes = [C.POINTER(K.AfScenario)]
        L.af_band_twin_ticks.restype = u32
        L.af_band_twin_ticks_fit.argtypes = [C.POINTER(K.AfScenario), C.c_char_p, C.c_int]
        L.af_band_twin_sumsq_fits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), u64,
                                              C.POINTER(u64), C.c_char_p, C.c_int]
        L.af_band_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), u64, C.POINTER(K.AfOptions), i32, u64, u64, u64,
            i32, vp, u64, u64, u32, vp, vp] + [vp] * 10
        L.af_band_twin_run_warp.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), u64, C.POINTER(K.AfOptions), u64, u64, u64, vp, u64,
            i32, vp, u64, u64, u32, vp, vp] + [vp] * 10
        _lib = L
    return _lib


def ticks(flat) -> int:
    """The ticks a replica that reaches the horizon takes (what ``af_fetch_bands`` reports as ``n_ticks``)."""
    return int(lib().af_band_twin_ticks(C.byref(flat.pod)))


def ticks_fit(flat) -> tuple[bool, str]:
    """The tick-count check ``af_bands_upload`` / ``af_run`` apply: (fits, why not)."""
    why = C.create_string_buffer(256)
    ok = lib().af_band_twin_ticks_fit(C.byref(flat.pod), why, 256)
    return bool(ok), why.value.decode()


def sumsq_fits(flat, group: int, *, request_capacity: int = 0, sweep=None) -> tuple[bool, int, str]:
    """The check ``af_bands_upload`` applies: (fits, bound on a gauge, what sets the bound)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    sw_p, keep = None, None
    if sweep is not None:
        sw, keep = sweep.pod(0, None)
        sw_p = C.byref(sw)
    bound, what = C.c_uint64(), C.create_string_buffer(256)
    ok = lib().af_band_twin_sumsq_fits(C.byref(flat.pod), sw_p, C.byref(opt), int(group), C.byref(bound), what, 256)
    del keep
    return bool(ok), int(bound.value), what.value.decode()


def new_rows(flat, n_groups: int) -> np.ndarray:
    """Zeroed difference rows of ``n_groups`` groups plus the one of replicas without a group."""
    return np.zeros(((n_groups + 1), 1 + 2 * flat.n_series, ticks(flat) + 1), dtype=np.uint64)


def scan(flat, rows: np.ndarray, n_groups: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Difference rows -> (count [G, T] u32, sum [G, S, T] u64, sumsq [G, S, T] u64), as af_run's scan kernel."""
    T, S = ticks(flat), flat.n_series
    v = np.cumsum(rows[:n_groups, :, :T], axis=2, dtype=np.uint64)      # u64 wraps: the device's modular arithmetic
    return v[:, 0, :].astype(np.uint32), v[:, 1:1 + S, :], v[:, 1 + S:, :]


def _outputs(flat, n: int, trace: int, clock_cap: int) -> dict:
    nser = flat.n_series
    tick_cap = lib().af_band_twin_trace_tick_capacity(C.byref(flat.pod))
    return {
        "stats": np.zeros(n, dtype=K.STATS_DTYPE),
        "sent": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "dropped": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "hist": np.zeros((n, K.AF_HIST_BINS), dtype=np.uint32),
        "thr": np.zeros((n, flat.horizon_s), dtype=np.uint32),
        "samp_sum": np.zeros((n, nser), dtype=np.uint64),
        "samp_max": np.zeros((n, nser), dtype=np.uint32),
        "trace_clocks": np.zeros((max(trace, 1), max(clock_cap, 1), 2), dtype=np.float64),
        "trace_series": np.zeros((max(trace, 1), nser, tick_cap), dtype=np.uint32),
        "trace_counts": np.zeros((max(n, 1), 2), dtype=np.uint32),
    }


def _groups(groups, n_groups):
    g = np.ascontiguousarray(groups if groups is not None else np.zeros(0), dtype=np.uint32)
    assert g.size == 0 or int(g.max()) < n_groups
    return g


def run_lane(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, bands: bool = True, trace: int = 0, clock_cap: int = 0, event_capacity: int = 2048,
             request_capacity: int = 16384, lane_bytes: int = 1816) -> dict:
    """The thread-per-replica engine over replicas ``[replica_begin, replica_begin + n)`` (sweep rows from replica 0);
    ``groups[i]`` = group of replica ``band_first + i``.  Returns its outputs plus ``band_rows`` (difference rows) and
    ``band_from`` (per local replica: the tick a stopped replica stopped at)."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = _outputs(flat, n, trace, clock_cap)
    g = _groups(groups, n_groups)
    out["band_rows"] = new_rows(flat, n_groups)
    out["band_from"] = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    sw_p, keep = None, None
    if sweep is not None:
        sw, keep = sweep.pod(0, None)
        sw_p = C.byref(sw)
    rc = L.af_band_twin_run_lane(C.byref(flat.pod), sw_p, 0, C.byref(opt), lane_bytes, seed, replica_begin, n,
                                 int(bands), g.ctypes.data, band_first, g.size, n_groups, out["band_rows"].ctypes.data,
                                 out["band_from"].ctypes.data, *[out[k].ctypes.data for k in OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_band_twin_error().decode())
    del keep
    return out


def run_warp(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, bands: bool = True, trace: int = 0, clock_cap: int = 0, event_capacity: int = 0,
             request_capacity: int = 0, redo=None, band_from=None, into: dict | None = None) -> dict:
    """The warp-per-replica engine.  First-hand (``redo=None``): every replica of the launch.  A re-run
    (``redo`` = local indices, ``band_from`` = the lane pass's stop ticks, ``into`` = the lane pass's outputs): those
    replicas again, as af_run's second pass, adding to ``into["band_rows"]`` and overwriting their outputs there."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = into if into is not None else _outputs(flat, n, trace, clock_cap)
    if "band_rows" not in out:
        out["band_rows"] = new_rows(flat, n_groups)
    g = _groups(groups, n_groups)
    lst = None if redo is None else np.ascontiguousarray(redo, dtype=np.uint32)
    frm = None if band_from is None else np.ascontiguousarray(band_from, dtype=np.uint32)
    sw_p, keep = None, None
    if sweep is not None:
        sw, keep = sweep.pod(0, None)
        sw_p = C.byref(sw)
    rc = L.af_band_twin_run_warp(C.byref(flat.pod), sw_p, 0, C.byref(opt), seed, replica_begin, n,
                                 None if lst is None else lst.ctypes.data, 0 if lst is None else lst.size,
                                 int(bands), g.ctypes.data, band_first, g.size, n_groups, out["band_rows"].ctypes.data,
                                 None if frm is None else frm.ctypes.data, *[out[k].ctypes.data for k in OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_band_twin_error().decode())
    del keep
    return out
