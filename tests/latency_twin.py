"""Python face of tests/host_twin/af_latency_twin.cpp: both state machines with per-window latency bands -- TEST
INFRASTRUCTURE ONLY.

The library is compiled on first use into a private temporary directory (``AF_LAT_TWIN_SO`` points at a build made by
hand instead).  Never imported by the product package.  Also the oracle side: :func:`bin_clocks` bins a replica's
``(start, finish)`` clocks the way the latency bands are defined, independently of the engines' code."""

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
import numpy as np

from asyncflow_b200 import _capi as K

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_latency_twin.cpp"
_lib = None
ROW = K.AF_HIST_BINS + 2


def build() -> Path:
    if os.environ.get("AF_LAT_TWIN_SO"):
        return Path(os.environ["AF_LAT_TWIN_SO"])
    d = Path(tempfile.mkdtemp(prefix="af_lat_twin_"))
    atexit.register(shutil.rmtree, d, True)
    so = d / "libaf_lat_twin.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                    str(_SRC)], check=True)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
        L.af_lat_twin_error.restype = C.c_char_p
        L.af_lat_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_lat_twin_fixed32.argtypes = [C.c_double]
        L.af_lat_twin_fixed32.restype = u64
        L.af_lat_twin_hist_bin.argtypes = [C.c_double]
        L.af_lat_twin_fits.argtypes = [i32, i32, u64, u64, C.c_char_p, C.c_int]
        L.af_lat_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), i32, u64, u64, u64, i32, i32,
            vp, u64, u64, u32, vp, vp, vp, vp] + [vp] * 10
        L.af_lat_twin_run_warp.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), u64, u64, u64, vp, u64, i32, i32,
            vp, u64, u64, u32, vp, vp, vp, vp] + [vp] * 10
        _lib = L
    return _lib


def windows(flat, w: int) -> int:
    return -(-int(flat.horizon_s) // int(w))


def fits(window_s: int, horizon_s: int, n_groups: int, mem_total: int) -> tuple[bool, str]:
    why = C.create_string_buffer(256)
    ok = lib().af_lat_twin_fits(int(window_s), int(horizon_s), int(n_groups), int(mem_total), why, 256)
    return bool(ok), why.value.decode()


def new_rows(flat, n_groups: int, w: int) -> np.ndarray:
    return np.zeros((n_groups + 1, max(windows(flat, w), 1), ROW), dtype=np.uint64)


def split(rows: np.ndarray, n_groups: int):
    """Rows -> (hist [G, W, AF_HIST_BINS], sum_hi [G, W], sum_lo [G, W]) of the fetched groups."""
    r = rows[:n_groups]
    return r[:, :, :K.AF_HIST_BINS], r[:, :, K.AF_HIST_BINS], r[:, :, K.AF_HIST_BINS + 1]


# ---- the oracle side: the definition, restated in Python ------------------------------------------------------------
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


# ---- the engines --------------------------------------------------------------------------------------------------
def _sweep(sweep):
    if sweep is None:
        return None, None
    sw, keep = sweep.pod(0, None)
    return C.byref(sw), keep


def run_lane(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, sampled: bool = False, window: int = 1, trace: int = 0, clock_cap: int = 0,
             event_capacity: int = 2048, request_capacity: int = 16384, lane_bytes: int = 1816) -> dict:
    """The thread-per-replica engine with latency bands of ``window`` seconds (0: off) and, when ``sampled``, the
    per-tick bands.  Returns its outputs plus ``lat_rows`` / ``lat_from`` and ``band_rows`` / ``band_from``."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = BT._outputs(flat, n, trace, clock_cap)
    g = BT._groups(groups, n_groups)
    out["band_rows"] = BT.new_rows(flat, n_groups)
    out["band_from"] = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    out["lat_rows"] = new_rows(flat, n_groups, max(window, 1))
    out["lat_from"] = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    sw_p, keep = _sweep(sweep)
    rc = L.af_lat_twin_run_lane(C.byref(flat.pod), sw_p, C.byref(opt), lane_bytes, seed, replica_begin, n,
                                int(sampled), int(window), g.ctypes.data, band_first, g.size, n_groups,
                                out["band_rows"].ctypes.data, out["band_from"].ctypes.data,
                                out["lat_rows"].ctypes.data, out["lat_from"].ctypes.data,
                                *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_lat_twin_error().decode())
    del keep
    return out


def run_warp(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, sampled: bool = False, window: int = 1, trace: int = 0, clock_cap: int = 0,
             event_capacity: int = 0, request_capacity: int = 0, redo=None, into: dict | None = None) -> dict:
    """The warp-per-replica engine.  First-hand (``redo=None``): every replica of the launch.  A re-run (``redo`` =
    local indices, ``into`` = the lane pass's outputs): those replicas again, as af_run's second pass, continuing
    from ``into["lat_from"]`` / ``into["band_from"]`` and adding to ``into``'s rows."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = into if into is not None else BT._outputs(flat, n, trace, clock_cap)
    out.setdefault("band_rows", BT.new_rows(flat, n_groups))
    out.setdefault("lat_rows", new_rows(flat, n_groups, max(window, 1)))
    g = BT._groups(groups, n_groups)
    lst = None if redo is None else np.ascontiguousarray(redo, dtype=np.uint32)
    bfrom = None if redo is None else np.ascontiguousarray(out["band_from"], dtype=np.uint32)
    lfrom = None if redo is None else np.ascontiguousarray(out["lat_from"], dtype=np.uint32)
    sw_p, keep = _sweep(sweep)
    rc = L.af_lat_twin_run_warp(C.byref(flat.pod), sw_p, C.byref(opt), seed, replica_begin, n,
                                None if lst is None else lst.ctypes.data, 0 if lst is None else lst.size,
                                int(sampled), int(window), g.ctypes.data, band_first, g.size, n_groups,
                                out["band_rows"].ctypes.data, None if bfrom is None else bfrom.ctypes.data,
                                out["lat_rows"].ctypes.data, None if lfrom is None else lfrom.ctypes.data,
                                *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_lat_twin_error().decode())
    del keep
    return out
