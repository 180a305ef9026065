"""Python face of tests/host_twin/af_dist_twin.cpp: both state machines with per-tick distribution bands -- TEST
INFRASTRUCTURE ONLY.

The library is compiled on first use into a private temporary directory (``AF_DIST_TWIN_SO`` points at a build made by
hand instead).  Never imported by the product package."""

from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import band_twin as BT
import latency_twin as LT
import numpy as np

from asyncflow_b200 import _capi as K

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_dist_twin.cpp"
_lib = None


def build() -> Path:
    if os.environ.get("AF_DIST_TWIN_SO"):
        return Path(os.environ["AF_DIST_TWIN_SO"])
    d = Path(tempfile.mkdtemp(prefix="af_dist_twin_"))
    atexit.register(shutil.rmtree, d, True)
    so = d / "libaf_dist_twin.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                    str(_SRC)], check=True)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
        L.af_dist_twin_error.restype = C.c_char_p
        L.af_dist_twin_gauge_bin.argtypes = [u32]
        L.af_dist_twin_gauge_bin.restype = u32
        L.af_dist_twin_fits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), vp, i32, u64,
                                        u64, C.POINTER(u32), C.POINTER(u32), C.c_char_p, C.c_int]
        L.af_dist_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), i32, u64, u64, u64, i32, i32,
            vp, u64, u64, u32, vp, vp, vp, vp, i32, vp, i32, i32, vp, vp] + [vp] * 10
        L.af_dist_twin_run_warp.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), u64, u64, u64, vp, u64, i32, i32,
            vp, u64, u64, u32, vp, vp, vp, vp, vp, i32, i32, vp, vp] + [vp] * 10
        _lib = L
    return _lib


def gauge_bin(v: int) -> int:
    return int(lib().af_dist_twin_gauge_bin(int(v)))


def fits(flat, series, n_groups: int, mem_total: int = 1 << 62, *, request_capacity: int = 0, sweep=None):
    """The checks ``af_dist_bands_configure`` / ``af_bands_upload`` / ``af_run`` apply: (fits, ticks, bins, why)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    s = np.ascontiguousarray(series, dtype=np.int32)
    sw_p, keep = LT._sweep(sweep)
    t, b, why = C.c_uint32(), C.c_uint32(), C.create_string_buffer(400)
    ok = lib().af_dist_twin_fits(C.byref(flat.pod), sw_p, C.byref(opt), s.ctypes.data, s.size, int(n_groups), int(mem_total),
                                 C.byref(t), C.byref(b), why, 400)
    del keep
    return bool(ok), int(t.value), int(b.value), why.value.decode()


def new_rows(flat, series, n_groups: int, request_capacity: int, sweep=None) -> np.ndarray:
    ok, T, B, why = fits(flat, series, n_groups, request_capacity=request_capacity, sweep=sweep)
    assert ok, why
    return np.zeros((n_groups + 1, max(len(series), 1), T + 1, B), dtype=np.uint32)


def scan(rows: np.ndarray, n_groups: int, T: int) -> np.ndarray:
    """Difference rows -> [G, n_dist, T, n_bins] u32, as af_dist_scan_kernel (u32 modular sums)."""
    return np.cumsum(rows[:n_groups, :, :T], axis=2, dtype=np.uint32)


def run_lane(flat, *, seed: int, n: int, series, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, sampled: bool = False, window: int = 0, lean: bool = False, trace: int = 0,
             clock_cap: int = 0, event_capacity: int = 2048, request_capacity: int = 16384, lane_bytes: int = 1816,
             bin_capacity: int = 0) -> dict:
    """The thread-per-replica engine with distribution bands of ``series`` (empty: off), optionally the per-tick
    (``sampled``) and latency (``window`` s) bands, lean or full build.  Returns its outputs plus ``dist_rows``,
    ``band_rows``, ``band_from``, ``lat_rows``, ``lat_from``.  The bins follow ``bin_capacity`` (default: the request
    capacity), as af_run sizes them by the caller's capacity for both passes."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = BT._outputs(flat, n, trace, clock_cap)
    g = BT._groups(groups, n_groups)
    s = np.ascontiguousarray(series, dtype=np.int32)
    out["band_rows"] = BT.new_rows(flat, n_groups)
    out["band_from"] = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    out["lat_rows"] = LT.new_rows(flat, n_groups, max(window, 1))
    out["lat_from"] = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    out["dist_rows"] = (new_rows(flat, s, n_groups, bin_capacity or request_capacity, sweep) if s.size
                        else np.zeros(1, dtype=np.uint32))
    slot = np.zeros(flat.n_series, dtype=np.int32)
    sw_p, keep = LT._sweep(sweep)
    rc = L.af_dist_twin_run_lane(C.byref(flat.pod), sw_p, C.byref(opt), lane_bytes, seed, replica_begin, n,
                                 int(sampled), int(window), g.ctypes.data, band_first, g.size, n_groups,
                                 out["band_rows"].ctypes.data, out["band_from"].ctypes.data,
                                 out["lat_rows"].ctypes.data, out["lat_from"].ctypes.data, int(lean),
                                 s.ctypes.data, s.size, bin_capacity, slot.ctypes.data, out["dist_rows"].ctypes.data,
                                 *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_dist_twin_error().decode())
    del keep
    return out


def run_warp(flat, *, seed: int, n: int, series, replica_begin: int = 0, sweep=None, groups=None, n_groups: int = 1,
             band_first: int = 0, sampled: bool = False, window: int = 0, trace: int = 0, clock_cap: int = 0,
             event_capacity: int = 0, request_capacity: int = 0, redo=None, into: dict | None = None,
             bin_capacity: int = 0) -> dict:
    """The warp-per-replica engine.  First-hand (``redo=None``) or, as af_run's second pass, a re-run of the local
    indices ``redo`` continuing from ``into``'s stop ticks and adding to ``into``'s rows."""
    L = lib()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = into if into is not None else BT._outputs(flat, n, trace, clock_cap)
    s = np.ascontiguousarray(series, dtype=np.int32)
    rq = request_capacity or 16384
    out.setdefault("band_rows", BT.new_rows(flat, n_groups))
    out.setdefault("lat_rows", LT.new_rows(flat, n_groups, max(window, 1)))
    out.setdefault("dist_rows", new_rows(flat, s, n_groups, bin_capacity or rq, sweep) if s.size else np.zeros(1, dtype=np.uint32))
    g = BT._groups(groups, n_groups)
    lst = None if redo is None else np.ascontiguousarray(redo, dtype=np.uint32)
    bfrom = None if redo is None else np.ascontiguousarray(out["band_from"], dtype=np.uint32)
    lfrom = None if redo is None or not window else np.ascontiguousarray(out["lat_from"], dtype=np.uint32)
    slot = np.zeros(flat.n_series, dtype=np.int32)
    sw_p, keep = LT._sweep(sweep)
    rc = L.af_dist_twin_run_warp(C.byref(flat.pod), sw_p, C.byref(opt), seed, replica_begin, n,
                                 None if lst is None else lst.ctypes.data, 0 if lst is None else lst.size,
                                 int(sampled), int(window), g.ctypes.data, band_first, g.size, n_groups,
                                 out["band_rows"].ctypes.data, None if bfrom is None else bfrom.ctypes.data,
                                 out["lat_rows"].ctypes.data, None if lfrom is None else lfrom.ctypes.data,
                                 s.ctypes.data, s.size, bin_capacity, slot.ctypes.data, out["dist_rows"].ctypes.data,
                                 *[out[k].ctypes.data for k in BT.OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_dist_twin_error().decode())
    del keep
    return out
