"""The CPU twin with per-replica timeline rows (tests/host_twin/af_twin_rows.cpp) -- TEST INFRASTRUCTURE ONLY.

``run`` / ``run_lane`` / ``run_warp`` take what ``twin``'s do, plus the rows: ``timeline`` (a SweepSpec that sweeps
event times; default ``sweep`` when it does), whose rows ``[timeline_first, timeline_first + timeline_rows)`` describe
replicas from ``timeline_first`` -- rows are addressed by replica id, as the twin addresses sweep rows.  The launch itself
is ``twin``'s, on a library that is af_twin.cpp plus the rows.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from contextlib import contextmanager
from pathlib import Path

import twin

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_rows.so"


def build() -> Path:
    sources = [_DIR / "af_twin_rows.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_rows.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    """The rows library, every af_twin_* function declared as ``twin.lib()`` declares it."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        for name, f in vars(twin.lib()).items():
            if name.startswith("af_twin_"):
                g = getattr(L, name)
                g.restype, g.argtypes = f.restype, f.argtypes
        L.af_twin_rows_set.restype = C.c_int
        L.af_twin_rows_set.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfTimeline),
                                       C.c_uint64]
        L.af_twin_rows_sizeof_timeline.restype = C.c_int
        _lib = L
    return _lib


@contextmanager
def rows(flat, sweep=None, sweep_first: int = 0, timeline=None, timeline_first: int = 0, timeline_rows=None):
    """Inside the block, ``twin``'s launches (and whatever calls them, such as ``TwinEngine``) run on the rows library
    with these rows set."""
    L = lib()
    if timeline is None and sweep is not None and sweep.timelines is not None:
        timeline, timeline_first = sweep, sweep_first
    tl, keep = (None, None) if timeline is None else timeline.timeline_pod(timeline_first, timeline_rows)
    sw_p, keep_sw = twin._sweep(sweep, sweep_first)
    rc = L.af_twin_rows_set(C.byref(flat.pod), sw_p, None if tl is None else C.byref(tl), int(timeline_first))
    if rc != 0:
        raise RuntimeError(L.af_twin_error().decode())
    saved, twin._lib = twin._lib, L
    try:
        yield
    finally:
        twin._lib = saved
        L.af_twin_rows_set(C.byref(flat.pod), None, None, 0)
        del keep, keep_sw


def run_lane(flat, *, timeline=None, timeline_first: int = 0, timeline_rows: int | None = None, **kw) -> dict:
    with rows(flat, kw.get("sweep"), kw.get("sweep_first", 0), timeline, timeline_first, timeline_rows):
        return twin.run_lane(flat, **kw)


def run_warp(flat, *, timeline=None, timeline_first: int = 0, timeline_rows: int | None = None, **kw) -> dict:
    with rows(flat, kw.get("sweep"), kw.get("sweep_first", 0), timeline, timeline_first, timeline_rows):
        return twin.run_warp(flat, **kw)


def run(flat, *, timeline=None, timeline_first: int = 0, timeline_rows: int | None = None, **kw) -> dict:
    with rows(flat, kw.get("sweep"), kw.get("sweep_first", 0), timeline, timeline_first, timeline_rows):
        return twin.run(flat, **kw)
