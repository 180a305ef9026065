"""The launch checks of load-balancer sweep rows (tests/host_twin/af_twin_lb.cpp) -- TEST INFRASTRUCTURE ONLY.

``sweep_fits`` is af_sweep_upload's check of the ``lb_covered`` / ``lb_algorithm`` columns, ``cover_fits`` af_run's check
of the rows against the outage marks each replica runs with; both return ``None`` when the launch is accepted, else the
engine's message.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import twin

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_lb.so"


def build() -> Path:
    sources = [_DIR / "af_twin_lb.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_lb.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.af_twin_lb_error.restype = C.c_char_p
        L.af_twin_lb_sweep_fits.restype = C.c_int
        L.af_twin_lb_sweep_fits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep)]
        L.af_twin_lb_cover_fits.restype = C.c_int
        L.af_twin_lb_cover_fits.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_uint64,
                                            C.POINTER(K.AfTimeline), C.c_uint64, C.c_uint64, C.c_uint64]
        _lib = L
    return _lib


def sweep_fits(flat, spec) -> str | None:
    sw, keep = spec.pod()
    ok = lib().af_twin_lb_sweep_fits(C.byref(flat.pod), C.byref(sw))
    del keep
    return None if ok else lib().af_twin_lb_error().decode()


def cover_fits(flat, spec, begin: int, end: int, *, sweep_first: int = 0, timeline=None, timeline_first: int = 0) -> str | None:
    """af_run's check of a launch of [begin, end): ``spec``'s rows from ``sweep_first``, ``timeline``'s (a SweepSpec with
    timelines, default none) from ``timeline_first``."""
    sw, keep = spec.pod()
    tl, keep_tl = (None, None) if timeline is None else timeline.timeline_pod()
    ok = lib().af_twin_lb_cover_fits(C.byref(flat.pod), C.byref(sw), int(sweep_first), None if tl is None else C.byref(tl),
                                     int(timeline_first), int(begin), int(end))
    del keep, keep_tl
    return None if ok else lib().af_twin_lb_error().decode()
