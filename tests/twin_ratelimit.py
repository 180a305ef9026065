"""The CPU twin with rate limits (tests/host_twin/af_twin_ratelimit.cpp) -- TEST INFRASTRUCTURE ONLY.

``run`` / ``run_lane`` / ``run_warp`` take what ``twin_deadline``'s do and add ``throttled`` ([n, n_servers + 1]: the
requests each server, then the load balancer, throttled at its rate limit) to the outputs; the limits come with the
scenario (``flatten.set_rate_limits``) and the sweep (``("server_rate"|"server_burst", server_id)``, ``("lb_rate",)``,
``("lb_burst",)`` columns).  ``into=`` (a warp re-run) keeps writing ``into["throttled"]``.  Also the C checks and the
GCRA rule on its own.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import twin
import twin_deadline

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_ratelimit.so"


def build() -> Path:
    sources = [_DIR / "af_twin_ratelimit.cpp", _DIR / "af_twin_deadline.cpp", _DIR / "af_twin_admission.cpp",
               _DIR / "af_twin_streams.cpp", _DIR / "af_twin_rows.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_ratelimit.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    """The rate-limit library, every af_twin_* function declared as ``twin_deadline.lib()`` declares it."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        for name, f in vars(twin_deadline.lib()).items():
            if name.startswith("af_twin_"):
                g = getattr(L, name)
                g.restype, g.argtypes = f.restype, f.argtypes
        L.af_twin_ratelimit_set.restype = None
        L.af_twin_ratelimit_set.argtypes = [C.c_void_p, C.c_double, C.c_int32]
        for name in ("af_twin_ratelimit_launch", "af_twin_ratelimit_lean", "af_twin_ratelimit_sweep_fits"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep)]
        L.af_twin_rl_pass.restype = C.c_int
        L.af_twin_rl_pass.argtypes = [C.POINTER(C.c_double), C.c_double, C.c_double, C.c_double]
        _lib = L
    return _lib


@contextmanager
def _on(throttled: np.ndarray, lb_rate: float, lb_burst: int):
    L = lib()
    L.af_twin_ratelimit_set(throttled.ctypes.data, lb_rate, lb_burst)
    saved, twin_deadline._lib = twin_deadline._lib, L      # twin_deadline routes its calls through this library
    try:
        yield
    finally:
        twin_deadline._lib = saved
        L.af_twin_ratelimit_set(None, 0.0, 0)


def _run(fn, flat, kw: dict) -> dict:
    into = kw.get("into")
    n = kw.get("n", 1)
    thr = into["throttled"] if into is not None and "throttled" in into else np.zeros((n, flat.n_servers + 1), np.uint32)
    with _on(thr, float(flat.pod.lb_rate_limit), int(flat.pod.lb_burst)):
        out = fn(flat, **kw)
    out["throttled"] = thr
    return out


def run_lane(flat, **kw) -> dict:
    return _run(twin_deadline.run_lane, flat, kw)


def run_warp(flat, **kw) -> dict:
    return _run(twin_deadline.run_warp, flat, kw)


def run(flat, **kw) -> dict:
    return _run(twin_deadline.run, flat, kw)


# ---- the C checks -----------------------------------------------------------------------------------------------------
def _call(fn, flat, spec) -> bool:
    sw, keep = (None, None) if spec is None else spec.pod()
    ok = fn(C.byref(flat.pod), None if sw is None else C.byref(sw))
    del keep
    return bool(ok)


def ratelimit_launch(flat, spec=None) -> bool:
    """``afh::ratelimit_launch``: whether af_run lays out the token buckets and fills the throttle counts."""
    return _call(lib().af_twin_ratelimit_launch, flat, spec)


def lean_launch(flat, spec=None) -> bool:
    """``aflh::lean_launch`` without traces: whether af_run takes the lean lane build."""
    return _call(lib().af_twin_ratelimit_lean, flat, spec)


def validate(flat) -> str | None:
    """af_scenario_upload's check: ``None`` when accepted, else the engine's message."""
    return None if lib().af_twin_admission_validate(C.byref(flat.pod)) else lib().af_twin_error().decode()


def sweep_fits(flat, columns: list[tuple[int, int]], values) -> str | None:
    """af_sweep_upload's check of the rate-limit columns on ``flat``'s scenario: ``None`` when accepted, else the
    engine's message.  Takes raw (field, index) columns and a [rows, columns] table, so values SweepSpec refuses can
    reach it."""
    vals = np.ascontiguousarray(values, dtype=np.float64)
    cols = (K.AfSweepColumn * len(columns))(*[K.AfSweepColumn(f, i) for f, i in columns])
    sw = K.AfSweep()
    sw.n_columns, sw.n_rows = len(columns), vals.shape[0]
    sw.columns = C.cast(cols, C.POINTER(K.AfSweepColumn))
    sw.values = vals.ctypes.data_as(C.POINTER(C.c_double))
    ok = lib().af_twin_ratelimit_sweep_fits(C.byref(flat.pod), C.byref(sw))
    return None if ok else lib().af_twin_error().decode()


def rl_pass(tat: float, now: float, rate: float, burst: int) -> tuple[bool, float]:
    """The engines' GCRA rule on one request: (passed, the site's tat after it)."""
    t = C.c_double(tat)
    ok = lib().af_twin_rl_pass(C.byref(t), now, rate, float(burst))
    return bool(ok), t.value
