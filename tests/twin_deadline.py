"""The CPU twin with request deadlines and a client timeout (tests/host_twin/af_twin_deadline.cpp) -- TEST
INFRASTRUCTURE ONLY.

``run`` / ``run_lane`` / ``run_warp`` take what ``twin_admission``'s do and add ``expired`` ([n, n_servers]: requests
each server dropped past its deadline) and ``late`` ([n]: completions later than the client timeout) to the outputs;
the values come with the scenario (``flatten.set_deadlines``) and the sweep (``("server_deadline", server_id)`` /
``("client_timeout",)`` columns).  ``into=`` (a warp re-run) keeps writing ``into["expired"]`` / ``into["late"]``.
Also the C checks.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import twin
import twin_admission

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_deadline.so"


def build() -> Path:
    sources = [_DIR / "af_twin_deadline.cpp", _DIR / "af_twin_admission.cpp", _DIR / "af_twin_streams.cpp",
               _DIR / "af_twin_rows.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_deadline.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    """The deadline library, every af_twin_* function declared as ``twin_admission.lib()`` declares it."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        for name, f in vars(twin_admission.lib()).items():
            if name.startswith("af_twin_"):
                g = getattr(L, name)
                g.restype, g.argtypes = f.restype, f.argtypes
        L.af_twin_deadline_set.restype = None
        L.af_twin_deadline_set.argtypes = [C.c_void_p, C.c_void_p, C.c_double]
        for name in ("af_twin_deadline_launch", "af_twin_deadline_lean"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep)]
        L.af_twin_deadline_sweep_fits.restype = C.c_int
        L.af_twin_deadline_sweep_fits.argtypes = [C.POINTER(K.AfSweep)]
        _lib = L
    return _lib


@contextmanager
def _on(expired: np.ndarray, late: np.ndarray, client_timeout: float):
    L = lib()
    L.af_twin_deadline_set(expired.ctypes.data, late.ctypes.data, client_timeout)
    saved, twin_admission._lib = twin_admission._lib, L      # twin_admission routes its calls through this library
    try:
        yield
    finally:
        twin_admission._lib = saved
        L.af_twin_deadline_set(None, None, 0.0)


def _run(fn, flat, kw: dict) -> dict:
    into = kw.get("into")
    n = kw.get("n", 1)
    exp = into["expired"] if into is not None and "expired" in into else np.zeros((n, flat.n_servers), np.uint32)
    late = into["late"] if into is not None and "late" in into else np.zeros(n, np.uint32)
    with _on(exp, late, float(flat.pod.client_timeout)):
        out = fn(flat, **kw)
    out["expired"], out["late"] = exp, late
    return out


def run_lane(flat, **kw) -> dict:
    return _run(twin_admission.run_lane, flat, kw)


def run_warp(flat, **kw) -> dict:
    return _run(twin_admission.run_warp, flat, kw)


def run(flat, **kw) -> dict:
    return _run(twin_admission.run, flat, kw)


# ---- the C checks -----------------------------------------------------------------------------------------------------
def _call(fn, flat, spec) -> bool:
    sw, keep = (None, None) if spec is None else spec.pod()
    ok = fn(C.byref(flat.pod), None if sw is None else C.byref(sw))
    del keep
    return bool(ok)


def deadline_launch(flat, spec=None) -> bool:
    """``afh::deadline_launch``: whether af_run lays out the deadline words and fills the expiry / late outputs."""
    return _call(lib().af_twin_deadline_launch, flat, spec)


def lean_launch(flat, spec=None) -> bool:
    """``aflh::lean_launch`` without traces: whether af_run takes the lean lane build."""
    return _call(lib().af_twin_deadline_lean, flat, spec)


def validate(flat) -> str | None:
    """af_scenario_upload's check: ``None`` when accepted, else the engine's message."""
    return None if lib().af_twin_admission_validate(C.byref(flat.pod)) else lib().af_twin_error().decode()


def sweep_fits(columns: list[tuple[int, int]], values) -> str | None:
    """af_sweep_upload's check of the deadline columns: ``None`` when accepted, else the engine's message.  Takes raw
    (field, index) columns and a [rows, columns] table, so values SweepSpec refuses can reach it."""
    vals = np.ascontiguousarray(values, dtype=np.float64)
    cols = (K.AfSweepColumn * len(columns))(*[K.AfSweepColumn(f, i) for f, i in columns])
    sw = K.AfSweep()
    sw.n_columns, sw.n_rows = len(columns), vals.shape[0]
    sw.columns = C.cast(cols, C.POINTER(K.AfSweepColumn))
    sw.values = vals.ctypes.data_as(C.POINTER(C.c_double))
    ok = lib().af_twin_deadline_sweep_fits(C.byref(sw))
    return None if ok else lib().af_twin_error().decode()
