"""The CPU twin with admission limits (tests/host_twin/af_twin_admission.cpp) -- TEST INFRASTRUCTURE ONLY.

``run`` / ``run_lane`` / ``run_warp`` take what ``twin_streams``'s do and add ``rejected`` ([n, n_servers]: requests each
server shed) to the outputs; the limits come with the scenario (``flatten.set_admission``) and the sweep
(``("server_max_in_service", server_id)`` columns).  ``into=`` (a warp re-run) keeps writing ``into["rejected"]``.  Also
the C checks of the limits.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import twin
import twin_streams

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_admission.so"


def build() -> Path:
    sources = [_DIR / "af_twin_admission.cpp", _DIR / "af_twin_streams.cpp", _DIR / "af_twin_rows.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_admission.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    """The admission library, every af_twin_* function declared as ``twin_streams.lib()`` declares it."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        for name, f in vars(twin_streams.lib()).items():
            if name.startswith("af_twin_"):
                g = getattr(L, name)
                g.restype, g.argtypes = f.restype, f.argtypes
        L.af_twin_admission_set.restype = None
        L.af_twin_admission_set.argtypes = [C.c_void_p]
        L.af_twin_admission_launch.restype = C.c_int
        L.af_twin_admission_launch.argtypes = [C.POINTER(K.AfScenario), C.POINTER(K.AfSweep)]
        L.af_twin_admission_validate.restype = C.c_int
        L.af_twin_admission_validate.argtypes = [C.POINTER(K.AfScenario)]
        L.af_twin_admission_sweep_fits.restype = C.c_int
        L.af_twin_admission_sweep_fits.argtypes = [C.POINTER(K.AfSweep)]
        _lib = L
    return _lib


@contextmanager
def _on(rejected: np.ndarray):
    L = lib()
    L.af_twin_admission_set(rejected.ctypes.data)
    saved, twin_streams._lib = twin_streams._lib, L
    try:
        yield
    finally:
        twin_streams._lib = saved
        L.af_twin_admission_set(None)


def _run(fn, flat, kw: dict) -> dict:
    into = kw.get("into")
    rej = into["rejected"] if into is not None and "rejected" in into else np.zeros((kw.get("n", 1), flat.n_servers), np.uint32)
    with _on(rej):
        out = fn(flat, **kw)
    out["rejected"] = rej
    return out


def run_lane(flat, **kw) -> dict:
    return _run(twin_streams.run_lane, flat, kw)


def run_warp(flat, **kw) -> dict:
    return _run(twin_streams.run_warp, flat, kw)


def run(flat, **kw) -> dict:
    return _run(twin_streams.run, flat, kw)


# ---- the C checks -----------------------------------------------------------------------------------------------------
def admission_launch(flat, spec=None) -> bool:
    """``afh::admission_launch``: whether af_run lays out the admission words for this launch."""
    sw, keep = (None, None) if spec is None else spec.pod()
    ok = lib().af_twin_admission_launch(C.byref(flat.pod), None if sw is None else C.byref(sw))
    del keep
    return bool(ok)


def validate(flat) -> str | None:
    """af_scenario_upload's check: ``None`` when accepted, else the engine's message."""
    return None if lib().af_twin_admission_validate(C.byref(flat.pod)) else lib().af_twin_error().decode()


def sweep_fits(columns: list[tuple[int, int]], values) -> str | None:
    """af_sweep_upload's check of the admission columns: ``None`` when accepted, else the engine's message.  Takes raw
    (field, index) columns and a [rows, columns] table, so values SweepSpec refuses can reach it."""
    vals = np.ascontiguousarray(values, dtype=np.float64)
    cols = (K.AfSweepColumn * len(columns))(*[K.AfSweepColumn(f, i) for f, i in columns])
    sw = K.AfSweep()
    sw.n_columns, sw.n_rows = len(columns), vals.shape[0]
    sw.columns = C.cast(cols, C.POINTER(K.AfSweepColumn))
    sw.values = vals.ctypes.data_as(C.POINTER(C.c_double))
    ok = lib().af_twin_admission_sweep_fits(C.byref(sw))
    return None if ok else lib().af_twin_error().decode()

