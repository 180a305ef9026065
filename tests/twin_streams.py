"""The CPU twin with timeline rows and random streams (tests/host_twin/af_twin_streams.cpp) -- TEST INFRASTRUCTURE ONLY.

``run`` / ``run_lane`` / ``run_warp`` take what ``twin_rows``'s do, plus ``streams``: the stream of replicas
``stream_first, stream_first + 1, ...`` (af_streams_upload's table; ``None``: every replica draws as its id).  The launch
itself is ``twin``'s, on a library that is af_twin_rows.cpp plus the table.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import twin
import twin_rows

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin_streams.so"


def build() -> Path:
    sources = [_DIR / "af_twin_streams.cpp", _DIR / "af_twin_rows.cpp", *twin._SRC]
    if not _SO.exists() or _SO.stat().st_mtime < max(p.stat().st_mtime for p in sources):
        _SO.parent.mkdir(exist_ok=True)
        tmp = _SO.with_name(f"{_SO.name}.{os.getpid()}")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
                        "-o", str(tmp), str(_DIR / "af_twin_streams.cpp")], check=True)
        tmp.replace(_SO)
    return _SO


_lib = None


def lib() -> C.CDLL:
    """The streams library, every af_twin_* function declared as ``twin_rows.lib()`` declares it."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        for name, f in vars(twin_rows.lib()).items():
            if name.startswith("af_twin_"):
                g = getattr(L, name)
                g.restype, g.argtypes = f.restype, f.argtypes
        L.af_twin_streams_set.restype = None
        L.af_twin_streams_set.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
        _lib = L
    return _lib


@contextmanager
def rows(flat, sweep=None, sweep_first: int = 0, timeline=None, timeline_first: int = 0, timeline_rows=None,
         streams=None, stream_first: int = 0):
    """Inside the block, ``twin``'s launches (and whatever calls them, such as ``TwinEngine``) run on the streams
    library with these timeline rows (``twin_rows.rows``) and this stream table set."""
    L = lib()
    table = None if streams is None else np.ascontiguousarray(streams, dtype=np.uint64)
    L.af_twin_streams_set(None if table is None else table.ctypes.data, 0 if table is None else table.size,
                          int(stream_first))
    saved, twin_rows._lib = twin_rows._lib, L
    try:
        with twin_rows.rows(flat, sweep, sweep_first, timeline, timeline_first, timeline_rows):
            yield
    finally:
        twin_rows._lib = saved
        L.af_twin_streams_set(None, 0, 0)


def _kw(kw: dict) -> tuple:
    return (kw.get("sweep"), kw.get("sweep_first", 0), kw.pop("timeline", None), kw.pop("timeline_first", 0),
            kw.pop("timeline_rows", None), kw.pop("streams", None), kw.pop("stream_first", 0))


def run_lane(flat, **kw) -> dict:
    with rows(flat, *_kw(kw)):
        return twin.run_lane(flat, **kw)


def run_warp(flat, **kw) -> dict:
    with rows(flat, *_kw(kw)):
        return twin.run_warp(flat, **kw)


def run(flat, **kw) -> dict:
    with rows(flat, *_kw(kw)):
        return twin.run(flat, **kw)
