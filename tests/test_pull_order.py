"""CPU tier: af_run hands replicas to lanes in a pull order (heaviest first by predicted work), not in id order.  A
replica's random numbers are keyed by its replica id and its outputs by its local index, so the order in which a lane
pulls them must not change one bit of any output: the state a replica leaves in the lane's shared memory and global
tier is reset when the next one starts, whichever that is.  Runs tests/host_twin/af_order_twin.cpp (compiled on first
use into a private temporary directory)."""

from __future__ import annotations

import atexit
import ctypes as C
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest
from helpers import PARITY_CASES, SEED, load_scenario

from asyncflow_b200 import SweepSpec, flatten
from asyncflow_b200 import _capi as K

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_order_twin.cpp"
_lib = None


def _twin() -> C.CDLL:
    global _lib
    if _lib is None:
        d = Path(tempfile.mkdtemp(prefix="af_order_twin_"))
        atexit.register(shutil.rmtree, d, True)
        so = d / "libaf_order_twin.so"
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                        str(_SRC)], check=True)
        L = C.CDLL(str(so))
        L.af_order_twin_error.restype = C.c_char_p
        L.af_order_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_order_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.c_uint64, C.POINTER(K.AfOptions), C.c_int32,
            C.c_uint64, C.c_uint64, C.c_uint64] + [C.c_void_p] * 11
        _lib = L
    return _lib


def _run(flat, *, n, order=None, seed=SEED, replica_begin=0, sweep=None, trace=0, clock_cap=0, lane_bytes=520,
         event_capacity=8192, request_capacity=400000) -> dict:
    L = _twin()
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    nser = flat.n_series
    tick_cap = L.af_order_twin_trace_tick_capacity(C.byref(flat.pod))
    out = {
        "stats": np.zeros(n, dtype=K.STATS_DTYPE),
        "sent": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "dropped": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "hist": np.zeros((n, K.AF_HIST_BINS), dtype=np.uint32),
        "thr": np.zeros((n, flat.horizon_s), dtype=np.uint32),
        "samp_sum": np.zeros((n, nser), dtype=np.uint64),
        "samp_max": np.zeros((n, nser), dtype=np.uint32),
        "trace_clocks": np.zeros((max(trace, 1), max(clock_cap, 1), 2), dtype=np.float64),
        "trace_series": np.zeros((max(trace, 1), nser, tick_cap), dtype=np.uint32),
        "trace_counts": np.zeros((n, 2), dtype=np.uint32),
    }
    sw_p, keep = None, None
    if sweep is not None:
        sw, keep = sweep.pod(0, None)
        sw_p = C.byref(sw)
    if order is not None:
        order = np.ascontiguousarray(order, dtype=np.uint32)
        assert order.shape == (n,) and np.array_equal(np.sort(order), np.arange(n))
    bufs = [out[k].ctypes.data for k in out]
    rc = L.af_order_twin_run_lane(C.byref(flat.pod), sw_p, 0, C.byref(opt), lane_bytes, seed, replica_begin, n,
                                  None if order is None else order.ctypes.data, *bufs)
    if rc != 0:
        raise RuntimeError(L.af_order_twin_error().decode())
    del keep
    return out


def _assert_same(got, ref):
    assert list(got) == list(ref)
    for k in ref:
        assert got[k].tobytes() == ref[k].tobytes(), k


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_random_pull_order_changes_no_output(name):
    flat = flatten(load_scenario(name, PARITY_CASES[name]))
    n = 5
    kw = dict(n=n, replica_begin=3, trace=2, clock_cap=300000)
    ref = _run(flat, **kw)
    _assert_same(_run(flat, order=np.random.default_rng(11).permutation(n), **kw), ref)


def test_pull_order_across_sweep_rows_with_different_splits():
    """Heavy and light rows of one sweep interleaved in the pull (each on its own split of the pool, some spilling both
    tables to the global tier): reversed order, same outputs."""
    flat = flatten(load_scenario("c1_my_service.yml", 4))
    users = np.array([5.0, 2000.0, 60.0, 900.0])
    spec = SweepSpec(flat, len(users), {("users_mean",): users})
    kw = dict(n=len(users), sweep=spec, trace=4, clock_cap=100000, lane_bytes=420, request_capacity=200000)
    ref = _run(flat, **kw)
    assert (ref["stats"]["flags"] == 0).all()
    assert ref["stats"]["completed"].min() > 0
    _assert_same(_run(flat, order=np.arange(len(users))[::-1], **kw), ref)
