"""CPU tier: the lean build of the lane engine's loop (run_lane<*, *, true>: no spikes, outages, traces, general edge
samplers or endpoint draws) gives the same outputs as the full build, bit for bit, on every launch that qualifies for it
(aflh::lean_launch) -- with per-replica pool splits, sweeps and both kinds of bands -- and the qualification rule
rejects each feature the lean loop leaves out."""

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

_SRC = Path(__file__).resolve().parent / "host_twin" / "af_lean_twin.cpp"
_lib = None
OUTPUTS = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "trace_clocks", "trace_series",
           "trace_counts")
#: scenarios -> whether they qualify as written; the others run as one_endpoint() makes them
SCENARIOS = {"c3_lb_two_servers.yml": True, "c1_my_service.yml": True, "chain_two_servers.yml": True,
             "tie_cpu_io.yml": False, "poisson_ties.yml": False, "overload_single.yml": False}
BANDS = ((False, False), (True, False), (False, True), (True, True))    # (per-tick bands, latency bands)


def one_endpoint(payload: dict) -> dict:
    """The scenario with each server's last endpoint only and every edge without a normal / exponential latency made
    exponential with the same mean: what the lean loop can run.  tie_cpu_io, poisson_ties and overload_single keep
    their one- and two-core servers under load -- CPU and RAM waiter queues, now-queue ties."""
    for s in payload["topology_graph"]["nodes"]["servers"]:
        s["endpoints"] = s["endpoints"][-1:]
    for e in payload["topology_graph"]["edges"]:
        if e["latency"].get("distribution") not in ("normal", "exponential"):
            e["latency"] = {"mean": e["latency"]["mean"], "distribution": "exponential"}
    return payload


def scenario(name: str) -> dict:
    h = PARITY_CASES.get(name)
    payload = load_scenario(name, min(h, 30) if h else None)
    return payload if SCENARIOS[name] else one_endpoint(payload)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        d = Path(tempfile.mkdtemp(prefix="af_lean_twin_"))
        atexit.register(shutil.rmtree, d, True)
        so = d / "libaf_lean_twin.so"
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", str(so),
                        str(_SRC)], check=True)
        L = C.CDLL(str(so))
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
        L.af_lean_twin_error.restype = C.c_char_p
        L.af_lean_twin_trace_tick_capacity.argtypes = [C.POINTER(K.AfScenario)]
        L.af_lean_twin_ticks.argtypes = [C.POINTER(K.AfScenario)]
        L.af_lean_twin_ticks.restype = u32
        L.af_lean_twin_qualifies.argtypes = [C.POINTER(K.AfScenario), i32]
        L.af_lean_twin_run_lane.argtypes = [
            C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions), i32, i32, u64, u64, u64, u64,
            i32, i32, i32, vp, u64, u64, u32, vp, vp, vp, vp] + [vp] * 10
        _lib = L
    return _lib


def qualifies(flat, trace_replicas: int = 0) -> bool:
    return bool(lib().af_lean_twin_qualifies(C.byref(flat.pod), trace_replicas))


def run_lane(flat, *, lean: bool, n: int, sweep=None, split: int = 0, sampled: bool = False, window: int = 0,
             lane_bytes: int = 604) -> dict:
    """The thread-per-replica engine over replicas [0, n) in groups i % 3: ``split`` 0 = every replica on the
    scenario's estimate, 1 = each sweep row on its own, 2 = a random split per replica."""
    L = lib()
    opt = K.AfOptions(2048, 16384, 0, 0, 1, 1, 0, 0)
    ticks = int(L.af_lean_twin_ticks(C.byref(flat.pod)))
    tick_cap = L.af_lean_twin_trace_tick_capacity(C.byref(flat.pod))
    n_groups = 3
    windows = -(-int(flat.horizon_s) // window) if window else 1
    out = {
        "stats": np.zeros(n, dtype=K.STATS_DTYPE),
        "sent": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "dropped": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "hist": np.zeros((n, K.AF_HIST_BINS), dtype=np.uint32),
        "thr": np.zeros((n, flat.horizon_s), dtype=np.uint32),
        "samp_sum": np.zeros((n, flat.n_series), dtype=np.uint64),
        "samp_max": np.zeros((n, flat.n_series), dtype=np.uint32),
        "trace_clocks": np.zeros((1, 1, 2), dtype=np.float64),
        "trace_series": np.zeros((1, flat.n_series, tick_cap), dtype=np.uint32),
        "trace_counts": np.zeros((n, 2), dtype=np.uint32),
        "band_rows": np.zeros((n_groups + 1, 1 + 2 * flat.n_series, ticks + 1), dtype=np.uint64),
        "band_from": np.full(n, 0xFFFFFFFF, dtype=np.uint32),
        "lat_rows": np.zeros((n_groups + 1, windows, K.AF_HIST_BINS + 2), dtype=np.uint64),
        "lat_from": np.full(n, 0xFFFFFFFF, dtype=np.uint32),
    }
    groups = np.ascontiguousarray(np.arange(n) % n_groups, dtype=np.uint32)
    sw_p, keep = None, None
    if sweep is not None:
        sw, keep = sweep.pod(0, None)
        sw_p = C.byref(sw)
    rc = L.af_lean_twin_run_lane(C.byref(flat.pod), sw_p, C.byref(opt), lane_bytes, split, 7, SEED, 0, n, int(lean),
                                 int(sampled), int(window), groups.ctypes.data, 0, n, n_groups,
                                 out["band_rows"].ctypes.data, out["band_from"].ctypes.data,
                                 out["lat_rows"].ctypes.data, out["lat_from"].ctypes.data,
                                 *[out[k].ctypes.data for k in OUTPUTS])
    if rc != 0:
        raise RuntimeError(L.af_lean_twin_error().decode())
    del keep
    return out


def assert_lean_equals_full(flat, **kw) -> dict:
    lean, full = run_lane(flat, lean=True, **kw), run_lane(flat, lean=False, **kw)
    for k, v in full.items():
        assert v.tobytes() == lean[k].tobytes(), (k, kw)
    return lean


@pytest.mark.parametrize("name", SCENARIOS)
def test_lean_loop_equals_full_loop(name):
    """Every scenario, every band combination, the scenario's split and random per-replica splits."""
    assert qualifies(flatten(load_scenario(name))) == SCENARIOS[name]
    flat = flatten(scenario(name))
    assert qualifies(flat)
    for sampled, lat in BANDS:
        for split in (0, 2):
            out = assert_lean_equals_full(flat, n=6, split=split, sampled=sampled, window=2 if lat else 0)
            assert out["stats"]["completed"].sum() > 0


def test_lean_loop_equals_full_loop_on_bench_sweep_rows():
    """configs[2]'s shape (normal-jitter edges) on rows of the bench's own RTT x jitter grid, each replica split by
    its row's estimate as af_run does, at the bench's per-lane budget (604 B at 12 warps/SM)."""
    import bench
    flat = flatten(bench.workload(0, 6))
    assert qualifies(flat)
    ids = np.linspace(0, 99_999, 24).astype(np.int64)
    spec = SweepSpec(flat, ids.size, bench._c3_cols(flat, ids, 100_000))
    for sampled, lat in BANDS:
        out = assert_lean_equals_full(flat, n=ids.size, sweep=spec, split=1, sampled=sampled, window=1 if lat else 0)
        assert (out["stats"]["completed"] > 0).all()


def test_qualification_rejects_every_feature_the_lean_loop_leaves_out():
    """Spikes and outages, a lognormal (general-sampler) edge, traced replicas, servers with two endpoints."""
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    assert flat.pod.n_spike_marks > 0 or flat.pod.n_outage_marks > 0
    assert not qualifies(flat)
    payload = load_scenario("c1_my_service.yml", 10)
    assert qualifies(flatten(payload)) and not qualifies(flatten(payload), trace_replicas=1)
    payload["topology_graph"]["edges"][1]["latency"] = {"mean": 0.003, "distribution": "log_normal", "variance": 0.001}
    assert not qualifies(flatten(payload))
    for name in ("c5_multihop32.yml", "mixed_lc.yml"):
        flat = flatten(load_scenario(name))
        assert any(flat.pod.servers[i].n_endpoints > 1 for i in range(flat.pod.n_servers)), name
        assert not qualifies(flat), name
    assert not qualifies(flatten(load_scenario("c4_lb8_events.yml")))
