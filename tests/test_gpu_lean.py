"""GPU tier: the lean lane kernel (af_lane_kernel<*, *, true>) gives the same outputs as the full one
(ASYNCFLOW_B200_LANE_FULL=1) bit for bit -- statistics, edge counters, sampled aggregates, histograms, throughput, per-tick
and latency bands -- in every pass structure that runs the lane kernel, and af_run reports lane_lean = 1 exactly when
the launch qualifies."""

from __future__ import annotations

import numpy as np
import pytest
from helpers import SEED, load_scenario
from test_lean_lane import SCENARIOS, scenario

from asyncflow_b200 import Engine, SweepSpec, flatten

pytestmark = pytest.mark.gpu

N = 13_000          # AUTO runs the lane kernel from 3 x SMs x 32 replicas (12 672 on an H100)
G = 5


def _run(flat, spec, mode, bands, *, trace=0):
    with Engine(0) as eng:
        eng.upload(flat)
        eng.set_mode(mode)
        eng.configure(trace_replicas=trace, trace_clock_capacity=1000 if trace else 0)
        eng.upload_sweep(spec, 0)
        if bands:
            eng.configure_bands(sampled=True, latency_window_s=2)
            eng.upload_bands((np.arange(N) % G).astype(np.uint32), 0, G)
        eng.run(SEED, 0, N)
        out = {"stats": eng.stats(), "edges": eng.edge_counts(), "sampled": eng.sampled(), "hist": eng.histograms(),
               "thr": eng.throughput()}
        if bands:
            out["bands"] = eng.bands()
            out["lat"] = eng.latency_bands()
        return eng.last_run_passes(), out


def _flat(arrays):
    if isinstance(arrays, tuple):
        return [a for x in arrays for a in _flat(x)]
    return [arrays]


def _assert_lean_equals_full(flat, spec, mode, bands, monkeypatch):
    monkeypatch.delenv("ASYNCFLOW_B200_LANE_FULL", raising=False)
    p_lean, lean = _run(flat, spec, mode, bands)
    monkeypatch.setenv("ASYNCFLOW_B200_LANE_FULL", "1")
    p_full, full = _run(flat, spec, mode, bands)
    monkeypatch.delenv("ASYNCFLOW_B200_LANE_FULL")
    assert p_lean["lane_pass"] == 1 and p_lean["lane_lean"] == 1, p_lean
    assert p_full["lane_pass"] == 1 and p_full["lane_lean"] == 0, p_full
    assert lean["stats"]["completed"].sum() > 0
    for k, v in full.items():
        for a, b in zip(_flat(v), _flat(lean[k])):
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (k, mode, bands)


def _users_sweep(flat):
    rng = np.random.default_rng(11)
    return SweepSpec(flat, N, {("users_mean",): rng.choice([10.0, 40.0, 120.0], N)})


@pytest.mark.parametrize("mode", ["auto", "lane", "two_pass"])
@pytest.mark.parametrize("name", SCENARIOS)
def test_lean_kernel_equals_full_kernel(name, mode, monkeypatch):
    payload = scenario(name)
    payload["sim_settings"]["total_simulation_time"] = 10
    flat = flatten(payload)
    spec = _users_sweep(flat)
    _assert_lean_equals_full(flat, spec, mode, False, monkeypatch)
    _assert_lean_equals_full(flat, spec, mode, True, monkeypatch)


@pytest.mark.parametrize("mode", ["auto", "lane", "two_pass"])
def test_lean_kernel_equals_full_kernel_on_bench_sweep_rows(mode, monkeypatch):
    import bench
    flat = flatten(bench.workload(0, 6))
    ids = np.arange(N, dtype=np.int64) * 7
    spec = SweepSpec(flat, N, bench._c3_cols(flat, ids, 100_000))
    _assert_lean_equals_full(flat, spec, mode, False, monkeypatch)
    _assert_lean_equals_full(flat, spec, mode, True, monkeypatch)


def test_lane_lean_reported_only_when_the_launch_qualifies(monkeypatch):
    monkeypatch.delenv("ASYNCFLOW_B200_LANE_FULL", raising=False)
    for name, trace in (("ev_spikes_outages.yml", 0), ("c5_multihop32.yml", 0), ("mixed_lc.yml", 0),
                        ("c1_my_service.yml", 2), ("tie_cpu_io.yml", 0)):
        payload = load_scenario(name)
        payload["sim_settings"]["total_simulation_time"] = 5
        flat = flatten(payload)
        p, _ = _run(flat, _users_sweep(flat), "lane", False, trace=trace)
        assert p["lane_pass"] == 1 and p["lane_lean"] == 0, (name, p)
    payload = load_scenario("c1_my_service.yml", 5)
    flat = flatten(payload)
    p, _ = _run(flat, _users_sweep(flat), "warp", False)
    assert p["lane_pass"] == 0 and p["lane_lean"] == 0, p
    p, _ = _run(flat, _users_sweep(flat), "lane", False)
    assert p["lane_lean"] == 1, p
