"""The engine's state machine (af_core.cuh, compiled for the host as a one-lane warp)
against the oracle and the golden vectors -- CPU tier.  This checks the event
semantics of the code the CUDA kernel runs; the kernel itself is checked by
tests/test_gpu_*.py on an H100."""

from __future__ import annotations

import des_port
import numpy as np
import pytest
import twin
from helpers import (PARITY_CASES, SEED, assert_matches_oracle, check_against_golden, load_golden,
                     load_scenario)

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_twin_reproduces_golden_vectors(name):
    gold = load_golden(name)
    payload = load_scenario(name, gold["horizon"])
    flat = flatten(payload)
    for vec in gold["vectors"]:
        r = twin.run(flat, seed=gold["seed"], replica_begin=vec["replica"], n=1, trace=1, clock_cap=200000)
        st = r["stats"][0]
        n, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0
        check_against_golden(
            vec, generated=int(st["generated"]), completed=n, clocks=r["trace_clocks"][0, :n],
            edge_sent=dict(zip(flat.edge_ids, map(int, r["sent"][0]))),
            edge_dropped=dict(zip(flat.edge_ids, map(int, r["dropped"][0]))),
            throughput=r["thr"][0], series=r["trace_series"][0][:, :nt], flat=flat)


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("name", ["c1_my_service.yml", "c3_lb_two_servers.yml"])
def test_twin_reproduces_the_baseline_horizons(name, engine):
    """README my_service.yml at its 60 s, the LB example at its YAML's 600 s (76 656 completions, 60 000 collector ticks):
    both state machines against the unmodified reference actors (tests/golden/*_full.json, hash-pinned)."""
    gold = load_golden(name.replace(".yml", "_full.yml"))
    flat = flatten(load_scenario(name, gold["horizon"]))
    for vec in gold["vectors"]:
        r = twin.run(flat, seed=gold["seed"], replica_begin=vec["replica"], n=1, trace=1, clock_cap=200000, engine=engine)
        st = r["stats"][0]
        n, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0
        check_against_golden(
            vec, generated=int(st["generated"]), completed=n, clocks=r["trace_clocks"][0, :n],
            edge_sent=dict(zip(flat.edge_ids, map(int, r["sent"][0]))),
            edge_dropped=dict(zip(flat.edge_ids, map(int, r["dropped"][0]))),
            throughput=r["thr"][0], series=r["trace_series"][0][:, :nt], flat=flat)


@pytest.mark.parametrize("name", ["c1_my_service.yml", "mixed_lc.yml", "poisson_ties.yml", "overload_single.yml"])
def test_twin_matches_oracle_including_aggregates(name):
    payload = load_scenario(name, 10 if name.startswith("c1") else None)
    flat = flatten(payload)
    reps = [2, 3, 4]
    r = twin.run(flat, seed=SEED, replica_begin=reps[0], n=len(reps), trace=len(reps), clock_cap=50000)
    for i, rep in enumerate(reps):
        o = des_port.simulate(payload, seed=SEED, replica=rep)
        st = r["stats"][i]
        n, nt = int(st["completed"]), int(st["n_ticks"])
        assert_matches_oracle(o, flat, stats=st, clocks=r["trace_clocks"][i, :n], sent=r["sent"][i],
                              dropped=r["dropped"][i], series=r["trace_series"][i][:, :nt],
                              throughput=r["thr"][i], hist=r["hist"][i])
        ser = r["trace_series"][i][:, :nt].astype(np.uint64)
        np.testing.assert_array_equal(r["samp_sum"][i], ser.sum(axis=1))
        np.testing.assert_array_equal(r["samp_max"][i], ser.max(axis=1) if nt else 0)


def test_sweep_rows_override_the_scenario():
    base = load_scenario("c1_my_service.yml", 8)
    flat = flatten(base)
    users = [20.0, 150.0, 400.0]
    spec = SweepSpec(flat, 3, {("users_mean",): users, ("edge_mean", "client-app"): [0.001, 0.01, 0.02],
                               ("server_cpu_cores", "app-1"): [1, 2, 4],
                               ("endpoint_ram", "app-1", 0): [120, 300, 64],
                               ("step_duration", "app-1", 0, 2): [0.012, 0.001, 0.05]})
    r = twin.run(flat, seed=SEED, replica_begin=0, n=3, sweep=spec, trace=3, clock_cap=60000)
    for i in range(3):
        p = load_scenario("c1_my_service.yml", 8)
        p["rqs_input"]["avg_active_users"]["mean"] = users[i]
        p["topology_graph"]["edges"][1]["latency"]["mean"] = [0.001, 0.01, 0.02][i]
        srv = p["topology_graph"]["nodes"]["servers"][0]
        srv["server_resources"]["cpu_cores"] = [1, 2, 4][i]
        srv["endpoints"][0]["steps"][1]["step_operation"]["necessary_ram"] = [120, 300, 64][i]
        srv["endpoints"][0]["steps"][2]["step_operation"]["io_waiting_time"] = [0.012, 0.001, 0.05][i]
        o = des_port.simulate(p, seed=SEED, replica=i)
        n = int(r["stats"][i]["completed"])
        assert_matches_oracle(o, flat, stats=r["stats"][i], clocks=r["trace_clocks"][i, :n],
                              sent=r["sent"][i], dropped=r["dropped"][i])


def test_capacity_overflow_is_flagged_not_silent():
    flat = flatten(load_scenario("overload_single.yml"))
    r = twin.run(flat, seed=SEED, n=1, request_capacity=200)
    assert r["stats"][0]["flags"] & K.FLAG_REQUEST_OVERFLOW
    r = twin.run(flat, seed=SEED, n=1, event_capacity=4)
    assert r["stats"][0]["flags"] & K.FLAG_EVENT_OVERFLOW
    r = twin.run(flat, seed=SEED, n=1, trace=1, clock_cap=10)
    assert r["stats"][0]["flags"] & K.FLAG_TRACE_TRUNCATED


def test_spill_tier_gives_the_same_answer_as_the_fast_tier():
    """peak in-flight requests (~4000) far exceed the 64 shared-memory slots."""
    payload = load_scenario("overload_single.yml")
    flat = flatten(payload)
    r = twin.run(flat, seed=SEED, replica_begin=5, n=1, trace=1, clock_cap=20000)
    assert r["stats"][0]["peak_requests"] > 1000
    o = des_port.simulate(payload, seed=SEED, replica=5)
    n = int(r["stats"][0]["completed"])
    assert_matches_oracle(o, flat, stats=r["stats"][0], clocks=r["trace_clocks"][0, :n],
                          sent=r["sent"][0], dropped=r["dropped"][0])


def test_histogram_percentile_matches_numpy_within_two_percent():
    rng = np.random.default_rng(3)
    lat = rng.lognormal(-3.5, 0.6, size=20000)
    bits = lat.view(np.uint64)
    idx = (bits >> np.uint64(52 - K.AF_HIST_SUB_BITS)).astype(np.int64) - ((1023 + K.AF_HIST_MIN_EXP) << K.AF_HIST_SUB_BITS)
    hist = np.bincount(np.clip(idx, 0, K.AF_HIST_BINS - 1), minlength=K.AF_HIST_BINS).astype(np.uint32)
    for q in (50.0, 95.0, 99.0):
        got = twin.lib().af_twin_hist_percentile(hist.ctypes.data, len(lat), q, lat.min(), lat.max())
        exact = float(np.percentile(lat, q))
        assert abs(got - exact) < 0.01 * exact


def test_partial_metric_sets_follow_the_collector_rule():
    """collector.py:60-66: server series are recorded only if ALL THREE are enabled; edges on their own."""
    payload = load_scenario("c1_my_service.yml", 6)
    payload["sim_settings"]["enabled_sample_metrics"] = ["ram_in_use", "edge_concurrent_connection"]
    flat = flatten(payload)
    o = des_port.simulate(payload, seed=SEED, replica=3)
    r = twin.run(flat, seed=SEED, replica_begin=3, n=1, trace=1, clock_cap=20000)
    st = r["stats"][0]
    n, nt = int(st["completed"]), int(st["n_ticks"])
    np.testing.assert_array_equal(r["trace_clocks"][0, :n], np.array(o["clocks"]).reshape(-1, 2))
    assert o["server_series"]["app-1"] == {"ram_in_use": []}
    assert (r["samp_sum"][0][:3] == 0).all()                       # the server triple is off
    conn = np.array(o["edge_series"]["gen-client"]["edge_concurrent_connection"], dtype=np.uint32)
    assert nt == len(conn)
    np.testing.assert_array_equal(r["trace_series"][0][3, :nt], conn)
