"""CPU tier: per-replica percentiles whose order statistics fall into one of the latency histogram's two end bins.

The histogram covers [2^-20, 2^12) s and clamps every latency outside it into its first or last bin.  A replica's
p50 / p95 / p99 read such a bin over [min(edge(0), lat_min), edge(1)) or [edge(B-1), max(edge(B), lat_max)], its exact
extremes: an overloaded replica on a horizon past 4096 s reports its tail, not the last bin's 4096 s.  The twin runs
the host definition (afh::hist_percentile); results.hist_percentiles with lo= / hi= is the same arithmetic."""

from __future__ import annotations

import numpy as np
import pytest
import twin
from helpers import SEED, load_scenario

from asyncflow_b200 import _capi as K
from asyncflow_b200 import flatten
from asyncflow_b200.results import hist_percentiles

QS = ((50.0, "p50"), (95.0, "p95"), (99.0, "p99"))
TOP = 2.0 ** (K.AF_HIST_MIN_EXP + K.AF_HIST_BINS // (1 << K.AF_HIST_SUB_BITS))     # 4096 s: the last bin's upper edge
BOTTOM = 2.0 ** K.AF_HIST_MIN_EXP


def overload_payload(horizon: int, users: float) -> dict:
    """overload_single.yml slowed to ~3 completions/s against ~13 arrivals/s: latencies grow with the run's length
    and pass 4096 s on horizons of about 7000 s and more."""
    p = load_scenario("overload_single.yml", horizon)
    p["rqs_input"]["avg_active_users"]["mean"] = users
    for ep in p["topology_graph"]["nodes"]["servers"][0]["endpoints"]:
        for st in ep["steps"]:
            if st["kind"] == "io_db":
                st["step_operation"]["io_waiting_time"] = 0.4
    p["sim_settings"]["sample_period_s"] = 1
    return p


#: (horizon s, users, replica): every one of them ends with latencies past 4096 s
LONG_CASES = [(9000, 8, 0), (9000, 8, 1), (7000, 6, 0)]
LONG_KW = dict(request_capacity=1 << 18, clock_cap=40_000)


def bin_of(lat: np.ndarray) -> np.ndarray:
    idx = (lat.view(np.uint64) >> np.uint64(52 - K.AF_HIST_SUB_BITS)).astype(np.int64) \
        - ((1023 + K.AF_HIST_MIN_EXP) << K.AF_HIST_SUB_BITS)
    return np.clip(idx, 0, K.AF_HIST_BINS - 1)


def twin_percentile(hist: np.ndarray, n: int, q: float, lo: float, hi: float) -> float:
    h = np.ascontiguousarray(hist, dtype=np.uint32)
    return float(twin.lib().af_twin_hist_percentile(h.ctypes.data, n, q, lo, hi))


def assert_percentiles(st, hist: np.ndarray, lat: np.ndarray) -> None:
    """st's p50/p95/p99: within 1 % of numpy's on the exact latencies, inside [lat_min, lat_max], and the bytes of both
    host definitions on (hist, completed, lat_min, lat_max)."""
    n = int(st["completed"])
    assert n == len(lat) == int(hist.sum()) and n > 0
    assert float(st["lat_min"]) == float(lat.min()) and float(st["lat_max"]) == float(lat.max())
    for q, key in QS:
        got, exact = float(st[key]), float(np.percentile(lat, q))
        assert abs(got - exact) <= 0.01 * exact, (key, got, exact)
        assert float(st["lat_min"]) <= got <= float(st["lat_max"]), (key, got)
        want = twin_percentile(hist, n, q, float(st["lat_min"]), float(st["lat_max"]))
        assert np.float64(got).tobytes() == np.float64(want).tobytes(), (key, got, want)
        py = hist_percentiles(hist, q, lo=np.float64(st["lat_min"]), hi=np.float64(st["lat_max"]))
        assert np.float64(got).tobytes() == np.float64(py).tobytes(), (key, got, float(py))


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("horizon,users,replica", LONG_CASES)
def test_percentiles_past_the_last_bin_follow_the_exact_latencies(engine, horizon, users, replica):
    flat = flatten(overload_payload(horizon, users))
    r = twin.run(flat, engine=engine, seed=SEED, replica_begin=replica, n=1, trace=1, **LONG_KW)
    st = r["stats"][0]
    assert st["flags"] == 0
    n = int(st["completed"])
    clocks = r["trace_clocks"][0, :n]
    lat = clocks[:, 1] - clocks[:, 0]
    assert lat.max() > TOP and int(r["hist"][0, -1]) > 0.01 * n        # the tail really is clamped into the last bin
    assert_percentiles(st, r["hist"][0], lat)


def test_both_state_machines_give_the_same_long_horizon_percentiles():
    flat = flatten(overload_payload(9000, 8))
    lane = twin.run(flat, engine="lane", seed=SEED, n=2, **LONG_KW)
    warp = twin.run(flat, engine="warp", seed=SEED, n=2, **LONG_KW)
    assert lane["stats"].tobytes() == warp["stats"].tobytes()
    assert lane["hist"].tobytes() == warp["hist"].tobytes()


def tiny_payload() -> dict:
    """Every edge and step well under a microsecond: the schema only asks for positive values, and most latencies
    fall below 2^-20 s, into the histogram's first bin."""
    p = load_scenario("c1_my_service.yml", 3)
    for e in p["topology_graph"]["edges"]:
        e["latency"] = {"mean": 2e-7, "distribution": "exponential"}
    for ep in p["topology_graph"]["nodes"]["servers"][0]["endpoints"]:
        for st in ep["steps"]:
            op = next(iter(st["step_operation"]))
            if op != "necessary_ram":
                st["step_operation"][op] = 1e-7
    return p


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_percentiles_below_the_first_bin_stay_inside_the_replica_range(engine):
    """Sub-microsecond latencies: an order statistic in bin 0 is read over [lat_min, edge(1)), not [2^-20, edge(1)),
    so a p50 below 2^-20 s is reported below 2^-20 s.  (Bin 0's contents are not uniform here, so the 1 % bound of the
    long-horizon cases does not apply.)"""
    flat = flatten(tiny_payload())
    r = twin.run(flat, engine=engine, seed=SEED, replica_begin=3, n=1, trace=1, clock_cap=20_000)
    st = r["stats"][0]
    assert st["flags"] == 0
    n = int(st["completed"])
    clocks = r["trace_clocks"][0, :n]
    lat = clocks[:, 1] - clocks[:, 0]
    edge1 = BOTTOM * (1 + 2.0 ** -K.AF_HIST_SUB_BITS)
    assert n > 100 and lat.min() < BOTTOM and np.percentile(lat, 50) < BOTTOM
    for q, key in QS:
        got = float(st[key])
        want = twin_percentile(r["hist"][0], n, q, float(st["lat_min"]), float(st["lat_max"]))
        py = hist_percentiles(r["hist"][0], q, lo=np.float64(st["lat_min"]), hi=np.float64(st["lat_max"]))
        assert np.float64(got).tobytes() == np.float64(want).tobytes() == np.float64(py).tobytes(), key
        if np.percentile(lat, q) < BOTTOM:
            assert float(st["lat_min"]) <= got < edge1, (key, got)
    assert float(st["p50"]) < BOTTOM


def hist_of(lat: np.ndarray) -> np.ndarray:
    return np.bincount(bin_of(lat), minlength=K.AF_HIST_BINS).astype(np.uint32)


def test_end_bin_rule_on_synthetic_histograms():
    """Latencies spread evenly over each end bin's open side: both host definitions agree bit for bit and are within
    1 % of numpy; histograms inside [2^-20, 2^12) s keep the bits of the plain bin edges."""
    rng = np.random.default_rng(17)
    cases = {
        "below": rng.uniform(4e-7, BOTTOM, 200_000),
        "above": rng.uniform(TOP, 9000.0, 200_000),
        "both": np.concatenate([rng.uniform(2e-7, BOTTOM, 100_000), rng.lognormal(-3, 1, 100_000),
                                rng.uniform(TOP, 6000.0, 400_000)]),
        "inside": rng.lognormal(-3.5, 0.6, 20_000),
    }
    rows = np.stack([hist_of(lat) for lat in cases.values()])
    lo = np.array([lat.min() for lat in cases.values()])
    hi = np.array([lat.max() for lat in cases.values()])
    for q in (1.0, 50.0, 95.0, 99.0, 99.9):             # "both": p1 in bin 0, p50 and up in the last bin
        got = hist_percentiles(rows, q, lo=lo, hi=hi)
        plain = hist_percentiles(rows, q)
        for i, (name, lat) in enumerate(cases.items()):
            want = twin_percentile(rows[i], len(lat), q, lo[i], hi[i])
            assert got[i].tobytes() == np.float64(want).tobytes(), (name, q)
            exact = float(np.percentile(lat, q))
            assert abs(got[i] - exact) <= 0.01 * exact, (name, q, got[i], exact)
            if name == "inside":
                assert got[i].tobytes() == plain[i].tobytes()
            elif q == 50.0:
                assert abs(plain[i] - exact) > 0.1 * exact, (name, q)        # what the clamped bins gave


def test_end_bin_rule_with_zero_one_and_two_completions():
    """NaN without completions; one completion in the last bin; two in bin 0 (the lo + 1 >= n branch at p99)."""
    h = np.zeros((3, K.AF_HIST_BINS), dtype=np.uint32)
    h[1, -1] = 1
    h[2, 0] = 2
    lo, hi = np.array([0.0, 5000.0, 1e-8]), np.array([0.0, 5000.0, 3e-8])
    for q, _ in QS:
        got = hist_percentiles(h, q, lo=lo, hi=hi)
        assert np.isnan(got[0]) and np.isnan(twin_percentile(h[0], 0, q, 0.0, 0.0))
        for i in (1, 2):
            want = twin_percentile(h[i], int(h[i].sum()), q, lo[i], hi[i])
            assert got[i].tobytes() == np.float64(want).tobytes(), (i, q)
    last_lo = TOP - TOP / 2 / (1 << K.AF_HIST_SUB_BITS)                  # 4080 s: the last bin's lower edge
    assert float(hist_percentiles(h[1], 50.0, lo=5000.0, hi=5000.0)) == last_lo + 0.5 * (5000.0 - last_lo)
    edge1 = BOTTOM * (1 + 2.0 ** -K.AF_HIST_SUB_BITS)
    assert float(hist_percentiles(h[2], 50.0, lo=1e-8, hi=3e-8)) == pytest.approx(1e-8 + 0.5 * (edge1 - 1e-8), rel=1e-12)
