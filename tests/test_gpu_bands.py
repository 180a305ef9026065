"""GPU tier: per-tick sampled-metric bands on the CUDA engine.  In every pass structure the device's bands are the
exact sums of its own traced series and equal the CPU band twin's bit for bit; a replica the thread-per-replica pass
flags and the warp-per-replica pass re-runs counts once, in full; at the bench workload's shape the bands agree with
the per-replica sampled sums; and no other output changes when bands are on."""

from __future__ import annotations

import band_ref
import numpy as np
import pytest
import twin
from helpers import SEED, load_scenario

from asyncflow_b200 import Engine, EngineError, SweepRunner, SweepSpec, flatten
from asyncflow_b200 import _capi as K

pytestmark = pytest.mark.gpu

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW


def traced_bands(eng: Engine, flat, n: int, groups: np.ndarray, n_groups: int):
    """Per-group sums of the device's own traced series (every replica traced, none stopped)."""
    T, S = twin.ticks(flat), flat.n_series
    cnt = np.zeros((n_groups, T), dtype=np.uint32)
    s = np.zeros((n_groups, S, T), dtype=np.uint64)
    sq = np.zeros((n_groups, S, T), dtype=np.uint64)
    for i in range(n):
        m = eng.trace_series(i).astype(np.uint64)
        assert m.shape == (S, T)
        g = int(groups[i])
        cnt[g] += 1
        s[g] += m
        sq[g] += m * m
    return cnt, s, sq


def assert_same(got, want):
    for name, a, b in zip(("count", "sum", "sumsq"), got, want):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), name


@pytest.mark.parametrize("mode", ["auto", "two_pass", "lane", "warp"])
def test_device_bands_equal_traced_sums_and_the_twin(mode):
    payload = load_scenario("c3_lb_two_servers.yml", 20)
    flat = flatten(payload)
    n, G = 320, 8
    rng = np.random.default_rng(5)
    spec = SweepSpec(flat, n, {("users_mean",): rng.choice([20.0, 60.0, 150.0], n)})
    groups = (np.arange(n) % G).astype(np.uint32)
    with Engine(0) as eng:
        eng.upload(flat)
        eng.set_mode(mode)
        eng.configure(trace_replicas=n, trace_clock_capacity=20000)
        eng.upload_sweep(spec, 0)
        eng.upload_bands(groups, 0, G)
        eng.run(SEED, 0, n)
        st = eng.stats()
        assert (st["flags"] & STOPS == 0).all()
        got = eng.bands()
        assert_same(got, traced_bands(eng, flat, n, groups, G))
    tw = twin.run_lane(flat, seed=SEED, n=n, sweep=spec, groups=groups, n_groups=G, sampled=True)
    assert_same(got, band_ref.scan(flat, tw["band_rows"], G))
    assert (got[0] == n // G).all()


def test_two_pass_stitches_the_flagged_replicas():
    """C2's topology at 1 000 users on a short horizon: the lane pass's nominal pools overflow, the warp pass re-runs
    those replicas from the tick they stopped at, and every replica counts once, in full."""
    payload = load_scenario("c1_my_service.yml", 6)
    payload["rqs_input"]["avg_active_users"]["mean"] = 1000
    flat = flatten(payload)
    n, G = 256, 4
    groups = (np.arange(n) % G).astype(np.uint32)
    ev_cap, rq_cap = 8192, 65536
    with Engine(0) as eng:
        eng.upload(flat)
        eng.set_mode("two_pass")
        eng.configure(event_capacity=ev_cap, request_capacity=rq_cap, trace_replicas=n, trace_clock_capacity=200000)
        eng.upload_bands(groups, 0, G)
        eng.run(SEED, 0, n)
        passes = eng.last_run_passes()
        st = eng.stats()
        got = eng.bands()
        traced = traced_bands(eng, flat, n, groups, G)
    assert passes["lane_replicas"] > 0 and passes["warp_replicas"] > 0, passes
    assert (st["flags"] & STOPS == 0).all()
    assert_same(got, traced)
    lane = twin.run_lane(flat, seed=SEED, n=n, groups=groups, n_groups=G, event_capacity=512, request_capacity=2048,
                         sampled=True)
    flagged = np.flatnonzero(lane["stats"]["flags"] & STOPS)
    assert flagged.size == passes["warp_replicas"]
    twin.run_warp(flat, seed=SEED, n=n, groups=groups, n_groups=G, event_capacity=ev_cap, request_capacity=rq_cap,
                redo=flagged, band_from=lane["band_from"], into=lane, sampled=True)
    assert_same(got, band_ref.scan(flat, lane["band_rows"], G))
    assert (got[0] == n // G).all()


def _bench_runner(bands, n=20_000):
    import bench
    w = bench.make_workload("c3", None, n)
    flat = flatten(w.payload)
    ids = np.arange(n, dtype=np.int64)
    return SweepRunner(flat, n, w.columns(flat, ids, n), seed=bench.SEED, histogram=True, throughput=True, bands=bands)


def test_bench_shape_band_totals_match_the_sampled_sums_and_change_nothing_else():
    n, G = 20_000, 20
    groups = (np.arange(n) * 7 % G).astype(np.uint32)
    off = _bench_runner(None, n)
    r_off = off.run()
    h_off = off.engine().histograms()
    off.close()
    on = _bench_runner(groups, n)
    r_on = on.run()
    h_on = on.engine().histograms()
    passes = on.engine().last_run_passes()
    on.close()
    assert passes["lane_pass"] == 1
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "throughput"):
        assert getattr(r_on, k).tobytes() == getattr(r_off, k).tobytes(), k
    assert h_on.tobytes() == h_off.tobytes()
    T = twin.ticks(on.flat)
    assert r_on.band_count.shape == (G, T)
    assert not (r_on.stats["flags"] & K.FLAG_LB_EMPTY).any()
    assert (r_on.band_count == np.bincount(groups, minlength=G)[:, None]).all()
    with np.errstate(over="ignore"):
        for g in range(G):
            want = r_on.samp_sum[groups == g].sum(axis=0, dtype=np.uint64)
            assert np.array_equal(r_on.band_sum[g].sum(axis=1, dtype=np.uint64), want), g
    assert r_on.band_sumsq.dtype == np.uint64 and (r_on.band_sumsq >= r_on.band_sum).all()


def test_upload_rejects_groups_whose_sum_of_squares_could_wrap():
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    spec = SweepSpec(flat, 8, {("server_ram_mb", flat.server_ids[0]): [512.0] * 7 + [2147483000.0]})
    with Engine(0) as eng:
        eng.upload(flat)
        eng.configure(request_capacity=1024)
        eng.upload_sweep(spec, 0)
        with pytest.raises(EngineError, match="swept ram_mb 2147483000"):
            eng.upload_bands(np.zeros(8, dtype=np.uint32), 0, 1)
        eng.upload_bands(np.arange(8, dtype=np.uint32) % 4, 0, 4)       # groups of 2: 2 x (2^31)^2 < 2^64
        eng.run(SEED, 0, 8)
        c, _, _ = eng.bands()
        assert (c == 2).all()


def test_upload_refuses_band_rows_the_kernels_could_overrun_or_the_device_cannot_hold():
    payload = load_scenario("c1_my_service.yml", 86_400)
    payload["sim_settings"]["sample_period_s"] = 0.001          # >= 5e7 ticks: more than a band row holds
    with Engine(0) as eng:
        eng.upload(flatten(payload))
        with pytest.raises(EngineError, match="ticks or more"):
            eng.upload_bands(np.zeros(4, dtype=np.uint32), 0, 1)
        eng.upload(flatten(load_scenario("c1_my_service.yml", 5)))
        with pytest.raises(EngineError, match="more than the device"):
            eng.upload_bands(np.zeros(1, dtype=np.uint32), 0, 4_000_000_000)
        eng.upload_bands(np.zeros(4, dtype=np.uint32), 0, 1)
        eng.upload(flatten(payload))                                # a scenario uploaded later is checked by af_run
        with pytest.raises(EngineError, match="ticks or more"):
            eng.run(SEED, 0, 4)
