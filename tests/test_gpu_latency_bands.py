"""GPU tier: per-window latency bands on the CUDA engine.  In every pass structure the device's rows are its own traced
clocks binned and equal the CPU twin's bit for bit; a replica the thread-per-replica pass flags and the
warp-per-replica pass re-runs counts once, in full; no other output changes with latency bands, sampled bands or both
on; two shards concatenated equal one run; and on C4 the +30 ms spike shows in the windowed mean latency while the
pooled p95 agrees with numpy on the traced latencies."""

from __future__ import annotations

import latency_twin as LT
import numpy as np
import pytest
from helpers import SEED, load_scenario

from asyncflow_b200 import Engine, EngineError, SweepRunner, SweepSpec, flatten
from asyncflow_b200 import _capi as K

pytestmark = pytest.mark.gpu

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW | K.FLAG_LB_EMPTY


def traced_rows(eng: Engine, flat, n: int, groups: np.ndarray, n_groups: int, w: int) -> np.ndarray:
    rows = LT.new_rows(flat, n_groups, w)
    for i in range(n):
        LT.bin_clocks(rows, int(groups[i]), eng.trace_clocks(i), w, int(flat.horizon_s))
    return rows


def assert_same(got, rows, n_groups):
    want = LT.split(rows, n_groups)
    for name, a, b in zip(("hist", "sum_hi", "sum_lo"), got, want):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), name


@pytest.mark.parametrize("mode", ["auto", "two_pass", "lane", "warp"])
def test_device_rows_equal_traced_clocks_and_the_twin(mode):
    payload = load_scenario("c3_lb_two_servers.yml", 20)
    flat = flatten(payload)
    n, G, w = 320, 8, 3
    rng = np.random.default_rng(5)
    spec = SweepSpec(flat, n, {("users_mean",): rng.choice([20.0, 60.0, 150.0], n)})
    groups = (np.arange(n) % G).astype(np.uint32)
    with Engine(0) as eng:
        eng.upload(flat)
        eng.set_mode(mode)
        eng.configure(trace_replicas=n, trace_clock_capacity=20000)
        eng.upload_sweep(spec, 0)
        eng.configure_bands(sampled=False, latency_window_s=w)
        eng.upload_bands(groups, 0, G)
        eng.run(SEED, 0, n)
        assert (eng.stats()["flags"] & STOPS == 0).all()
        got = eng.latency_bands()
        assert_same(got, traced_rows(eng, flat, n, groups, G, w), G)
    tw = LT.run_lane(flat, seed=SEED, n=n, sweep=spec, groups=groups, n_groups=G, window=w)
    assert_same(got, tw["lat_rows"], G)


def test_two_pass_stitches_the_flagged_replicas():
    payload = load_scenario("c1_my_service.yml", 6)
    payload["rqs_input"]["avg_active_users"]["mean"] = 1000
    flat = flatten(payload)
    n, G, w = 256, 4, 1
    groups = (np.arange(n) % G).astype(np.uint32)
    ev_cap, rq_cap = 8192, 65536
    res = {}
    for mode in ("two_pass", "warp"):
        with Engine(0) as eng:
            eng.upload(flat)
            eng.set_mode(mode)
            eng.configure(event_capacity=ev_cap, request_capacity=rq_cap, trace_replicas=n, trace_clock_capacity=200000)
            eng.configure_bands(latency_window_s=w)
            eng.upload_bands(groups, 0, G)
            eng.run(SEED, 0, n)
            res[mode] = (eng.last_run_passes(), eng.stats().copy(), eng.latency_bands(),
                         traced_rows(eng, flat, n, groups, G, w))
    passes, st, got, traced = res["two_pass"]
    assert passes["lane_replicas"] > 0 and passes["warp_replicas"] > 0, passes
    assert (st["flags"] & STOPS == 0).all()
    assert_same(got, traced, G)
    for a, b in zip(got, res["warp"][2]):
        assert np.array_equal(a, b)
    assert int(got[0].sum()) == int(st["completed"].sum())         # every completion once


def _bench_runner(n, **kw):
    import bench
    wl = bench.make_workload("c3", None, n)
    flat = flatten(wl.payload)
    ids = np.arange(n, dtype=np.int64)
    return SweepRunner(flat, n, wl.columns(flat, ids, n), seed=bench.SEED, histogram=True, throughput=True, **kw)


def test_on_off_changes_no_other_output():
    n, G = 20_000, 20
    groups = (np.arange(n) * 7 % G).astype(np.uint32)
    keys = ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "throughput")
    out = {}
    for name, kw in (("off", {}), ("lat", dict(bands=groups, latency_window_s=1, sampled_bands=False)),
                     ("sampled", dict(bands=groups)), ("both", dict(bands=groups, latency_window_s=1))):
        r = _bench_runner(n, **kw)
        out[name] = (r.run(), r.engine().histograms().copy(), r.engine().last_run_passes())
        r.close()
    for name in ("lat", "sampled", "both"):
        for k in keys:
            assert getattr(out[name][0], k).tobytes() == getattr(out["off"][0], k).tobytes(), (name, k)
        assert out[name][1].tobytes() == out["off"][1].tobytes(), name
    assert out["both"][2]["lane_pass"] == 1
    for k in ("band_count", "band_sum", "band_sumsq"):
        assert getattr(out["both"][0], k).tobytes() == getattr(out["sampled"][0], k).tobytes(), k
    for k in ("lat_hist", "lat_sum_hi", "lat_sum_lo"):
        assert getattr(out["both"][0], k).tobytes() == getattr(out["lat"][0], k).tobytes(), k
    r = out["lat"][0]
    st = r.stats
    ok = (st["flags"] & STOPS) == 0
    assert ok.all()
    n_g = r.lat_hist.sum(axis=(1, 2))
    want = np.bincount(groups, weights=st["completed"], minlength=G)
    assert np.array_equal(n_g, want.astype(np.uint64))
    thr = np.zeros((G, r.throughput.shape[1]), dtype=np.uint64)
    np.add.at(thr, groups, r.throughput.astype(np.uint64))
    assert np.array_equal(r.lat_hist.sum(axis=2), thr)              # w = 1: the windows are the throughput buckets


def test_two_shards_concatenated_equal_one_run():
    from asyncflow_b200 import SweepResults
    n, G = 4000, 5
    groups = (np.arange(n) % G).astype(np.uint32)
    r = _bench_runner(n, bands=groups, latency_window_s=4)
    one = r.run()
    a, b = r.run(0, 1500), r.run(1500, n)
    r.close()
    cat = SweepResults.concatenate([a, b])
    for k in ("lat_hist", "lat_sum_hi", "lat_sum_lo", "band_count", "band_sum", "band_sumsq", "group_size"):
        assert np.array_equal(getattr(cat, k), getattr(one, k)), k
    g1, g2 = one.group_latency(), cat.group_latency()
    assert np.array_equal(g1["mean"], g2["mean"], equal_nan=True)


def test_physical_spike_shows_in_the_windowed_latency():
    payload = load_scenario("c4_lb8_events.yml")
    flat = flatten(payload)
    n = 300
    r = SweepRunner(flat, n, seed=SEED, bands=np.zeros(n, dtype=np.uint32), latency_window_s=1, sampled_bands=False,
                    trace_replicas=n, trace_clock_capacity=200_000)
    res = r.run()
    r.close()
    assert not (res.stats["flags"] & STOPS).any()
    out = res.group_latency()
    t, n_w, mean = out["t"], out["n"][0].astype(np.float64), out["mean"][0]
    spike = (t > 110) & (t <= 155)
    base = (t > 20) & (t <= 95)
    m_spike = float((mean[spike] * n_w[spike]).sum() / n_w[spike].sum())
    m_base = float((mean[base] * n_w[base]).sum() / n_w[base].sum())
    assert m_spike - m_base >= 0.027, (m_spike, m_base)
    lats = np.concatenate([tr.clocks[:, 1] - tr.clocks[:, 0] for tr in res.traced])
    assert lats.size == int(out["total"]["n"][0])
    assert abs(float(out["total"]["p95"][0]) / float(np.percentile(lats, 95)) - 1) < 0.01


def test_configure_refuses_a_negative_window_and_rows_the_device_cannot_hold():
    with Engine(0) as eng:
        eng.upload(flatten(load_scenario("c1_my_service.yml", 86_400)))
        with pytest.raises(EngineError, match="window of -1 s"):
            eng.configure_bands(latency_window_s=-1)
        eng.configure_bands(sampled=False, latency_window_s=1)
        with pytest.raises(EngineError, match="more than the device"):
            eng.upload_bands(np.zeros(4, dtype=np.uint32), 0, 1_000_000)
        eng.upload_bands(np.zeros(4, dtype=np.uint32), 0, 1)
        with pytest.raises(EngineError, match="more than the device"):
            eng.upload_bands(np.zeros(4, dtype=np.uint32), 0, 500_000)
