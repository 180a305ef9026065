"""GPU tier: per-replica event timelines (af_timeline_upload) on the device -- every pass structure against the CPU twin
and the oracle, the stitched re-run, rows equal to the scenario's, shards, balancing, retries, exact percentiles, the
drill-down runner and the example."""

from __future__ import annotations

import runpy
import sys

import des_port
import numpy as np
import pytest
import twin_rows
from event_rows import event_time_columns
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from test_gpu_multiwave import CAPS, device_run, sm_count

from asyncflow_b200 import Engine, SweepRunner, SweepSpec, flatten

pytestmark = pytest.mark.gpu

BEGIN = 1000
H = 10


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def _payload(horizon: int = H) -> dict:
    return load_scenario("ev_spikes_outages.yml", horizon)


def _rows(flat, m: int, seed: int, *, users=None, amp: bool = True) -> SweepSpec:
    cols = event_time_columns(flat, m, np.random.default_rng(seed), spike_delta=amp)
    if users is not None:
        cols[("users_mean",)] = np.random.default_rng(seed + 1).choice(users, m)
    return SweepSpec(flat, m, cols)


OUT = ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr")


def _same(dev: dict, ref: dict, keys=OUT) -> None:
    for k in keys:
        assert np.array_equal(dev[k], ref[k]), k


@pytest.mark.parametrize("mode", ["auto", "lane", "warp", "two_pass"])
def test_every_pass_structure_equals_the_twin_over_several_waves(eng, mode):
    payload = _payload()
    flat = flatten(payload)
    n = 3 * sm_count() * 32 + 17
    spec = _rows(flat, BEGIN + n, 5)
    eng.set_mode(mode)
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, trace=3, clock_cap=100000, **CAPS)
    ref = twin_rows.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN, engine="lane", **CAPS)
    _same(dev, ref)
    assert (dev["stats"]["flags"] == 0).all()
    for j in range(3):
        p = spec.payload_for(payload, BEGIN + j)
        o = des_port.simulate(p, seed=SEED, replica=BEGIN + j)
        st = dev["stats"][j]
        assert_matches_oracle(o, flatten(p), stats=st, clocks=dev["clocks"][j], sent=dev["sent"][j],
                              dropped=dev["dropped"][j], series=dev["series"][j], throughput=dev["thr"][j])
    eng.set_mode("auto")


def test_the_stitched_rerun_equals_warp(eng):
    flat = flatten(_payload())
    n = 2 * sm_count() * 32
    spec = _rows(flat, BEGIN + n, 6, users=[30.0, 200.0, 3000.0])
    eng.set_mode("two_pass")
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["warp_pass"] == 1 and p["warp_replicas"] > 0, p
    eng.set_mode("warp")
    ref = device_run(eng, flat, n, sweep=spec, **CAPS)
    eng.set_mode("auto")
    _same(dev, ref)


def test_rows_equal_to_the_scenario_are_bit_identical_with_every_band_kind(eng):
    flat = flatten(_payload(40))
    n = 6 * sm_count() * 32
    cols = {("users_mean",): np.random.default_rng(2).choice([20.0, 60.0, 120.0], n)}
    same = dict(cols)
    for e in flat.events:
        same[("event_start", e.event_id)] = np.full(n, e.t_start)
        same[("event_end", e.event_id)] = np.full(n, e.t_end)
    groups = np.arange(n) % 3
    kw = dict(seed=SEED, bands=groups, latency_window_s=2, dist_series=[("ready_queue_len", "srv-1")], occupancy=True,
              pinned=False)
    a = SweepRunner(_payload(40), n, cols, **kw)
    b = SweepRunner(_payload(40), n, same, **kw)
    assert b.spec.timelines is not None and a.spec.timelines is None
    ra, rb = a.run(), b.run()
    a.close(), b.close()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "band_count", "band_sum", "band_sumsq",
              "lat_hist", "lat_sum_hi", "lat_sum_lo", "dist_hist", "occupancy"):
        assert np.array_equal(getattr(ra, k), getattr(rb, k)), k


def _runner(n: int, seed: int = 7, users=(10.0, 60.0, 300.0), **kw) -> SweepRunner:
    payload = _payload()
    flat = flatten(payload)
    cols = event_time_columns(flat, n, np.random.default_rng(seed), spike_delta=True)
    cols[("users_mean",)] = np.random.default_rng(seed + 1).choice(users, n)
    return SweepRunner(payload, n, cols, seed=SEED, pinned=False, **kw)


def test_two_shards_equal_one_launch():
    n = 2 * sm_count() * 32 + 5
    sw = _runner(n)
    whole = sw.run()
    a, b = sw.run(0, n // 2), sw.run(n // 2, n)
    sw.close()
    for k in ("stats", "edge_sent", "samp_sum"):
        assert np.array_equal(np.concatenate([getattr(a, k), getattr(b, k)]), getattr(whole, k)), k


def test_balance_keeps_each_rows_timeline():
    n = sm_count() * 32 + 9
    bal = _runner(n, balance=True)
    assert bal.order is not None
    res = bal.run()
    plain = SweepRunner(_payload(), n, {sel: arr for sel, arr in bal._run_spec.selectors}, seed=SEED, pinned=False)
    ref = plain.run()                                  # replica id p runs row order[p] in both
    bal.close(), plain.close()
    ids = bal.replica_ids
    for k in ("stats", "edge_sent", "samp_sum"):
        assert np.array_equal(getattr(res, k), getattr(ref, k)[ids]), k


def test_retry_overflow_reruns_with_each_replicas_own_timeline():
    n = 256
    heavy = (10.0, 300.0, 3000.0)                      # 3000 users overload the servers: queues of thousands
    sw = _runner(n, 9, heavy, request_capacity=48, event_capacity=64)
    res = sw.run(retry_overflow=True)
    big = _runner(n, 9, heavy, request_capacity=1 << 16, event_capacity=1 << 16)
    ref = big.run()
    sw.close(), big.close()
    assert getattr(res, "reran", False) and (ref.stats["flags"] == 0).all()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max"):
        assert np.array_equal(getattr(res, k), getattr(ref, k)), k


def test_exact_percentiles_and_the_drill_down_runner():
    n = 64
    sw = _runner(n, 12, balance=True)
    res = sw.run()
    rows = [1, 17, 40]
    sw.exact_percentiles(res, rows)
    for r in rows:
        o = des_port.simulate(sw.payload_for(r), seed=SEED, replica=int(sw.replica_ids[r]))
        c = np.asarray(o["clocks"], dtype=np.float64).reshape(-1, 2)
        want = np.percentile(c[:, 1] - c[:, 0], [50, 95, 99])
        assert [res.stats[q][r] for q in ("p50", "p95", "p99")] == list(want)
        one = sw.replica_runner(r).run()
        assert one.generated == int(res.stats["generated"][r]) and len(one.clocks) == int(res.stats["completed"][r])
        assert np.array_equal(np.asarray(one.clocks), c)
    sw.close()


def test_the_outage_duration_example_runs(monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_outage_duration.py", "40"])
    runpy.run_path(str(ROOT / "examples" / "sweep_outage_duration.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "320 replicas in one launch" in out and "0 overflowed" in out and "down  60 s" in out
