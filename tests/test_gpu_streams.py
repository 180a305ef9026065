"""GPU tier: random streams (af_streams_upload) on the device -- every pass structure and both builds of the lane loop
against the CPU twin and the oracle, the stitched re-run, an identity table with every band kind, shards, balancing,
retries, exact percentiles, the drill-down runner and the example."""

from __future__ import annotations

import runpy
import sys

import des_port
import numpy as np
import pytest
import twin_streams
from event_rows import event_time_columns
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from test_gpu_multiwave import CAPS, device_run, sm_count

from asyncflow_b200 import Engine, SweepRunner, SweepSpec, flatten

pytestmark = pytest.mark.gpu

BEGIN = 1000
H = 10
OUT = ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr")


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.upload_streams(None)
    e.close()


def _table(n: int) -> tuple[np.ndarray, int]:
    """Streams of replicas BEGIN + 1 .. BEGIN + n - 6: repeats, streams >= 2^32; the others draw as their own id."""
    i = np.arange(n - 7, dtype=np.uint64)
    return (i % np.uint64(97)) * np.uint64(2**33) + np.uint64(3), BEGIN + 1


def _stream_of(table, first, replica: int) -> int:
    return int(table[replica - first]) if first <= replica < first + table.size else replica


def _spec(payload, m: int, seed: int, users=(20.0, 60.0, 150.0)) -> SweepSpec:
    flat = flatten(payload)
    rng = np.random.default_rng(seed)
    cols = event_time_columns(flat, m, rng) if flat.events else {}
    cols[("users_mean",)] = rng.choice(users, m)
    return SweepSpec(flat, m, cols)


def _same(dev: dict, ref: dict, keys=OUT) -> None:
    for k in keys:
        assert np.array_equal(dev[k], ref[k]), k


@pytest.mark.parametrize("scenario,mode,full", [("ev_spikes_outages.yml", m, False) for m in ("auto", "lane", "warp", "two_pass")]
                         + [("c3_lb_two_servers.yml", "auto", False), ("c3_lb_two_servers.yml", "auto", True)])
def test_every_pass_structure_equals_the_twin_over_several_waves(eng, scenario, mode, full, monkeypatch):
    if full:
        monkeypatch.setenv("ASYNCFLOW_B200_LANE_FULL", "1")
    else:
        monkeypatch.delenv("ASYNCFLOW_B200_LANE_FULL", raising=False)
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 3 * sm_count() * 32 + 17
    spec = _spec(payload, BEGIN + n, 5)
    table, first = _table(n)
    eng.set_mode(mode)
    eng.upload_streams(table, first)
    trace = 0 if scenario.startswith("c3") and not full else 3      # (a traced replica rules the lean loop out)
    wpb = 0 if mode == "auto" else 1                                   # (AUTO runs lanes at 4 warps per block or more)
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=wpb, trace=trace, clock_cap=100000, **CAPS)
    eng.upload_streams(None)
    eng.set_mode("auto")
    if mode == "auto":
        assert dev["passes"]["lane_pass"] == 1
    if scenario.startswith("c3"):
        assert dev["passes"]["lane_pass"] == 1 and dev["passes"]["lane_lean"] == int(not full), dev["passes"]
    ref = twin_streams.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN, engine="lane",
                           streams=table, stream_first=first, **CAPS)
    _same(dev, ref)
    assert (dev["stats"]["flags"] == 0).all()
    for j in range(trace):
        p = spec.payload_for(payload, BEGIN + j)
        o = des_port.simulate(p, seed=SEED, replica=_stream_of(table, first, BEGIN + j))
        assert_matches_oracle(o, flatten(p), stats=dev["stats"][j], clocks=dev["clocks"][j], sent=dev["sent"][j],
                              dropped=dev["dropped"][j], series=dev["series"][j], throughput=dev["thr"][j])


def test_the_stitched_rerun_equals_warp_and_the_twin(eng):
    payload = load_scenario("ev_spikes_outages.yml", H)
    flat = flatten(payload)
    n = 2 * sm_count() * 32
    spec = _spec(payload, BEGIN + n, 6, users=(30.0, 200.0, 3000.0))
    table, first = _table(n)
    eng.upload_streams(table, first)
    eng.set_mode("two_pass")
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["warp_pass"] == 1 and p["warp_replicas"] > 0, p
    eng.set_mode("warp")
    ref = device_run(eng, flat, n, sweep=spec, **CAPS)
    eng.set_mode("auto")
    eng.upload_streams(None)
    _same(dev, ref)
    tw = twin_streams.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN, engine="warp",
                          streams=table, stream_first=first, **CAPS)
    _same(dev, tw)


@pytest.mark.parametrize("mode", ["two_pass", "warp"])
def test_an_identity_table_is_bit_identical_with_every_band_kind(mode):
    payload = load_scenario("ev_spikes_outages.yml", 40)
    n = 6 * sm_count() * 32
    cols = {("users_mean",): np.random.default_rng(2).choice([20.0, 60.0, 3000.0], n)}
    kw = dict(seed=SEED, bands=np.arange(n) % 3, latency_window_s=2, dist_series=[("ready_queue_len", "srv-1")],
              occupancy=True, pinned=False)
    a = SweepRunner(payload, n, cols, **kw)
    b = SweepRunner(payload, n, cols, streams=np.arange(n), **kw)
    for sw in (a, b):
        sw.engine().set_mode(mode)
    ra, rb = a.run(), b.run()
    a.close(), b.close()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "band_count", "band_sum", "band_sumsq",
              "lat_hist", "lat_sum_hi", "lat_sum_lo", "dist_hist", "occupancy"):
        assert np.array_equal(getattr(ra, k), getattr(rb, k)), k


def _runner(n: int, seed: int = 7, users=(10.0, 60.0, 300.0), streams=None, **kw) -> SweepRunner:
    payload = load_scenario("ev_spikes_outages.yml", H)
    flat = flatten(payload)
    rng = np.random.default_rng(seed)
    cols = event_time_columns(flat, n, rng)
    cols[("users_mean",)] = rng.choice(users, n)
    if streams is None:
        streams = rng.integers(0, 2**63, n // 4, dtype=np.uint64)[np.arange(n) % (n // 4)] * np.uint64(2) + np.uint64(1)
    return SweepRunner(payload, n, cols, seed=SEED, pinned=False, streams=streams, **kw)


def test_shards_and_balance_keep_each_rows_stream():
    n = 2 * sm_count() * 32 + 5
    sw = _runner(n)
    whole = sw.run()
    a, b = sw.run(0, n // 2), sw.run(n // 2, n)
    bal = _runner(n, balance=True, deal=2)
    assert bal.order is not None
    rb = bal.run()
    sw.close(), bal.close()
    for k in ("stats", "edge_sent", "samp_sum"):
        assert np.array_equal(np.concatenate([getattr(a, k), getattr(b, k)]), getattr(whole, k)), k
        assert np.array_equal(getattr(rb, k), getattr(whole, k)), k
    assert np.array_equal(rb.streams, whole.streams) and np.array_equal(whole.streams, sw.stream_ids)


def test_retry_overflow_reruns_with_each_rows_stream():
    n = 256
    heavy = (10.0, 300.0, 3000.0)
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
        o = des_port.simulate(sw.payload_for(r), seed=SEED, replica=int(sw.stream_ids[r]))
        c = np.asarray(o["clocks"], dtype=np.float64).reshape(-1, 2)
        want = np.percentile(c[:, 1] - c[:, 0], [50, 95, 99])
        assert [res.stats[q][r] for q in ("p50", "p95", "p99")] == list(want)
        one = sw.replica_runner(r).run()
        assert one.generated == int(res.stats["generated"][r]) and len(one.clocks) == int(res.stats["completed"][r])
        assert np.array_equal(np.asarray(one.clocks), c)
    sw.close()


def test_the_paired_steps_example_runs(monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_paired_steps.py", "--replicas", "200", "--horizon", "10"])
    runpy.run_path(str(ROOT / "examples" / "sweep_paired_steps.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "1200 replicas in one launch" in out and out.count("users ") == 6
