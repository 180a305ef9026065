"""GPU tier: rate limits (``("server_rate"|"server_burst", server)`` / ``("lb_rate",)`` / ``("lb_burst",)`` sweep
columns; DESIGN.md §3.14) on the device -- a rate x burst x LB rate x users x cap grid of more than 10^4 rows in every
pass structure (the full lane build: a launch with a rate limit never runs the lean one), over several waves from a
replica id > 0, against the CPU twin (``throttled`` included) and traced replicas against the oracle; a rate column of
zeros bit-identical to no column with every accumulating output on; shards, ``balance=``, retries, exact percentiles and
the drill-down runner; the example."""

from __future__ import annotations

import runpy
import sys

import des_deadline
import des_ratelimit
import numpy as np
import pytest
import twin_ratelimit
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from test_gpu_multiwave import BEGIN, CAPS, device_run, sm_count

from asyncflow_b200 import Engine, SweepRunner, SweepSpec, flatten
from asyncflow_b200.results import SweepResults

pytestmark = pytest.mark.gpu

H = 10
OUT = ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr", "rejected", "throttled")


@pytest.fixture(scope="module")
def eng():
    with Engine(0) as e:
        yield e


def _arrival_rate(payload) -> float:
    o = des_deadline.simulate(payload, seed=SEED, replica=0)
    return max(1.0, o["generated"] / float(payload["sim_settings"]["total_simulation_time"]))


def grid(payload, m: int, seed: int) -> dict:
    """Columns of (rate and burst per server, LB rate and burst, users, cap per server) rows drawn at random: rates 0
    (none) or a share of the scenario's arrival rate, bursts 1 to 40, users x1 to x4, caps 0 (none) to 6; on c4 its
    outage and spike moved into the horizon."""
    flat = flatten(payload)
    rng = np.random.default_rng(seed)
    lam = _arrival_rate(payload)
    share = np.array([0.0, 0.1, 0.3, 0.6, 1.2])
    cols: dict = {("server_rate", s): rng.choice(share * lam, m) for s in flat.server_ids}
    cols.update({("server_burst", s): rng.integers(1, 41, m) for s in flat.server_ids})
    cols[("lb_rate",)] = rng.choice(np.array([0.0, 0.5, 1.0, 2.0]) * lam, m)
    cols[("lb_burst",)] = rng.integers(1, 41, m)
    cols.update({("server_max_in_service", s): rng.integers(0, 7, m).astype(np.float64) for s in flat.server_ids})
    cols[("users_mean",)] = rng.choice([1.0, 2.0, 4.0], m) * float(flat.pod.users_mean)
    if any(e.event_id == "ev-srv3-down" for e in flat.events):
        cols[("event_start", "ev-srv3-down")] = rng.choice([2.0, 5.0], m)
        cols[("event_end", "ev-srv3-down")] = rng.choice([6.0, 9.0], m)
        cols[("event_start", "ev-spike")] = np.full(m, 3.0)
        cols[("event_end", "ev-spike")] = np.full(m, 8.0)
    return cols


_twin: dict = {}


@pytest.mark.parametrize("scenario,mode", [("c3_lb_two_servers.yml", "auto"), ("c3_lb_two_servers.yml", "lane")]
                         + [("c4_lb8_events.yml", m) for m in ("auto", "lane", "warp", "two_pass")])
def test_a_rate_limit_grid_equals_the_twin_over_several_waves(eng, scenario, mode):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 3 * sm_count() * 32 + 17                      # > 10^4 rows: several waves of lanes
    assert n >= 10_000
    spec = SweepSpec(flat, BEGIN + n, grid(payload, BEGIN + n, 7))
    eng.set_mode(mode)
    trace = 3
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=0 if mode == "auto" else 1, trace=trace,
                     clock_cap=100000, **CAPS)
    dev["rejected"], dev["throttled"] = eng.server_rejected(), eng.throttled()
    eng.set_mode("auto")
    if mode in ("lane", "two_pass") or (mode == "auto" and dev["passes"]["lane_pass"]):
        assert dev["passes"]["lane_pass"] == 1 and dev["passes"]["lane_lean"] == 0, dev["passes"]
    if scenario not in _twin:
        _twin[scenario] = twin_ratelimit.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN,
                                             engine="lane", **CAPS)
    ref = _twin[scenario]
    for k in OUT:
        assert np.array_equal(dev[k], ref[k]), k
    assert dev["throttled"][:, :flat.n_servers].sum() > 0 and dev["throttled"][:, flat.n_servers].sum() > 0
    st = dev["stats"]
    ok = st["flags"] == 0
    gone = (st["completed"].astype(np.int64) + dev["dropped"].sum(axis=1) + dev["rejected"].sum(axis=1)
            + dev["throttled"].sum(axis=1))
    assert (gone[ok] <= st["generated"][ok]).all()
    for j in range(trace):
        assert st["flags"][j] == 0
        p, ov = spec.payload_and_overload(payload, BEGIN + j)
        o = des_ratelimit.simulate(p, seed=SEED, replica=BEGIN + j, admission=ov["admission"],
                                   rate_limit=ov["rate_limit"], lb_rate_limit=ov["lb_rate_limit"])
        assert_matches_oracle(o, flat, stats=st[j], clocks=dev["clocks"][j], sent=dev["sent"][j],
                              dropped=dev["dropped"][j], throughput=dev["thr"][j])
        assert [int(x) for x in dev["throttled"][j]] == ([o["server_throttled"][s] for s in flat.server_ids]
                                                         + [o["lb_throttled"]])


@pytest.mark.parametrize("scenario", ["c3_lb_two_servers.yml", "c4_lb8_events.yml"])
def test_a_zero_rate_column_is_bit_identical_to_no_column(scenario):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 2 * sm_count() * 32
    rng = np.random.default_rng(3)
    users = {("users_mean",): rng.choice([1.0, 3.0], n) * float(flat.pod.users_mean)}
    zeros = {**users, **{("server_rate", s): np.zeros(n) for s in flat.server_ids}, ("lb_rate",): np.zeros(n),
             ("lb_burst",): np.full(n, 3)}
    kw = dict(seed=SEED, pinned=False, bands=np.arange(n) % 3, latency_window_s=5,
              dist_series=[("ready_queue_len", flat.server_ids[0])], occupancy=True, throughput=True)
    a = SweepRunner(payload, n, users, **kw)
    b = SweepRunner(payload, n, zeros, **kw)
    ra, rb = a.run(), b.run()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "throughput", "band_count", "band_sum",
              "band_sumsq", "lat_hist", "lat_sum_hi", "lat_sum_lo", "dist_hist", "occupancy", "server_rejected",
              "server_expired", "late", "server_throttled", "lb_throttled"):
        x, y = getattr(ra, k), getattr(rb, k)
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), k
    assert not rb.server_throttled.any() and not rb.lb_throttled.any()
    a.close()
    b.close()


def test_shards_balance_retries_and_drill_down():
    payload = load_scenario("c4_lb8_events.yml", H)
    flat = flatten(payload)
    n = 512
    cols = grid(payload, n, 11)
    streams = (np.arange(n) // 4).tolist()            # four rows per stream: paired rows
    want_r = SweepRunner(payload, n, cols, seed=SEED, pinned=False, streams=streams)
    want = want_r.run()
    assert want.server_throttled.sum() > 0 and want.lb_throttled.sum() > 0 and not want.overflowed.any()
    small = SweepRunner(payload, n, cols, seed=SEED, request_capacity=64, event_capacity=64, pinned=False, streams=streams)
    res = small.run(retry_overflow=True)
    assert not res.overflowed.any()
    np.testing.assert_array_equal(res.server_throttled, want.server_throttled)
    np.testing.assert_array_equal(res.lb_throttled, want.lb_throttled)
    bal = SweepRunner(payload, n, cols, seed=SEED, pinned=False, streams=streams, balance=True)
    rb = bal.run()
    np.testing.assert_array_equal(rb.server_throttled, want.server_throttled)
    np.testing.assert_array_equal(rb.lb_throttled, want.lb_throttled)
    shards = SweepResults.concatenate([want_r.run(0, 200), want_r.run(200, n)])
    np.testing.assert_array_equal(shards.server_throttled, want.server_throttled)
    np.testing.assert_array_equal(shards.lb_throttled, want.lb_throttled)
    rows = [0, 5, n - 1]
    want_r.exact_percentiles(want, rows)
    for i in rows:
        one = want_r.replica_runner(i).run()
        assert one.server_throttled == dict(zip(flat.server_ids, map(int, want.server_throttled[i])))
        assert one.lb_throttled == int(want.lb_throttled[i])
        assert one.generated == int(want.stats["generated"][i])
        lat = np.asarray(one.clocks)[:, 1] - np.asarray(one.clocks)[:, 0]
        assert len(lat) == int(want.stats["completed"][i])
        if len(lat):
            assert float(np.percentile(lat, 99)) == float(want.stats["p99"][i])
    for r in (want_r, small, bal):
        r.close()


def test_the_example_runs(monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_rate_limit.py", "--reps", "16", "--horizon", "30"])
    runpy.run_path(str(ROOT / "examples" / "sweep_rate_limit.py"), run_name="__main__")
    assert "in one launch" in capsys.readouterr().out
