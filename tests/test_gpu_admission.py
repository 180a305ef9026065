"""GPU tier: admission limits (``("server_max_in_service", server)`` sweep columns; DESIGN.md §3.12) on the device -- a
cap x users x fleet grid of more than 10^4 rows in every pass structure (the full lane build: a launch with a limit
never runs the lean one), over several
waves from a replica id > 0, against the CPU twin (``server_rejected`` included) and traced replicas against the oracle;
a column of zeros bit-identical to no column with every accumulating output on; shards, ``balance=``, retries, exact
percentiles and the drill-down runner; the example."""

from __future__ import annotations

import runpy
import sys

import des_admission
import numpy as np
import pytest
import twin_admission
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from lb_rows import uncoverable
from test_gpu_multiwave import BEGIN, CAPS, device_run, sm_count

from asyncflow_b200 import Engine, SweepRunner, SweepSpec, flatten
from asyncflow_b200.results import SweepResults

pytestmark = pytest.mark.gpu

H = 10
OUT = ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr", "rejected")


@pytest.fixture(scope="module")
def eng():
    with Engine(0) as e:
        yield e


def grid(payload, m: int, seed: int) -> dict:
    """Columns of (cap per server, users, fleet) rows drawn at random: caps 0 (none) to 6, users x1 to x4, and on c4
    fleets of the first k servers a row may uncover (lb_rows.uncoverable) with its outage and spike in the horizon."""
    flat = flatten(payload)
    rng = np.random.default_rng(seed)
    cols: dict = {("server_max_in_service", s): rng.integers(0, 7, m).astype(np.float64) for s in flat.server_ids}
    cols[("users_mean",)] = rng.choice([1.0, 2.0, 4.0], m) * float(flat.pod.users_mean)
    lb = payload["topology_graph"]["nodes"].get("load_balancer")
    if lb is not None and len(lb["server_covered"]) > 2:
        free, _ = uncoverable(payload)                # (the kept server is always behind the load balancer)
        k = rng.integers(0, len(free) + 1, m)
        cols.update({("lb_covered", s): (k > j).astype(np.float64) for j, s in enumerate(free)})
    if any(e.event_id == "ev-srv3-down" for e in flat.events):     # c4's outage and spike moved into the horizon
        cols[("event_start", "ev-srv3-down")] = rng.choice([2.0, 5.0], m)
        cols[("event_end", "ev-srv3-down")] = rng.choice([6.0, 9.0], m)
        cols[("event_start", "ev-spike")] = np.full(m, 3.0)
        cols[("event_end", "ev-spike")] = np.full(m, 8.0)
    return cols


_twin: dict = {}


@pytest.mark.parametrize("scenario,mode", [("c3_lb_two_servers.yml", "auto"), ("c3_lb_two_servers.yml", "lane")]
                         + [("c4_lb8_events.yml", m) for m in ("auto", "lane", "warp", "two_pass")])
def test_a_cap_grid_equals_the_twin_over_several_waves(eng, scenario, mode):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 3 * sm_count() * 32 + 17                      # > 10^4 rows: several waves of lanes
    assert n >= 10_000
    spec = SweepSpec(flat, BEGIN + n, grid(payload, BEGIN + n, 7))
    eng.set_mode(mode)
    full = scenario.startswith("c4")
    trace = 3 if full else 0
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=0 if mode == "auto" else 1, trace=trace,
                     clock_cap=100000, **CAPS)
    dev["rejected"] = eng.server_rejected()
    eng.set_mode("auto")
    if not full or mode in ("lane", "two_pass"):       # (a launch with a limit runs the full lane build)
        assert dev["passes"]["lane_pass"] == 1 and dev["passes"]["lane_lean"] == 0, dev["passes"]
    if scenario not in _twin:
        _twin[scenario] = twin_admission.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN,
                                             engine="lane", **CAPS)
    ref = _twin[scenario]
    for k in OUT:
        assert np.array_equal(dev[k], ref[k]), k
    assert dev["rejected"].sum() > 0                  # (a row without caps may overflow a pool: flagged like the twin's)
    for j in range(trace):
        assert dev["stats"]["flags"][j] == 0
        p, adm = spec.payload_and_admission(payload, BEGIN + j)
        o = des_admission.simulate(p, seed=SEED, replica=BEGIN + j, admission=adm)
        red = flatten(p)
        keep = [flat.edge_ids.index(e) for e in red.edge_ids]
        assert_matches_oracle(o, red, stats=dev["stats"][j], clocks=dev["clocks"][j], sent=dev["sent"][j][keep],
                              dropped=dev["dropped"][j][keep], throughput=dev["thr"][j])
        assert [int(x) for x in dev["rejected"][j]] == [o["server_rejected"][s] for s in flat.server_ids]


@pytest.mark.parametrize("scenario", ["c3_lb_two_servers.yml", "c4_lb8_events.yml"])
def test_a_zero_column_is_bit_identical_to_no_column(scenario):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 2 * sm_count() * 32
    rng = np.random.default_rng(3)
    users = {("users_mean",): rng.choice([1.0, 3.0], n) * float(flat.pod.users_mean)}
    zeros = {**users, **{("server_max_in_service", s): np.zeros(n) for s in flat.server_ids}}
    kw = dict(seed=SEED, pinned=False, bands=np.arange(n) % 3, latency_window_s=5, dist_series=[("ready_queue_len", flat.server_ids[0])],
              occupancy=True, throughput=True)
    a = SweepRunner(payload, n, users, **kw)
    b = SweepRunner(payload, n, zeros, **kw)
    ra, rb = a.run(), b.run()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max", "throughput", "band_count", "band_sum",
              "band_sumsq", "lat_hist", "lat_sum_hi", "lat_sum_lo", "dist_hist", "occupancy", "server_rejected"):
        x, y = getattr(ra, k), getattr(rb, k)
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), k
    assert not rb.server_rejected.any()
    a.close()
    b.close()


def test_shards_balance_retries_and_drill_down():
    payload = load_scenario("c4_lb8_events.yml", H)
    flat = flatten(payload)
    n = 512
    cols = grid(payload, n, 11)
    streams = (np.arange(n) // 4).tolist()            # four caps per stream: paired rows
    want_r = SweepRunner(payload, n, cols, seed=SEED, pinned=False, streams=streams)
    want = want_r.run()
    assert want.server_rejected.sum() > 0 and not want.overflowed.any()
    small = SweepRunner(payload, n, cols, seed=SEED, request_capacity=64, event_capacity=64, pinned=False, streams=streams)
    res = small.run(retry_overflow=True)
    assert not res.overflowed.any()
    np.testing.assert_array_equal(res.server_rejected, want.server_rejected)
    bal = SweepRunner(payload, n, cols, seed=SEED, pinned=False, streams=streams, balance=True)
    np.testing.assert_array_equal(bal.run().server_rejected, want.server_rejected)
    shards = SweepResults.concatenate([want_r.run(0, 200), want_r.run(200, n)])
    np.testing.assert_array_equal(shards.server_rejected, want.server_rejected)
    np.testing.assert_array_equal(shards.stats["completed"], want.stats["completed"])
    rows = [0, 5, n - 1]
    want_r.exact_percentiles(want, rows)
    for i in rows:
        one = want_r.replica_runner(i).run()
        assert one.server_rejected == dict(zip(flat.server_ids, map(int, want.server_rejected[i])))
        assert one.generated == int(want.stats["generated"][i])
        lat = np.asarray(one.clocks)[:, 1] - np.asarray(one.clocks)[:, 0]
        assert len(lat) == int(want.stats["completed"][i])
        if len(lat):
            assert float(np.percentile(lat, 99)) == float(want.stats["p99"][i])
    for r in (want_r, small, bal):
        r.close()


def test_the_example_runs(monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_admission.py", "--reps", "16", "--horizon", "30"])
    runpy.run_path(str(ROOT / "examples" / "sweep_admission.py"), run_name="__main__")
    assert "in one launch" in capsys.readouterr().out
