"""GPU tier: load-balancer rows (``("lb_covered", server)`` / ``("lb_algorithm",)`` sweep columns) on the device -- a
fleet x algorithm x users grid of more than 10^4 rows in every pass structure, the lean and the full lane builds, over
several waves from a replica id > 0, against the CPU twin and the oracle; the four accumulating outputs; the drill-down
runner; retries of overflowed rows; the example."""

from __future__ import annotations

import runpy
import sys

import des_port
import numpy as np
import pytest
import twin_rows
from helpers import ROOT, SEED, load_scenario
from lb_rows import check_replica, lb_servers
from test_gpu_fuzz import acc_device, acc_groups, acc_twin, assert_views_equal, twin_views
from test_gpu_multiwave import BEGIN, CAPS, device_run, sm_count

from asyncflow_b200 import Engine, SweepRunner, SweepSpec, flatten
from asyncflow_b200.results import occ_frac_bits

pytestmark = pytest.mark.gpu

H = 10
OUT = ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr")
ALGOS = ("round_robin", "least_connection")


@pytest.fixture(scope="module")
def eng():
    with Engine(0) as e:
        yield e


def grid(payload, m: int, seed: int, users=(0.5, 1.0, 2.0)) -> SweepSpec:
    """Rows of (fleet = the first k covered servers, algorithm, users) drawn at random; c4's spike and outage of srv-3
    moved into the horizon (every row then carries a timeline row, with srv-3's marks off in fleets without it)."""
    flat = flatten(payload)
    rng = np.random.default_rng(seed)
    srv = lb_servers(payload)
    k = rng.integers(1, len(srv) + 1, m)
    cols: dict = {("lb_covered", s): (k > j).astype(np.float64) for j, s in enumerate(srv)}
    cols[("lb_algorithm",)] = rng.choice(ALGOS, m).tolist()
    cols[("users_mean",)] = rng.choice(users, m) * float(flat.pod.users_mean)
    if any(e.event_id == "ev-srv3-down" for e in flat.events):
        cols[("event_start", "ev-srv3-down")] = rng.choice([2.0, 5.0], m)
        cols[("event_end", "ev-srv3-down")] = rng.choice([6.0, 9.0], m)
        cols[("event_start", "ev-spike")] = np.full(m, 3.0)
        cols[("event_end", "ev-spike")] = np.full(m, 8.0)
    return SweepSpec(flat, m, cols)


_twin: dict = {}


def _same(dev: dict, ref: dict) -> None:
    for k in OUT:
        assert np.array_equal(dev[k], ref[k]), k


@pytest.mark.parametrize("scenario,mode", [("c3_lb_two_servers.yml", "auto"), ("c3_lb_two_servers.yml", "lane")]
                         + [("c4_lb8_events.yml", m) for m in ("auto", "lane", "warp", "two_pass")])
def test_a_fleet_policy_grid_equals_the_twin_over_several_waves(eng, scenario, mode):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = 3 * sm_count() * 32 + 17                      # > 10^4 rows: several waves of lanes
    spec = grid(payload, BEGIN + n, 3)
    assert n >= 10_000
    eng.set_mode(mode)
    full = scenario.startswith("c4")
    trace = 3 if full else 0                           # (a traced replica rules the lean loop out)
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=0 if mode == "auto" else 1, trace=trace,
                     clock_cap=100000, **CAPS)
    eng.set_mode("auto")
    if not full or mode in ("lane", "two_pass"):
        assert dev["passes"]["lane_pass"] == 1 and dev["passes"]["lane_lean"] == int(not full), dev["passes"]
    if scenario not in _twin:                         # (both state machines give the same outputs: one reference)
        _twin[scenario] = twin_rows.run(flat, seed=SEED, replica_begin=BEGIN, n=n, sweep=spec, sweep_first=BEGIN,
                                        engine="lane", **CAPS)
    _same(dev, _twin[scenario])
    assert (dev["stats"]["flags"] == 0).all()
    for j in range(trace):
        p = spec.payload_for(payload, BEGIN + j)
        check_replica(des_port.simulate(p, seed=SEED, replica=BEGIN + j), flat, p, stats=dev["stats"][j],
                      sent=dev["sent"][j], dropped=dev["dropped"][j], thr=dev["thr"][j], clocks=dev["clocks"][j],
                      series=dev["series"][j])


@pytest.mark.parametrize("scenario", ["c3_lb_two_servers.yml", "c4_lb8_events.yml"])
@pytest.mark.parametrize("mode", ["two_pass", "warp"])
def test_the_accumulating_outputs_equal_the_twin(scenario, mode):
    payload = load_scenario(scenario, H)
    flat = flatten(payload)
    n = sm_count() * 32 + 5
    spec = grid(payload, BEGIN + n, 4, users=(0.5, 1.0, 3.0))
    groups = acc_groups(n)
    ram = max(int(flat.pod.servers[i].ram_mb) for i in range(flat.n_servers))      # (the grid sweeps no ram_mb)
    f = occ_frac_bits(max(CAPS["request_capacity"], ram), int(flat.horizon_s))
    out, views = acc_device(flat, spec, n, groups, f, mode, CAPS)
    tw = acc_twin(flat, spec, n, groups, f, CAPS, run=twin_rows.run_lane if mode != "warp" else twin_rows.run_warp)
    for k in ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist"):
        assert np.array_equal(out[k], tw[k]), k
    assert_views_equal(views, twin_views(flat, tw))


def test_drill_down_and_retries_reproduce_the_rows():
    payload = load_scenario("c4_lb8_events.yml", H)
    n = 512
    spec = grid(payload, n, 5, users=(0.5, 1.0, 6.0))
    cols = {sel: arr for sel, arr in spec.selectors}
    cols[("lb_algorithm",)] = [("round_robin", "least_connection")[int(v)] for v in cols[("lb_algorithm",)]]
    small = SweepRunner(payload, n, cols, seed=SEED, request_capacity=64, event_capacity=64, pinned=False)
    res = small.run(retry_overflow=True)
    big = SweepRunner(payload, n, cols, seed=SEED, pinned=False)
    want = big.run()
    assert not res.overflowed.any() and not want.overflowed.any()
    for k in ("generated", "completed", "n_events", "lat_sum", "lat_max"):
        assert np.array_equal(res.stats[k], want.stats[k]), k
    assert np.array_equal(res.edge_sent, want.edge_sent)
    for i in (0, 1, n - 1):
        one = small.replica_runner(i).run()
        assert one.generated == int(want.stats["generated"][i])
        lat = np.asarray(one.clocks)[:, 1] - np.asarray(one.clocks)[:, 0]
        assert len(lat) == int(want.stats["completed"][i]) and float(lat.max()) == float(want.stats["lat_max"][i])
    small.close()
    big.close()


def test_the_example_runs(monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_fleet_size.py", "--reps", "20", "--horizon", "20"])
    runpy.run_path(str(ROOT / "examples" / "sweep_fleet_size.py"), run_name="__main__")
    assert "in one launch" in capsys.readouterr().out
