"""CPU tier: per-tick sampled-metric bands (af_bands_upload / af_fetch_bands).  Both state machines, driven with their
difference rows by the CPU twin (tests/twin.py), must give per group and tick exactly the integer sums of the
oracle's sampled series over the group's replicas: first-hand, stitched (a replica the thread-per-replica pass stops
and the warp-per-replica pass re-runs from its stop tick), truncated (a stopped replica that is not re-run), and with
every other output unchanged by the bands."""

from __future__ import annotations

import band_ref
import des_port
import fuzz
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario, oracle_series_matrix
from twin_engine import TwinEngine

from asyncflow_b200 import SweepRunner, SweepSpec, flatten
from asyncflow_b200 import _capi as K

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW
REDO = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW      # what af_run's second pass re-runs


def oracle_matrix(payload, flat, replica: int) -> np.ndarray:
    """[n_series, T] series of one oracle replica (a series the scenario does not sample is 0)."""
    o = des_port.simulate(payload, seed=SEED, replica=replica)
    m = oracle_series_matrix(o, flat).astype(np.uint64)
    T = twin.ticks(flat)
    assert m.shape[1] in (0, T)
    return m if m.shape[1] == T else np.zeros((flat.n_series, T), dtype=np.uint64)


def expected(flat, mats: list[np.ndarray], groups, n_groups: int, upto=None):
    """Per-group sums of the series matrices; replica i contributes ticks < upto[i] (default: all)."""
    T, S = twin.ticks(flat), flat.n_series
    cnt = np.zeros((n_groups, T), dtype=np.uint64)
    s = np.zeros((n_groups, S, T), dtype=np.uint64)
    sq = np.zeros((n_groups, S, T), dtype=np.uint64)
    for i, (m, g) in enumerate(zip(mats, groups)):
        k = T if upto is None else min(int(upto[i]), T)
        cnt[g, :k] += 1
        s[g, :, :k] += m[:, :k]
        sq[g, :, :k] += m[:, :k] * m[:, :k]
    return cnt.astype(np.uint32), s, sq


def assert_bands(flat, rows, n_groups, want):
    got = band_ref.scan(flat, rows, n_groups)
    for name, a, b in zip(("count", "sum", "sumsq"), got, want):
        assert a.dtype == b.dtype and np.array_equal(a, b), name


def test_band_twin_reports_the_kernels_tick_count():
    flat = flatten(load_scenario("c1_my_service.yml", 7))
    assert abs(twin.ticks(flat) - 7 / flat.sample_period) <= 1
    o = des_port.simulate(load_scenario("c1_my_service.yml", 7), seed=SEED, replica=0)
    assert oracle_series_matrix(o, flat).shape[1] == twin.ticks(flat)


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_bands_equal_the_oracle_sums(name, engine):
    payload = load_scenario(name, PARITY_CASES[name])
    flat = flatten(payload)
    n, begin = 4, 2
    groups = np.array([1, 0, 1, 0], dtype=np.uint32)
    run = twin.run_lane if engine == "lane" else twin.run_warp
    out = run(flat, seed=SEED, n=n, replica_begin=begin, groups=groups, n_groups=2, band_first=begin, sampled=True)
    assert (out["stats"]["flags"] & STOPS == 0).all()
    mats = [oracle_matrix(payload, flat, begin + i) for i in range(n)]
    want = expected(flat, mats, groups, 2)
    assert (want[0] == 2).all()
    assert_bands(flat, out["band_rows"], 2, want)


def _overloaded():
    payload = load_scenario("overload_single.yml")
    return payload, flatten(payload)


def test_flagged_replicas_rerun_from_their_stop_tick_give_the_full_sums():
    payload, flat = _overloaded()
    n = 6
    groups = np.array([0, 1, 2, 0, 1, 2], dtype=np.uint32)
    lane = twin.run_lane(flat, seed=SEED, n=n, groups=groups, n_groups=3, event_capacity=24, request_capacity=12, lane_bytes=520,
                         sampled=True)
    flagged = np.flatnonzero(lane["stats"]["flags"] & REDO)
    assert flagged.size >= 1, "no replica stopped: the capacities do not force the second pass"
    assert all(0 < int(lane["band_from"][i]) < twin.ticks(flat) for i in flagged)
    out = twin.run_warp(flat, seed=SEED, n=n, groups=groups, n_groups=3, redo=flagged, band_from=lane["band_from"], into=lane,
                         sampled=True)
    assert (out["stats"]["flags"] & STOPS == 0).all()
    mats = [oracle_matrix(payload, flat, i) for i in range(n)]
    assert_bands(flat, out["band_rows"], 3, expected(flat, mats, groups, 3))
    # the stitched replicas' other outputs are the warp engine's first-hand ones
    full = twin.run_warp(flat, seed=SEED, n=n, groups=groups, n_groups=3, sampled=True)
    for k in ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr"):
        assert out[k].tobytes() == full[k].tobytes(), k


def test_a_stopped_replica_leaves_its_group_at_its_stop_tick():
    """Not re-run (LANE mode, or a flag the second pass does not take): the replica counts up to its stop tick, its sums
    are the oracle's truncated there, and the frozen ticks to the horizon add nothing."""
    payload, flat = _overloaded()
    n, T = 6, twin.ticks(flat)
    groups = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint32)
    out = twin.run_lane(flat, seed=SEED, n=n, groups=groups, n_groups=2, event_capacity=24, request_capacity=12, lane_bytes=520,
                        sampled=True)
    stopped = (out["stats"]["flags"] & STOPS) != 0
    assert stopped.any() and (out["stats"]["n_ticks"] == T).all()      # (n_ticks counts the frozen ticks)
    upto = np.where(stopped, out["band_from"], T).astype(np.int64)
    assert (upto[stopped] < T).all()
    mats = [oracle_matrix(payload, flat, i) for i in range(n)]
    assert_bands(flat, out["band_rows"], 2, expected(flat, mats, groups, 2, upto))
    cnt = band_ref.scan(flat, out["band_rows"], 2)[0]
    i = int(np.flatnonzero(stopped)[0])
    k, g = int(upto[i]), int(groups[i])
    assert cnt[g, k] < 3 and (cnt[g, :int(upto[groups == g].min())] == 3).all()


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_bands_change_no_other_output(engine):
    payload, flat = _overloaded()
    run = twin.run_lane if engine == "lane" else twin.run_warp
    kw = dict(seed=SEED, n=5, replica_begin=1, groups=np.array([0, 1, 0, 1, 0], dtype=np.uint32), n_groups=2,
              band_first=1, trace=3, clock_cap=5000, event_capacity=24, request_capacity=12)
    if engine == "lane":
        kw["lane_bytes"] = 520
    on, off = run(flat, sampled=True, **kw), run(flat, sampled=False, **kw)
    assert (on["stats"]["flags"] & STOPS).any()
    for k in twin.OUTPUTS:
        assert on[k].tobytes() == off[k].tobytes(), k
    assert not off["band_rows"].any() and on["band_rows"].any()


@pytest.mark.parametrize("seed", [3, 17, 41])
def test_fuzzed_scenarios_and_sweeps(seed):
    payload = fuzz.scenario(seed)
    flat = flatten(payload)
    n = 4
    spec = SweepSpec(flat, n, fuzz.sweep_columns(seed, payload, n))
    groups = np.array([0, 1, 1, 0], dtype=np.uint32)
    mats = [oracle_matrix(spec.payload_for(payload, i), flat, i) for i in range(n)]
    want = expected(flat, mats, groups, 2)
    for run in (twin.run_lane, twin.run_warp):
        out = run(flat, seed=SEED, n=n, sweep=spec, groups=groups, n_groups=2, sampled=True)
        assert (out["stats"]["flags"] & STOPS == 0).all()
        assert_bands(flat, out["band_rows"], 2, want)


def test_replicas_without_a_group_contribute_nothing():
    payload = load_scenario("c3_lb_two_servers.yml", 12)
    flat = flatten(payload)
    groups = np.array([0, 0], dtype=np.uint32)                 # replicas 1, 2 of 0..3
    out = twin.run_lane(flat, seed=SEED, n=4, groups=groups, n_groups=1, band_first=1, sampled=True)
    mats = [oracle_matrix(payload, flat, r) for r in (1, 2)]
    assert_bands(flat, out["band_rows"], 1, expected(flat, mats, groups, 1))


def test_sumsq_wrap_is_rejected_and_names_the_bound():
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    ok, bound, what = twin.sumsq_fits(flat, 1000, request_capacity=4096)
    assert ok and bound >= 4096
    ok, bound, what = twin.sumsq_fits(flat, 1 << 40, request_capacity=(1 << 20) - 1)
    assert not ok and bound == (1 << 20) - 1 and "request capacity" in what
    spec = SweepSpec(flat, 2, {("server_ram_mb", flat.server_ids[0]): [512.0, 2147483000.0]})
    ok, bound, what = twin.sumsq_fits(flat, 5, request_capacity=1024, sweep=spec)
    assert not ok and bound == 2147483000 and "swept ram_mb" in what
    assert twin.sumsq_fits(flat, 3, request_capacity=1024, sweep=spec)[0]


# ---- SweepRunner: groups are given per SWEEP ROW and follow the rows through the launch order ---------------------------
class BandTwinEngine(TwinEngine):
    """TwinEngine with the two band methods, on the band twin's lane engine."""

    def upload_bands(self, groups, first_replica: int = 0, n_groups=None) -> None:
        self.band_groups = None if groups is None else np.asarray(groups, dtype=np.uint32)
        self.band_first = int(first_replica)
        self.n_groups = n_groups if n_groups is not None or groups is None else int(self.band_groups.max()) + 1
        self.calls.append(("upload_bands", None if groups is None else self.band_groups.copy(), first_replica))

    def run(self, seed, begin, end) -> None:
        super().run(seed, begin, end)
        g = getattr(self, "band_groups", None)
        self._bands = None
        if g is not None:
            ng = self.n_groups
            out = twin.run_lane(self.flat, seed=seed, n=end - begin, replica_begin=begin, sweep=self.sweep, groups=g,
                                n_groups=ng, band_first=self.band_first, sampled=True)
            self._bands = band_ref.scan(self.flat, out["band_rows"], ng)

    def bands(self):
        return self._bands


USERS = [40.0, 250.0, 15.0, 120.0, 70.0, 180.0]


def _runner(**kw) -> SweepRunner:
    sw = SweepRunner(load_scenario("c1_my_service.yml", 5), len(USERS), {("users_mean",): USERS}, seed=SEED,
                     pinned=False, **kw)
    sw._engine = BandTwinEngine()
    sw._engine.upload(sw.flat)
    return sw


def test_sweep_runner_groups_rows_under_a_balanced_launch_order():
    row_group = np.array([0, 1, 2, 0, 1, 2])
    sw = _runner(balance=True, bands=row_group)
    assert sw.order is not None
    res = sw.run()
    up = [c for c in sw._engine.calls if c[0] == "upload_bands"][-1]
    assert np.array_equal(up[1][sw.replica_ids], row_group)        # replica id replica_ids[row] carries row's group
    mats = [oracle_matrix(sw.payload_for(r), sw.flat, int(sw.replica_ids[r])) for r in range(len(USERS))]
    want = expected(sw.flat, mats, row_group, 3)
    for a, b in zip((res.band_count, res.band_sum, res.band_sumsq), want):
        assert np.array_equal(a, b)
    gb = res.group_bands("ready_queue_len", sw.flat.server_ids[0])
    assert gb["mean"].shape == (3, twin.ticks(sw.flat)) and np.array_equal(gb["n"], want[0])
    s0 = want[1][:, 0, :].astype(np.float64)
    np.testing.assert_allclose(gb["mean"], s0 / 2)
    assert np.allclose(gb["t"], np.arange(twin.ticks(sw.flat)) * sw.flat.sample_period)


def test_sweep_runner_shard_maps_rows_through_replica_ids():
    sw = _runner(balance=True, deal=2, bands=True)
    res = sw.run(2, 5)                                              # replica ids 2, 3, 4
    rows = sw.rows_of(2, 5)
    assert res.band_count.shape[0] == 1 and (res.band_count == 3).all()
    mats = [oracle_matrix(sw.payload_for(int(r)), sw.flat, int(sw.replica_ids[int(r)])) for r in rows]
    want = expected(sw.flat, mats, [0, 0, 0], 1)
    assert np.array_equal(res.band_sum, want[1])


def test_group_bands_statistics():
    from asyncflow_b200.results import SweepResults
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    T, S = 4, flat.n_series
    res = SweepResults(flat, np.zeros(0, dtype=K.STATS_DTYPE), np.zeros((0, flat.n_edges)), np.zeros((0, flat.n_edges)),
                       np.zeros((0, S)), np.zeros((0, S)))
    vals = np.array([[1, 2, 3, 4], [3, 2, 5, 0], [2, 2, 1, 0]], dtype=np.uint64)     # three replicas, series 0
    res.band_count = np.array([[3, 3, 3, 1]], dtype=np.uint32)
    res.band_sum = np.zeros((1, S, T), dtype=np.uint64)
    res.band_sumsq = np.zeros((1, S, T), dtype=np.uint64)
    res.band_sum[0, 0] = vals.sum(axis=0) - np.array([0, 0, 0, 3])
    res.band_sumsq[0, 0] = (vals * vals).sum(axis=0) - np.array([0, 0, 0, 9])
    gb = res.group_bands("ready_queue_len", flat.server_ids[0], level=0.95)
    np.testing.assert_allclose(gb["mean"][0, :3], vals[:, :3].mean(axis=0))
    np.testing.assert_allclose(gb["std"][0, :3], vals[:, :3].std(axis=0, ddof=1))
    half = 1.959963984540054 * vals[:, :3].std(axis=0, ddof=1) / np.sqrt(3)
    np.testing.assert_allclose(gb["hi"][0, :3] - gb["mean"][0, :3], half)
    np.testing.assert_allclose(gb["mean"][0, :3] - gb["lo"][0, :3], half)
    assert gb["mean"][0, 3] == 1.0 and np.isnan(gb["std"][0, 3]) and np.isnan(gb["lo"][0, 3]) and np.isnan(gb["hi"][0, 3])


def test_outage_example_dry_run(monkeypatch, capsys):
    """examples/sweep_outage_bands.py on the band twin (two repetitions per spike size), so its plumbing cannot rot."""
    import runpy
    import sys

    import asyncflow_b200.runner as R
    from helpers import ROOT
    monkeypatch.setattr(R, "Engine", lambda device=0: BandTwinEngine(device))
    monkeypatch.setattr(sys, "argv", ["sweep_outage_bands.py", "2"])
    runpy.run_path(str(ROOT / "examples" / "sweep_outage_bands.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "6 replicas (2 per spike size)" in out and "   180 |" in out and "nan" not in out.split("   180 |")[1].split("\n")[0]


def test_bench_bands_tool_dry_run(monkeypatch, capsys):
    """tools/bench_bands.py on the band twin (a few replicas of the bench workload), so its plumbing cannot rot."""
    import runpy
    import sys

    import asyncflow_b200.runner as R
    from helpers import ROOT
    monkeypatch.setattr(R, "Engine", lambda device=0: BandTwinEngine(device))
    monkeypatch.setattr(sys, "argv", ["bench_bands.py", "--replicas", "6", "--horizon", "3", "--groups", "1,3", "--reps", "2"])
    runpy.run_path(str(ROOT / "tools" / "bench_bands.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "bands G=3" in out and "identical with bands on and off: True" in out
    import json
    row = json.loads(out.strip().splitlines()[-1])
    assert row["outputs_identical"] and row["off"] > 0 and row["G3"] > 0


def test_a_horizon_with_more_ticks_than_the_band_rows_hold_is_refused():
    payload = load_scenario("c1_my_service.yml", 86_400)
    payload["sim_settings"]["sample_period_s"] = 0.001
    flat = flatten(payload)
    assert twin.ticks(flat) == 50_000_000
    ok, why = twin.ticks_fit(flat)
    assert not ok and "86400" in why and "ticks or more" in why
    with pytest.raises(RuntimeError, match="ticks or more"):
        twin.run_lane(flat, seed=SEED, n=1, groups=np.zeros(1, dtype=np.uint32), n_groups=1, sampled=True)
    payload["sim_settings"]["total_simulation_time"] = 49_000                        # 4.9e7 ticks: they fit
    assert twin.ticks_fit(flatten(payload))[0]
