"""Request deadlines and the client timeout (DESIGN.md §3.13) on the CPU: the oracle's specification
(tests/des_deadline.py), both state machines of the twin bit for bit against it, the equivalences that make a deadline
free when it cannot fire, the accounting of every request, each refusal in Python and in C, and the front end."""

from __future__ import annotations

import zlib
from pathlib import Path

import des_admission
import des_deadline
import fuzz
import numpy as np
import pytest
import twin_deadline
from helpers import SCEN, SEED, assert_matches_oracle, load_scenario

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten, set_admission, set_deadlines
from asyncflow_b200.results import SweepResults

ROOT = Path(__file__).resolve().parent.parent
OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "rejected", "expired", "late")
CASES = [("c1_my_service.yml", 20), ("c3_lb_two_servers.yml", 30), ("c4_lb8_events.yml", 20), ("mixed_lc.yml", None),
         ("chain_two_servers.yml", None), ("c5_multihop32.yml", 4), ("tie_cpu_io.yml", None)] + \
        [f"fuzz:{s}" for s in (302, 322, 329)]
BUILDS = ["lane", "warp"]      # (a launch with a deadline runs the full lane build: aflh::lean_launch)


def _payload(case):
    if isinstance(case, str) and case.startswith("fuzz:"):
        return fuzz.scenario(int(case[5:]))
    return load_scenario(*case)


def _run(flat, build, **kw):
    if build == "lane":
        return twin_deadline.run_lane(flat, event_capacity=4096, request_capacity=200000, **kw)
    return twin_deadline.run_warp(flat, **kw)


def _oracle(payload, replica, ov):
    return des_deadline.simulate(payload, seed=SEED, replica=replica, admission=ov["admission"],
                                 deadline=ov["deadline"], client_timeout=ov["client_timeout"])


def _check(o: dict, flat, r: dict, i: int, traced: bool = False) -> None:
    """Replica i of twin launch r equals oracle run o (its clocks and series too when it was traced)."""
    st = r["stats"][i]
    k, nt = int(st["completed"]), int(st["n_ticks"])
    assert st["flags"] == 0
    assert_matches_oracle(o, flat, stats=st, clocks=r["trace_clocks"][i, :k] if traced else None, sent=r["sent"][i],
                          dropped=r["dropped"][i], throughput=r["thr"][i],
                          series=r["trace_series"][i][:, :nt] if traced else None)
    assert [int(x) for x in r["rejected"][i]] == [o["server_rejected"][s] for s in flat.server_ids]
    assert [int(x) for x in r["expired"][i]] == [o["server_expired"][s] for s in flat.server_ids]
    assert int(r["late"][i]) == o["late"]


def _latencies(payload) -> np.ndarray:
    o = des_deadline.simulate(payload, seed=SEED, replica=0)
    lat = np.array([b - a for a, b in o["clocks"]], dtype=np.float64)
    return lat if lat.size else np.array([1.0])


# ---- the oracle ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(p.name for p in SCEN.glob("*.yml")))
def test_no_deadline_is_the_admission_oracle_unchanged(name):
    payload = load_scenario(name, 10)
    ref = des_admission.simulate(payload, seed=SEED, replica=1)
    servers = [s["id"] for s in payload["topology_graph"]["nodes"]["servers"]]
    for deadline, timeout in ((None, None), ({}, 0.0), (dict.fromkeys(servers, 0.0), 0.0), (dict.fromkeys(servers, 10.0), 10.0)):
        o = des_deadline.simulate(payload, seed=SEED, replica=1, deadline=deadline, client_timeout=timeout)
        assert o.pop("server_expired") == dict.fromkeys(servers, 0)
        assert o.pop("late") == 0
        assert o == ref


def _two_at_once(horizon: int = 2) -> dict:
    """One server, one core, 64 MB of RAM per request, one 0.5 s CPU step; two users firing ~ together."""
    edge = lambda i, s, t: {"id": i, "source": s, "target": t, "latency": {"mean": 0.001, "distribution": "exponential"},  # noqa: E731
                            "dropout_rate": 0.0}
    return {
        "rqs_input": {"id": "gen", "avg_active_users": {"mean": 2000}, "avg_request_per_minute_per_user": {"mean": 60}},
        "topology_graph": {
            "nodes": {"client": {"id": "client"},
                      "servers": [{"id": "srv", "server_resources": {"cpu_cores": 1, "ram_mb": 1 << 20},
                                   "endpoints": [{"endpoint_name": "/x", "steps": [
                                       {"kind": "ram", "step_operation": {"necessary_ram": 64}},
                                       {"kind": "cpu_bound_operation", "step_operation": {"cpu_time": 0.5}}]}]}]},
            "edges": [edge("gen-client", "gen", "client"), edge("client-srv", "client", "srv"),
                      edge("srv-client", "srv", "client")]},
        "sim_settings": {"total_simulation_time": horizon, "sample_period_s": 0.1,
                         "enabled_sample_metrics": ["ram_in_use", "ready_queue_len", "event_loop_io_sleep"]},
    }


def test_a_request_that_waited_past_its_deadline_expires_when_it_gets_the_core():
    p = _two_at_once(1)
    free = des_deadline.simulate(p, seed=SEED, replica=0)
    o = des_deadline.simulate(p, seed=SEED, replica=0, deadline={"srv": 0.25})
    assert o["generated"] == free["generated"] > 2
    # the first request is served (age ~0 at its check), the second waited 0.5 s for the core: it expires when it gets
    # it, at once, and so does every waiter older than 0.25 s (~500 of them, ~2000 arrivals per second) at that same
    # instant; the first younger one keeps the core and finishes after the 1 s horizon
    assert o["completed"] == 1 and o["clocks"][0] == free["clocks"][0]
    assert 400 < o["server_expired"]["srv"] < 600
    assert o["edge_sent"]["srv-client"] == 1
    # its RAM went back: nothing is held at the end but what the requests still in service hold
    ram = o["server_series"]["srv"]["ram_in_use"]
    assert max(ram) <= 64 * (o["edge_sent"]["client-srv"] - o["server_expired"]["srv"])


def test_the_deadline_is_strict():
    p = load_scenario("c3_lb_two_servers.yml", 30)
    sid = p["topology_graph"]["nodes"]["servers"][0]["id"]
    ages: list = []
    des_deadline.simulate(p, seed=SEED, replica=3, ages=ages)
    age = max(a for s, _, a in ages if s == sid)
    assert age > 0.0
    at = des_deadline.simulate(p, seed=SEED, replica=3, deadline={sid: age})
    below = des_deadline.simulate(p, seed=SEED, replica=3, deadline={sid: float(np.nextafter(age, 0.0))})
    assert at["server_expired"][sid] == 0
    assert below["server_expired"][sid] >= 1
    # and both state machines draw the line at the same f64
    flat = flatten(p)
    for d, o in ((age, at), (float(np.nextafter(age, 0.0)), below)):
        set_deadlines(flat, {sid: d})
        for build in BUILDS:
            r = _run(flat, build, seed=SEED, n=1, replica_begin=3)
            _check(o, flat, r, 0)


def test_the_client_counts_late_completions_from_the_clocks():
    p = load_scenario("c3_lb_two_servers.yml", 30)
    lat = _latencies(p)
    t = float(np.quantile(lat, 0.7))
    o = des_deadline.simulate(p, seed=SEED, replica=0, client_timeout=t)
    assert o["late"] == sum(1 for a, b in o["clocks"] if b - a > t) > 0
    assert o["completed"] == des_admission.simulate(p, seed=SEED, replica=0)["completed"]


def test_oracle_refuses_unknown_servers_and_bad_values():
    p = load_scenario("c1_my_service.yml", 5)
    sid = p["topology_graph"]["nodes"]["servers"][0]["id"]
    with pytest.raises(KeyError, match="nope"):
        des_deadline.simulate(p, seed=SEED, replica=0, deadline={"nope": 1.0})
    for bad in (-1.0, float("nan"), float("inf"), True):
        with pytest.raises(ValueError):
            des_deadline.simulate(p, seed=SEED, replica=0, deadline={sid: bad})
        with pytest.raises(ValueError):
            des_deadline.simulate(p, seed=SEED, replica=0, client_timeout=bad)


# ---- both state machines against the oracle -------------------------------------------------------------------------------
def _deadline_columns(flat, payload, n: int, rng, caps: bool) -> dict:
    lat = _latencies(payload)
    choices = np.array([0.0, *np.quantile(lat, [0.05, 0.3, 0.6, 0.9])])
    cols = {("server_deadline", s): rng.choice(choices, n) for s in flat.server_ids}
    cols[("client_timeout",)] = rng.choice(choices, n)
    if caps:
        cols.update({("server_max_in_service", s): rng.integers(0, 6, n).astype(float) for s in flat.server_ids})
    return cols


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("case", CASES, ids=str)
def test_rows_equal_the_oracle(case, build):
    payload = _payload(case)
    flat = flatten(payload)
    n = 6
    h = zlib.crc32(str(case).encode())
    rng = np.random.default_rng(h)
    cols = _deadline_columns(flat, payload, n, rng, caps=h % 2 == 0)
    cols[("users_mean",)] = rng.choice([1.0, 2.0, 4.0], n) * float(flat.pod.users_mean)
    spec = SweepSpec(flat, n, cols)
    streams = [5, 5, 9, 5, 2, 9]                  # rows sharing a stream see the same traffic whatever their deadlines
    r = _run(flat, build, seed=SEED, n=n, sweep=spec, streams=streams, trace=n, clock_cap=200000)
    expired = late = 0
    for i in range(n):
        p, ov = spec.payload_and_overload(payload, i)
        o = _oracle(p, streams[i], ov)
        _check(o, flat, r, i, traced=True)
        expired += sum(o["server_expired"].values())
        late += o["late"]
    assert late > 0, "no row had a late completion: the case does not exercise the timeout"
    if case not in (("c5_multihop32.yml", 4),):
        assert expired > 0, "no row dropped a request: the case does not exercise the deadline"


@pytest.mark.parametrize("build", BUILDS)
def test_scenario_deadlines_with_caps_equal_the_oracle(build):
    payload = load_scenario("mixed_lc.yml")
    flat = flatten(payload)
    lat = _latencies(payload)
    adm = {s: 1 + i for i, s in enumerate(flat.server_ids)}
    dl = {s: float(np.quantile(lat, 0.2 + 0.2 * i)) for i, s in enumerate(flat.server_ids)}
    t = float(np.quantile(lat, 0.5))
    set_admission(flat, adm)
    set_deadlines(flat, dl, client_timeout=t)
    r = _run(flat, build, seed=SEED, n=3, trace=3, clock_cap=200000)
    for i in range(3):
        o = des_deadline.simulate(payload, seed=SEED, replica=i, admission=adm, deadline=dl, client_timeout=t)
        _check(o, flat, r, i, traced=True)
        assert (np.array([b - a for a, b in o["clocks"]]) > t).sum() == int(r["late"][i])


def test_rows_with_bands_occupancy_lb_and_event_rows():
    payload = load_scenario("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    n = 4
    rng = np.random.default_rng(4)
    cols = _deadline_columns(flat, payload, n, rng, caps=True)
    cols[("lb_algorithm",)] = ["round_robin", "least_connection", "round_robin", "least_connection"]
    cols[("event_start", "ev-srv3-down")] = [2.0, 6.0, 2.0, 6.0]
    cols[("event_end", "ev-srv3-down")] = [9.0, 14.0, 14.0, 9.0]
    cols[("event_start", "ev-spike")] = np.full(n, 4.0)
    cols[("event_end", "ev-spike")] = np.full(n, 11.0)
    spec = SweepSpec(flat, n, cols)
    kw = dict(seed=SEED, n=n, sweep=spec, streams=[1, 1, 1, 1], groups=np.array([0, 1, 0, 1]), n_groups=2,
              sampled=True, window=5, series=[0, 3 * flat.n_servers], f=20)
    for build in BUILDS:
        r = _run(flat, build, **kw)
        for i in range(n):
            p, ov = spec.payload_and_overload(payload, i)
            _check(_oracle(p, 1, ov), flat, r, i)
        assert r["occ"].any() and r["band_rows"].any() and r["lat_rows"].any() and r["dist_rows"].any()
        assert r["expired"].any() and r["late"].any()


def test_pool_splits_and_occupancies_give_the_same_results():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 6
    spec = SweepSpec(flat, n, _deadline_columns(flat, payload, n, np.random.default_rng(9), caps=True))
    ref = _run(flat, "lane", seed=SEED, n=n, sweep=spec)
    for lane_bytes, split in ((1000, "random"), (4000, "rows"), (1816, "scenario")):
        r = twin_deadline.run_lane(flat, seed=SEED, n=n, sweep=spec, event_capacity=4096, request_capacity=200000,
                                   lane_bytes=lane_bytes, split=split, split_seed=3)
        for k in OUT:
            np.testing.assert_array_equal(ref[k], r[k], err_msg=f"{k} {lane_bytes} {split}")


def test_a_warp_rerun_keeps_writing_the_counts():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 4
    spec = SweepSpec(flat, n, _deadline_columns(flat, payload, n, np.random.default_rng(2), caps=False))
    ref = _run(flat, "warp", seed=SEED, n=n, sweep=spec)
    out = _run(flat, "lane", seed=SEED, n=n, sweep=spec)
    out["expired"][[1, 3]] = 0
    out["late"][[1, 3]] = 0
    twin_deadline.run_warp(flat, seed=SEED, n=n, sweep=spec, redo=[1, 3], into=out)
    np.testing.assert_array_equal(out["expired"], ref["expired"])
    np.testing.assert_array_equal(out["late"], ref["late"])


# ---- equivalences -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build", BUILDS)
def test_a_zero_column_or_one_past_the_horizon_is_no_column(build):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    n = 4
    users = {("users_mean",): np.array([1.0, 3.0, 6.0, 10.0]) * float(flat.pod.users_mean)}
    plain = SweepSpec(flat, n, users)
    kw = dict(seed=SEED, n=n, groups=np.array([0, 1, 0, 1]), n_groups=2, sampled=True, window=5, series=[1], f=24)
    a = _run(flat, build, sweep=plain, **kw)
    assert not twin_deadline.deadline_launch(flat, plain)
    for v in (0.0, float(flat.horizon_s), 1e9):
        cols = {**users, **{("server_deadline", s): np.full(n, v) for s in flat.server_ids}, ("client_timeout",): np.full(n, v)}
        spec = SweepSpec(flat, n, cols)
        assert twin_deadline.deadline_launch(flat, spec) and not twin_deadline.lean_launch(flat, spec)
        b = _run(flat, build, sweep=spec, **kw)
        for k in (*OUT, "band_rows", "lat_rows", "dist_rows", "occ"):
            if k in ("expired", "late"):
                assert not b[k].any()
            else:
                np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} {v}")


def test_rows_of_one_stream_draw_the_same_arrivals_whatever_their_deadline():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 4
    lat = _latencies(payload)
    spec = SweepSpec(flat, n, {("users_mean",): np.full(n, 4.0 * float(flat.pod.users_mean)),
                               ("server_deadline", flat.server_ids[0]): [0.0, *np.quantile(lat, [0.1, 0.5, 0.9])]})
    r = twin_deadline.run(flat, seed=SEED, n=n, sweep=spec, streams=[8] * n)
    gen_edge = flat.pod.gen_edge
    assert len(set(r["stats"]["generated"].tolist())) == 1
    assert len(set(r["sent"][:, gen_edge].tolist())) == 1
    assert r["expired"][0].sum() == 0 and r["expired"][1].sum() >= r["expired"][2].sum() >= r["expired"][3].sum()
    assert r["expired"][1].sum() > 0


@pytest.mark.parametrize("build", BUILDS)
def test_every_request_is_accounted_for(build):
    payload = load_scenario("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    n = 8
    rng = np.random.default_rng(11)
    spec = SweepSpec(flat, n, {**_deadline_columns(flat, payload, n, rng, caps=True),
                               ("users_mean",): rng.choice([1.0, 3.0], n) * float(flat.pod.users_mean)})
    r = _run(flat, build, seed=SEED, n=n, sweep=spec, trace=2, clock_cap=200000)
    st = r["stats"]
    gone = st["completed"].astype(np.int64) + r["dropped"].sum(axis=1) + r["rejected"].sum(axis=1) + r["expired"].sum(axis=1)
    assert (gone <= st["generated"]).all()
    assert (r["late"] <= st["completed"]).all()
    assert r["expired"].sum() > 0 and r["late"].sum() > 0
    for i in range(2):                              # traced: late = completions with finish - start > T
        k = int(st["completed"][i])
        c = r["trace_clocks"][i, :k]
        t = spec.deadlines_for(i)[1]
        assert int(r["late"][i]) == (int(((c[:, 1] - c[:, 0]) > t).sum()) if t else 0)


def test_a_launch_with_a_deadline_or_a_timeout_runs_the_full_lane_build():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin_deadline.lean_launch(flat) and not twin_deadline.deadline_launch(flat)
    set_deadlines(flat, {flat.server_ids[0]: 0.0}, client_timeout=0.0)
    assert twin_deadline.lean_launch(flat) and not twin_deadline.deadline_launch(flat)
    set_deadlines(flat, {flat.server_ids[0]: 0.5})
    assert not twin_deadline.lean_launch(flat) and twin_deadline.deadline_launch(flat)
    set_deadlines(flat, {flat.server_ids[0]: 0.0}, client_timeout=2.0)
    assert not twin_deadline.lean_launch(flat) and twin_deadline.deadline_launch(flat)
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    spec = SweepSpec(flat, 2, {("client_timeout",): [0.0, 0.0]})
    assert not twin_deadline.lean_launch(flat, spec) and twin_deadline.deadline_launch(flat, spec)


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [-1, -0.5, np.nan, np.inf, True, "soon"])
def test_python_refuses_a_bad_value_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    with pytest.raises(ValueError, match="sweep row 1"):
        SweepSpec(flat, 3, {("server_deadline", flat.server_ids[0]): [2, bad, 3]})
    with pytest.raises(ValueError, match="sweep row 1"):
        SweepSpec(flat, 3, {("client_timeout",): [2, bad, 3]})
    with pytest.raises(ValueError, match="deadline"):
        set_deadlines(flat, {flat.server_ids[0]: bad})
    with pytest.raises(ValueError, match="client_timeout"):
        set_deadlines(flat, None, client_timeout=bad)


def test_python_refuses_an_unknown_server():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    with pytest.raises(KeyError, match="nope"):
        SweepSpec(flat, 2, {("server_deadline", "nope"): [1, 2]})
    with pytest.raises(KeyError, match="nope"):
        set_deadlines(flat, {"nope": 1.0})


@pytest.mark.parametrize("bad", [-1.0, -1e-300, np.nan, np.inf, -np.inf])
def test_c_refuses_a_bad_value_naming_the_row(bad):
    for field in K.DEADLINE_FIELDS.values():
        assert twin_deadline.sweep_fits([(field, 0)], [[0.0], [7.5]]) is None
        why = twin_deadline.sweep_fits([(field, 0)], [[1.0], [bad]])
        assert why is not None and "row 1" in why


def test_c_refuses_bad_scenario_values():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin_deadline.validate(flat) is None
    for bad in (-1.0, np.nan, np.inf):
        flat.pod.servers[1].deadline = bad
        assert "deadline" in twin_deadline.validate(flat)
        flat.pod.servers[1].deadline = 0.0
        flat.pod.client_timeout = bad
        assert "client_timeout" in twin_deadline.validate(flat)
        flat.pod.client_timeout = 0.0
    assert twin_deadline.validate(flat) is None


# ---- front end --------------------------------------------------------------------------------------------------------------
def test_payload_for_refuses_a_deadline_row_and_payload_and_overload_gives_it():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    s0, s1 = flat.server_ids
    spec = SweepSpec(flat, 3, {("server_deadline", s0): [0.0, 0.4, 0.0], ("client_timeout",): [0.0, 0.0, 1.5],
                               ("server_max_in_service", s1): [0, 0, 3], ("users_mean",): [10.0, 20.0, 30.0]})
    assert spec.payload_for(payload, 0)["rqs_input"]["avg_active_users"]["mean"] == 10.0
    for i in (1, 2):
        with pytest.raises(ValueError, match="payload_and_overload"):
            spec.payload_for(payload, i)
        with pytest.raises(ValueError, match="payload_and_overload"):
            spec.payload_and_admission(payload, i)
    p, ov = spec.payload_and_overload(payload, 2)
    assert ov == {"admission": {s1: 3}, "deadline": {s0: 0.0}, "client_timeout": 1.5}
    assert p["rqs_input"]["avg_active_users"]["mean"] == 30.0 and p["topology_graph"] == payload["topology_graph"]


def test_sweep_runner_front_end():
    from asyncflow_b200 import runner as R
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    s0 = flatten(payload).server_ids[0]
    sr = R.SweepRunner(payload, 3, {("server_deadline", s0): [0.0, 0.2, 0.5], ("client_timeout",): [1.0, 1.0, 2.0]},
                       streams=[4, 4, 6])
    p, ov = sr.payload_and_overload(2)
    assert ov["deadline"] == {s0: 0.5} and ov["client_timeout"] == 2.0
    run = sr.replica_runner(2)
    assert run.deadline == {s0: 0.5} and run.client_timeout == 2.0 and run.replica == 6
    assert run.simulation_input == p
    n, ns = 3, sr.flat.n_servers
    res = SweepResults(sr.flat, np.zeros(n, K.STATS_DTYPE), np.zeros((n, sr.flat.n_edges), np.uint32),
                       np.zeros((n, sr.flat.n_edges), np.uint32), np.zeros((n, sr.flat.n_series), np.uint64),
                       np.zeros((n, sr.flat.n_series), np.uint32))
    assert res.server_expired.shape == (n, ns) and res.late.shape == (n,)
    res.stats["completed"] = [10, 20, 30]
    res.server_expired = np.arange(n * ns, dtype=np.uint32).reshape(n, ns)
    res.late = np.array([1, 2, 3], dtype=np.uint32)
    res.rows = np.arange(n)
    pytest.importorskip("pandas")
    df = sr.frame(res)
    assert df[f"server_deadline:{s0}"].tolist() == [0.0, 0.2, 0.5] and df["client_timeout"].tolist() == [1.0, 1.0, 2.0]
    assert df["expired"].tolist() == res.server_expired.sum(axis=1).tolist()
    assert df["late"].tolist() == [1, 2, 3] and df["goodput"].tolist() == [9, 18, 27]
    t = res.take([2, 0])
    np.testing.assert_array_equal(t.server_expired, res.server_expired[[2, 0]])
    np.testing.assert_array_equal(t.late, res.late[[2, 0]])
    c = SweepResults.concatenate([res.take([0]), res.take([1, 2])])
    np.testing.assert_array_equal(c.server_expired, res.server_expired)
    np.testing.assert_array_equal(c.late, res.late)


def test_the_example_and_the_tool_dry_run():
    import subprocess
    import sys
    for script in ("examples/sweep_deadline.py", "tools/bench_deadline.py"):
        r = subprocess.run([sys.executable, str(ROOT / script), "--dry-run"], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr
