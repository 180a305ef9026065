"""Admission limits (DESIGN.md §3.12) on the CPU: the oracle's specification (tests/des_admission.py), both state machines
of the twin bit for bit against it, the equivalences that make a limit free when it does not bind, the accounting of
every request, each refusal in Python and in C, and the front end."""

from __future__ import annotations

import zlib
from pathlib import Path

import des_admission
import des_port
import fuzz
import numpy as np
import pytest
import twin_admission
from helpers import SCEN, SEED, assert_matches_oracle, load_scenario

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten, set_admission
from asyncflow_b200.results import SweepResults

ROOT = Path(__file__).resolve().parent.parent
OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "rejected")
CASES = [("c1_my_service.yml", 20), ("c3_lb_two_servers.yml", 30), ("c4_lb8_events.yml", 20), ("mixed_lc.yml", None),
         ("c5_multihop32.yml", 4)] + [f"fuzz:{s}" for s in (302, 322, 329)]
BUILDS = ["lane", "warp"]      # (a launch with a limit runs the full lane build: aflh::lean_launch)


def _payload(case):
    if isinstance(case, str) and case.startswith("fuzz:"):
        return fuzz.scenario(int(case[5:]))
    return load_scenario(*case)


def _run(flat, build, **kw):
    if build == "lane":
        return twin_admission.run_lane(flat, event_capacity=4096, request_capacity=200000, **kw)
    return twin_admission.run_warp(flat, **kw)


def _check(o: dict, flat, r: dict, i: int, traced: bool = False) -> None:
    """Replica i of twin launch r equals oracle run o (its clocks and series too when it was traced)."""
    st = r["stats"][i]
    k, nt = int(st["completed"]), int(st["n_ticks"])
    assert st["flags"] == 0
    assert_matches_oracle(o, flat, stats=st, clocks=r["trace_clocks"][i, :k] if traced else None, sent=r["sent"][i],
                          dropped=r["dropped"][i], throughput=r["thr"][i],
                          series=r["trace_series"][i][:, :nt] if traced else None)
    assert [int(x) for x in r["rejected"][i]] == [o["server_rejected"][s] for s in flat.server_ids]


# ---- the oracle ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(p.name for p in SCEN.glob("*.yml")))
def test_no_limit_is_the_oracle_unchanged(name):
    payload = load_scenario(name, 10)
    ref = des_port.simulate(payload, seed=SEED, replica=1)
    servers = [s["id"] for s in payload["topology_graph"]["nodes"]["servers"]]
    for admission in (None, {}, dict.fromkeys(servers, 0)):
        o = des_admission.simulate(payload, seed=SEED, replica=1, admission=admission)
        assert o.pop("server_rejected") == dict.fromkeys(servers, 0)
        assert o == ref


def _two_at_once(horizon: int = 2) -> dict:
    """One server, one core, one 0.5 s CPU step; two users firing ~ together; edges with no spread and no dropout."""
    edge = lambda i, s, t: {"id": i, "source": s, "target": t, "latency": {"mean": 0.001, "distribution": "exponential"},  # noqa: E731
                            "dropout_rate": 0.0}
    return {
        "rqs_input": {"id": "gen", "avg_active_users": {"mean": 2000}, "avg_request_per_minute_per_user": {"mean": 60}},
        "topology_graph": {
            "nodes": {"client": {"id": "client"},
                      "servers": [{"id": "srv", "server_resources": {"cpu_cores": 1, "ram_mb": 1024},
                                   "endpoints": [{"endpoint_name": "/x", "steps": [
                                       {"kind": "cpu_bound_operation", "step_operation": {"cpu_time": 0.5}}]}]}]},
            "edges": [edge("gen-client", "gen", "client"), edge("client-srv", "client", "srv"),
                      edge("srv-client", "srv", "client")]},
        "sim_settings": {"total_simulation_time": horizon, "sample_period_s": 0.1},
    }


def test_a_limit_of_one_sheds_what_arrives_while_one_is_in_service():
    p = _two_at_once(1)
    free = des_admission.simulate(p, seed=SEED, replica=0)
    capped = des_admission.simulate(p, seed=SEED, replica=0, admission={"srv": 1})
    assert free["generated"] == capped["generated"] > 2
    # one request in service for 0.5 s at a time, ~2000 arrivals per second: the first two arrive within a millisecond,
    # so the first is served and the second shed.  In a 1 s horizon the server admits one request per 0.5 s; what it
    # neither admitted nor shed was still on its in-edge at the horizon
    assert capped["completed"] == 1 and capped["clocks"][0] == free["clocks"][0]
    assert free["edge_sent"]["srv-client"] == 1 and free["completed"] == 1
    admitted = capped["edge_sent"]["client-srv"] - capped["server_rejected"]["srv"]
    assert capped["server_rejected"]["srv"] > 2000 and 1 <= admitted <= 3
    assert capped["edge_sent"]["srv-client"] == 1


def test_oracle_refuses_unknown_servers_and_bad_limits():
    p = load_scenario("c1_my_service.yml", 5)
    sid = p["topology_graph"]["nodes"]["servers"][0]["id"]
    with pytest.raises(KeyError, match="nope"):
        des_admission.simulate(p, seed=SEED, replica=0, admission={"nope": 1})
    for bad in (1.5, -1):
        with pytest.raises(ValueError):
            des_admission.simulate(p, seed=SEED, replica=0, admission={sid: bad})


# ---- both state machines against the oracle -------------------------------------------------------------------------------
def _cap_columns(flat, n: int, rng, kind: str) -> dict:
    if kind == "one":
        vals = np.ones(n)
    elif kind == "two":
        vals = np.full(n, 2.0)
    elif kind == "small":
        vals = rng.integers(0, 4, n).astype(float)
    else:
        vals = rng.integers(0, 40, n).astype(float)
    return {("server_max_in_service", s): rng.permutation(vals) for s in flat.server_ids}


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("case", CASES, ids=str)
def test_rows_equal_the_oracle(case, build):
    payload = _payload(case)
    flat = flatten(payload)
    n = 6
    rng = np.random.default_rng(zlib.crc32(str(case).encode()))
    cols = _cap_columns(flat, n, rng, ["one", "two", "small", "random"][zlib.crc32(str(case).encode()) % 4])
    cols[("users_mean",)] = rng.choice([1.0, 2.0, 4.0], n) * float(flat.pod.users_mean)
    spec = SweepSpec(flat, n, cols)
    streams = [5, 5, 9, 5, 2, 9]                         # rows sharing a stream see the same traffic whatever the cap
    trace = n
    r = _run(flat, build, seed=SEED, n=n, sweep=spec, streams=streams, trace=trace, clock_cap=200000)
    shed = 0
    for i in range(n):
        p, adm = spec.payload_and_admission(payload, i)
        o = des_admission.simulate(p, seed=SEED, replica=streams[i], admission=adm)
        _check(o, flat, r, i, traced=trace > 0)
        shed += sum(o["server_rejected"].values())
    assert shed > 0, "no row shed a request: the case does not exercise the limit"


@pytest.mark.parametrize("build", BUILDS)
def test_scenario_limits_equal_the_oracle(build):
    payload = load_scenario("mixed_lc.yml")
    flat = flatten(payload)
    adm = {s: 1 + i for i, s in enumerate(flat.server_ids)}
    set_admission(flat, adm)
    r = _run(flat, build, seed=SEED, n=3, trace=3, clock_cap=200000)
    for i in range(3):
        _check(des_admission.simulate(payload, seed=SEED, replica=i, admission=adm), flat, r, i, traced=True)


def test_rows_with_bands_occupancy_lb_and_event_rows():
    payload = load_scenario("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    n = 4
    rng = np.random.default_rng(4)
    cols = _cap_columns(flat, n, rng, "small")
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
            p, adm = spec.payload_and_admission(payload, i)
            _check(des_admission.simulate(p, seed=SEED, replica=1, admission=adm), flat, r, i)
        assert r["occ"].any() and r["band_rows"].any() and r["lat_rows"].any() and r["dist_rows"].any()
        assert r["rejected"].any()


# ---- equivalences -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build", BUILDS)
def test_a_zero_column_is_no_column(build):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    n = 4
    users = {("users_mean",): np.array([1.0, 3.0, 6.0, 10.0]) * float(flat.pod.users_mean)}
    plain = SweepSpec(flat, n, users)
    zeros = SweepSpec(flat, n, {**users, **{("server_max_in_service", s): np.zeros(n) for s in flat.server_ids}})
    assert not twin_admission.admission_launch(flat, plain) and twin_admission.admission_launch(flat, zeros)
    kw = dict(seed=SEED, n=n, groups=np.array([0, 1, 0, 1]), n_groups=2, sampled=True, window=5, series=[1], f=24)
    a, b = _run(flat, build, sweep=plain, **kw), _run(flat, build, sweep=zeros, **kw)
    for k in (*OUT, "band_rows", "lat_rows", "dist_rows", "occ"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


@pytest.mark.parametrize("build", BUILDS)
def test_a_limit_that_never_binds_changes_nothing(build):
    payload = load_scenario("mixed_lc.yml")
    flat = flatten(payload)
    n = 3
    free = _run(flat, build, seed=SEED, n=n)
    # the most requests a server ever holds is below everything in flight at once: the replica's peak of records
    peak = int(free["stats"]["peak_requests"].max())
    spec = SweepSpec(flat, n, {("server_max_in_service", s): np.full(n, peak) for s in flat.server_ids})
    capped = _run(flat, build, seed=SEED, n=n, sweep=spec)
    for k in OUT:
        np.testing.assert_array_equal(free[k], capped[k], err_msg=k)
    assert not capped["rejected"].any()


def test_rows_of_one_stream_draw_the_same_arrivals_whatever_their_cap():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    n = 4
    spec = SweepSpec(flat, n, {("users_mean",): np.full(n, 4.0 * float(flat.pod.users_mean)),
                               ("server_max_in_service", flat.server_ids[0]): [0, 1, 3, 10]})
    r = twin_admission.run(flat, seed=SEED, n=n, sweep=spec, streams=[8] * n)
    gen_edge = flat.pod.gen_edge
    assert len(set(r["stats"]["generated"].tolist())) == 1
    assert len(set(r["sent"][:, gen_edge].tolist())) == 1
    assert r["rejected"][0].sum() == 0 and r["rejected"][1].sum() > r["rejected"][2].sum() >= r["rejected"][3].sum()


@pytest.mark.parametrize("build", BUILDS)
def test_every_request_is_accounted_for(build):
    flat = flatten(load_scenario("c4_lb8_events.yml", 20))
    n = 8
    rng = np.random.default_rng(11)
    spec = SweepSpec(flat, n, {**_cap_columns(flat, n, rng, "small"),
                               ("users_mean",): rng.choice([1.0, 3.0], n) * float(flat.pod.users_mean)})
    r = _run(flat, build, seed=SEED, n=n, sweep=spec)
    gone = r["stats"]["completed"].astype(np.int64) + r["dropped"].sum(axis=1) + r["rejected"].sum(axis=1)
    assert (gone <= r["stats"]["generated"]).all()
    assert r["rejected"].sum() > 0


def test_a_launch_with_a_limit_runs_the_full_lane_build():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin_admission.twin.lean_qualifies(flat)
    set_admission(flat, {flat.server_ids[0]: 0})
    assert twin_admission.twin.lean_qualifies(flat)
    set_admission(flat, {flat.server_ids[0]: 3})
    assert not twin_admission.twin.lean_qualifies(flat) and twin_admission.admission_launch(flat)


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [-1, 1.5, np.nan, np.inf, 2.0 ** 31, True, "three"])
def test_python_refuses_a_bad_limit_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    with pytest.raises(ValueError, match="sweep row 1"):
        SweepSpec(flat, 3, {("server_max_in_service", flat.server_ids[0]): [2, bad, 3]})
    with pytest.raises(ValueError, match="admission"):
        set_admission(flat, {flat.server_ids[0]: bad})


def test_python_refuses_an_unknown_server():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    with pytest.raises(KeyError, match="nope"):
        SweepSpec(flat, 2, {("server_max_in_service", "nope"): [1, 2]})
    with pytest.raises(KeyError, match="nope"):
        set_admission(flat, {"nope": 1})


@pytest.mark.parametrize("bad", [-1.0, 0.5, np.nan, np.inf, 2.0 ** 31])
def test_c_refuses_a_bad_limit_naming_the_row(bad):
    field = K.ADMISSION_FIELDS["server_max_in_service"]
    assert twin_admission.sweep_fits([(field, 0)], [[0.0], [7.0]]) is None
    why = twin_admission.sweep_fits([(field, 0)], [[1.0], [bad]])
    assert why is not None and "row 1" in why


def test_c_refuses_a_negative_scenario_limit():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin_admission.validate(flat) is None
    flat.pod.servers[1].max_in_service = -2
    assert "max_in_service" in twin_admission.validate(flat)


# ---- front end --------------------------------------------------------------------------------------------------------------
def test_payload_for_refuses_a_capped_row_and_payload_and_admission_gives_it():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    s0, s1 = flat.server_ids
    spec = SweepSpec(flat, 2, {("server_max_in_service", s0): [0, 4], ("users_mean",): [10.0, 20.0]})
    assert spec.payload_for(payload, 0)["rqs_input"]["avg_active_users"]["mean"] == 10.0
    with pytest.raises(ValueError, match="payload_and_admission"):
        spec.payload_for(payload, 1)
    p, adm = spec.payload_and_admission(payload, 1)
    assert adm == {s0: 4} and p["rqs_input"]["avg_active_users"]["mean"] == 20.0
    assert p["topology_graph"] == payload["topology_graph"]


def test_sweep_runner_front_end(monkeypatch):
    from asyncflow_b200 import runner as R
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    s0 = flatten(payload).server_ids[0]
    sr = R.SweepRunner(payload, 3, {("server_max_in_service", s0): [0, 2, 5]}, streams=[4, 4, 6])
    p, adm = sr.payload_and_admission(2)
    assert adm == {s0: 5}
    run = sr.replica_runner(2)
    assert run.admission == {s0: 5} and run.replica == 6 and run.simulation_input == p
    n, ns = 3, sr.flat.n_servers
    res = SweepResults(sr.flat, np.zeros(n, K.STATS_DTYPE), np.zeros((n, sr.flat.n_edges), np.uint32),
                       np.zeros((n, sr.flat.n_edges), np.uint32), np.zeros((n, sr.flat.n_series), np.uint64),
                       np.zeros((n, sr.flat.n_series), np.uint32))
    res.server_rejected = np.arange(n * ns, dtype=np.uint32).reshape(n, ns)
    res.rows = np.arange(n)
    pd = pytest.importorskip("pandas")
    df = sr.frame(res)
    assert isinstance(df, pd.DataFrame)
    assert df[f"server_max_in_service:{s0}"].tolist() == [0, 2, 5]
    assert df["rejected"].tolist() == res.server_rejected.sum(axis=1).tolist()
    t = res.take([2, 0])
    np.testing.assert_array_equal(t.server_rejected, res.server_rejected[[2, 0]])
    c = SweepResults.concatenate([res.take([0]), res.take([1, 2])])
    np.testing.assert_array_equal(c.server_rejected, res.server_rejected)


def test_the_example_and_the_tool_dry_run():
    import subprocess
    import sys
    for script in ("examples/sweep_admission.py", "tools/bench_admission.py"):
        r = subprocess.run([sys.executable, str(ROOT / script), "--dry-run"], cwd=ROOT, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr
