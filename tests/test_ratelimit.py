"""Rate limits (DESIGN.md §3.14) on the CPU: the oracle's specification (tests/des_ratelimit.py), the GCRA rule the
engines share, both state machines of the twin bit for bit against the oracle, the equivalences that make a limit free
when it cannot fire, the accounting of every request, each refusal in Python and in C, and the front end."""

from __future__ import annotations

import math
import zlib
from pathlib import Path

import des_deadline
import des_ratelimit
import fuzz
import lb_rows
import numpy as np
import pytest
import twin_ratelimit
from helpers import SCEN, SEED, assert_matches_oracle, load_scenario

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten, set_rate_limits
from asyncflow_b200.results import SweepResults

ROOT = Path(__file__).resolve().parent.parent
OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "rejected", "expired", "late", "throttled")
CASES = [("c1_my_service.yml", 20), ("c3_lb_two_servers.yml", 30), ("c4_lb8_events.yml", 20), ("mixed_lc.yml", None),
         ("chain_two_servers.yml", None), ("c5_multihop32.yml", 4), ("tie_cpu_io.yml", None)] + \
        [f"fuzz:{s}" for s in (302, 322, 329)]
BUILDS = ["lane", "warp"]      # (a launch with a rate limit runs the full lane build: aflh::lean_launch)


def _payload(case):
    if isinstance(case, str) and case.startswith("fuzz:"):
        return fuzz.scenario(int(case[5:]))
    return load_scenario(*case)


def _run(flat, build, **kw):
    if build == "lane":
        return twin_ratelimit.run_lane(flat, event_capacity=4096, request_capacity=200000, **kw)
    return twin_ratelimit.run_warp(flat, **kw)


def _oracle(payload, replica, ov, **kw):
    return des_ratelimit.simulate(payload, seed=SEED, replica=replica, admission=ov["admission"],
                                  deadline=ov["deadline"], client_timeout=ov["client_timeout"],
                                  rate_limit=ov.get("rate_limit"), lb_rate_limit=ov.get("lb_rate_limit"), **kw)


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
    assert [int(x) for x in r["throttled"][i]] == [o["server_throttled"][s] for s in flat.server_ids] + [o["lb_throttled"]]


def _arrival_rate(payload) -> float:
    """Requests per second the scenario generates (the oracle's count over its horizon)."""
    o = des_deadline.simulate(payload, seed=SEED, replica=0)
    return max(1.0, o["generated"] / float(payload["sim_settings"]["total_simulation_time"]))


# ---- the rule ------------------------------------------------------------------------------------------------------------
def _py_rule(tat: float, now: float, r: float, b: int) -> tuple[bool, float]:
    tau = 1.0 / r
    lim = (b - 1) * tau
    if tat - now > lim:
        return False, tat
    return True, max(tat, now) + tau


@pytest.mark.parametrize(("r", "b"), [(1.0, 1), (3.0, 1), (7.0, 4), (1000.0, 50), (0.1, 2), (450.0, 13), (4.0, 3)])
@pytest.mark.parametrize("now", [0.0, 12.375, 0.1])
def test_the_check_function_is_the_python_rule(r, b, now):
    tau = 1.0 / r
    lim = (b - 1) * tau
    # tat - now == L exactly: the largest tat whose f64 difference is L passes; the next one throttles
    tat = now + lim
    while tat - now > lim:
        tat = math.nextafter(tat, -math.inf)
    while math.nextafter(tat, math.inf) - now <= lim:
        tat = math.nextafter(tat, math.inf)
    above = math.nextafter(tat, math.inf)
    assert tat - now <= lim < above - now
    for t in (tat, above, now - 3.0, now, 0.0, now + 0.5 * lim, now + 2 * lim + 1.0):
        assert twin_ratelimit.rl_pass(t, now, r, b) == _py_rule(t, now, r, b), (t, now, r, b)
    if tat - now == lim:
        assert twin_ratelimit.rl_pass(tat, now, r, b) == (True, max(tat, now) + tau)
    assert twin_ratelimit.rl_pass(above, now, r, b) == (False, above)
    assert twin_ratelimit.rl_pass(now - 3.0, now, r, b) == (True, now + tau)   # tat < now: passes, resets to now + tau


def test_the_bucket_starts_full():
    for b in (1, 2, 5):
        tat, passed = 0.0, 0
        for _ in range(b + 3):
            ok, tat = twin_ratelimit.rl_pass(tat, 0.0, 10.0, b)
            passed += ok
        assert passed == b


# ---- the oracle ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(p.name for p in SCEN.glob("*.yml")))
def test_no_limit_is_the_deadline_oracle_unchanged(name):
    payload = load_scenario(name, 10)
    ref = des_deadline.simulate(payload, seed=SEED, replica=1)
    servers = [s["id"] for s in payload["topology_graph"]["nodes"]["servers"]]
    lb = payload["topology_graph"]["nodes"].get("load_balancer")
    for rl, lbl in ((None, None), ({}, None), (dict.fromkeys(servers, (0.0, 5)), (0.0, 3) if lb else None)):
        o = des_ratelimit.simulate(payload, seed=SEED, replica=1, rate_limit=rl, lb_rate_limit=lbl)
        assert o.pop("server_throttled") == dict.fromkeys(servers, 0)
        assert o.pop("lb_throttled") == 0
        assert o == ref


@pytest.mark.parametrize("b", [1, 3, 10])
def test_a_rate_that_never_refills_passes_exactly_the_first_burst(b):
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    s0 = flat.server_ids[0]
    for site, kw in ((s0, {"rate_limit": {s0: (1e-6, b)}}), (flat.lb_id, {"lb_rate_limit": (1e-6, b)})):
        checks: list = []
        o = des_ratelimit.simulate(payload, seed=SEED, replica=0, checks=checks, **kw)
        mine = [c for c in checks if c[0] == site]
        assert len(mine) == len(checks) > b
        assert [c[6] for c in mine] == [True] * b + [False] * (len(mine) - b)
        assert o["lb_throttled"] + o["server_throttled"][s0] == len(mine) - b


def test_burst_one_spaces_admissions_by_tau():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    r = 0.6 * _arrival_rate(payload)
    checks: list = []
    o = des_ratelimit.simulate(payload, seed=SEED, replica=2, lb_rate_limit=(r, 1), checks=checks)
    tau = 1.0 / r
    admitted = [c[2] for c in checks if c[6]]
    assert o["lb_throttled"] > 0 and len(admitted) > 10
    for a, b in zip(admitted, admitted[1:]):
        assert b >= a + tau


@pytest.mark.parametrize(("frac", "b"), [(0.3, 1), (0.5, 8), (0.8, 40)])
def test_no_window_admits_more_than_the_burst_and_the_rate(frac, b):
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    r = frac * _arrival_rate(payload)
    checks: list = []
    des_ratelimit.simulate(payload, seed=SEED, replica=4, lb_rate_limit=(r, b), checks=checks)
    t = np.array([c[2] for c in checks if c[6]])
    assert t.size > 50
    for w in (0.01, 0.1, 1.0, 5.0):
        hi = np.searchsorted(t, t + w, side="right")    # admissions in [t_i, t_i + w]
        assert (hi - np.arange(t.size)).max() <= b + math.floor(r * w) + 1


def test_oracle_refuses_unknown_servers_and_bad_values():
    p = load_scenario("c1_my_service.yml", 5)
    sid = p["topology_graph"]["nodes"]["servers"][0]["id"]
    with pytest.raises(KeyError, match="nope"):
        des_ratelimit.simulate(p, seed=SEED, replica=0, rate_limit={"nope": (1.0, 1)})
    for bad in ((-1.0, 1), (float("nan"), 1), (float("inf"), 1), (True, 1), (1.0, -1), (1.0, 1.5), (1.0, True), 3.0):
        with pytest.raises(ValueError):
            des_ratelimit.simulate(p, seed=SEED, replica=0, rate_limit={sid: bad})
    with pytest.raises(ValueError, match="load balancer"):
        des_ratelimit.simulate(p, seed=SEED, replica=0, lb_rate_limit=(5.0, 1))


# ---- both state machines against the oracle -------------------------------------------------------------------------------
def _rate_columns(flat, payload, n: int, rng, caps: bool, deadlines: bool) -> dict:
    lam = _arrival_rate(payload)
    rates = np.array([0.0, 0.2, 0.5, 0.9, 3.0]) * lam / max(1, flat.n_servers) * 1.5
    cols = {("server_rate", s): rng.choice(rates, n) for s in flat.server_ids}
    cols.update({("server_burst", s): rng.integers(1, 12, n) for s in flat.server_ids})
    if flat.lb_id is not None:
        cols[("lb_rate",)] = rng.choice(np.array([0.0, 0.3, 0.7, 2.0]) * lam, n)
        cols[("lb_burst",)] = rng.integers(1, 30, n)
    if caps:
        cols.update({("server_max_in_service", s): rng.integers(0, 6, n).astype(float) for s in flat.server_ids})
    if deadlines:
        o = des_deadline.simulate(payload, seed=SEED, replica=0)
        lat = np.array([b - a for a, b in o["clocks"]] or [1.0])
        cols[("server_deadline", flat.server_ids[0])] = rng.choice([0.0, *np.quantile(lat, [0.3, 0.8])], n)
        cols[("client_timeout",)] = rng.choice([0.0, float(np.quantile(lat, 0.6))], n)
    return cols


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("case", CASES, ids=str)
def test_rows_equal_the_oracle(case, build):
    payload = _payload(case)
    flat = flatten(payload)
    n = 6
    h = zlib.crc32(str(case).encode())
    rng = np.random.default_rng(h)
    cols = _rate_columns(flat, payload, n, rng, caps=h % 2 == 0, deadlines=h % 3 == 0)
    cols[("users_mean",)] = rng.choice([1.0, 2.0, 4.0], n) * float(flat.pod.users_mean)
    spec = SweepSpec(flat, n, cols)
    streams = [5, 5, 9, 5, 2, 9]                  # rows sharing a stream see the same traffic whatever their limits
    r = _run(flat, build, seed=SEED, n=n, sweep=spec, streams=streams, trace=n, clock_cap=200000)
    throttled = 0
    for i in range(n):
        p, ov = spec.payload_and_overload(payload, i)
        o = _oracle(p, streams[i], ov)
        _check(o, flat, r, i, traced=True)
        throttled += sum(o["server_throttled"].values()) + o["lb_throttled"]
    assert throttled > 0, "no row throttled a request: the case does not exercise the limit"


@pytest.mark.parametrize("build", BUILDS)
def test_scenario_limits_equal_the_oracle(build):
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    lam = _arrival_rate(payload)
    rl = {s: (0.4 * lam, 3 + i) for i, s in enumerate(flat.server_ids)}
    lb = (0.9 * lam, 20)
    set_rate_limits(flat, rl, lb=lb)
    assert twin_ratelimit.ratelimit_launch(flat) and not twin_ratelimit.lean_launch(flat)
    r = _run(flat, build, seed=SEED, n=3, trace=3, clock_cap=200000)
    for i in range(3):
        o = des_ratelimit.simulate(payload, seed=SEED, replica=i, rate_limit=rl, lb_rate_limit=lb)
        _check(o, flat, r, i, traced=True)
        assert o["lb_throttled"] > 0 and sum(o["server_throttled"].values()) > 0


def test_rows_with_bands_occupancy_lb_rows_and_event_rows():
    payload = load_scenario("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    n = 4
    rng = np.random.default_rng(4)
    cols = _rate_columns(flat, payload, n, rng, caps=True, deadlines=True)
    cols[("lb_algorithm",)] = ["round_robin", "least_connection", "round_robin", "least_connection"]
    cols[("lb_covered", lb_rows.uncoverable(payload)[0][0])] = [1, 0, 1, 1]
    cols[("event_start", "ev-srv3-down")] = [2.0, 6.0, 2.0, 6.0]
    cols[("event_end", "ev-srv3-down")] = [9.0, 14.0, 14.0, 9.0]
    cols[("event_start", "ev-spike")] = np.full(n, 4.0)
    cols[("event_end", "ev-spike")] = np.full(n, 11.0)
    cols[("lb_rate",)] = np.array([0.4, 0.6, 0.8, 0.0]) * _arrival_rate(payload)
    spec = SweepSpec(flat, n, cols)
    kw = dict(seed=SEED, n=n, sweep=spec, streams=[1, 1, 1, 1], groups=np.array([0, 1, 0, 1]), n_groups=2,
              sampled=True, window=5, series=[0, 3 * flat.n_servers], f=20)
    for build in BUILDS:
        r = _run(flat, build, **kw)
        for i in range(n):
            p, ov = spec.payload_and_overload(payload, i)
            o = _oracle(p, 1, ov)
            lb_rows.check_replica(o, flat, p, stats=r["stats"][i], sent=r["sent"][i], dropped=r["dropped"][i],
                                  thr=r["thr"][i])
            assert [int(x) for x in r["rejected"][i]] == [o["server_rejected"][s] for s in flat.server_ids]
            assert [int(x) for x in r["expired"][i]] == [o["server_expired"][s] for s in flat.server_ids]
            assert int(r["late"][i]) == o["late"]
            assert [int(x) for x in r["throttled"][i]] == ([o["server_throttled"][s] for s in flat.server_ids]
                                                           + [o["lb_throttled"]])
        assert r["occ"].any() and r["band_rows"].any() and r["lat_rows"].any() and r["dist_rows"].any()
        assert r["throttled"][:, flat.n_servers].any()


def test_pool_splits_give_the_same_results():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 6
    spec = SweepSpec(flat, n, _rate_columns(flat, payload, n, np.random.default_rng(9), caps=True, deadlines=True))
    ref = _run(flat, "lane", seed=SEED, n=n, sweep=spec)
    assert ref["throttled"].any()
    for lane_bytes, split in ((1000, "random"), (4000, "rows"), (1816, "scenario")):
        r = twin_ratelimit.run_lane(flat, seed=SEED, n=n, sweep=spec, event_capacity=4096, request_capacity=200000,
                                    lane_bytes=lane_bytes, split=split, split_seed=3)
        for k in OUT:
            np.testing.assert_array_equal(ref[k], r[k], err_msg=f"{k} {lane_bytes} {split}")


def test_a_warp_rerun_keeps_writing_the_counts():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 4
    spec = SweepSpec(flat, n, _rate_columns(flat, payload, n, np.random.default_rng(2), caps=False, deadlines=False))
    ref = _run(flat, "warp", seed=SEED, n=n, sweep=spec)
    out = _run(flat, "lane", seed=SEED, n=n, sweep=spec)
    np.testing.assert_array_equal(out["throttled"], ref["throttled"])
    out["throttled"][[1, 3]] = 0
    twin_ratelimit.run_warp(flat, seed=SEED, n=n, sweep=spec, redo=[1, 3], into=out)
    np.testing.assert_array_equal(out["throttled"], ref["throttled"])


# ---- equivalences -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build", BUILDS)
def test_a_zero_rate_column_or_a_rate_that_never_binds_is_no_column(build):
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 4
    users = {("users_mean",): np.array([1.0, 3.0, 6.0, 10.0]) * float(flat.pod.users_mean)}
    plain = SweepSpec(flat, n, users)
    kw = dict(seed=SEED, n=n, groups=np.array([0, 1, 0, 1]), n_groups=2, sampled=True, window=5, series=[1], f=24)
    a = _run(flat, build, sweep=plain, **kw)
    assert not twin_ratelimit.ratelimit_launch(flat, plain)
    big = int(a["stats"]["generated"].max()) + 1
    for rate, burst in ((0.0, 1), (0.0, 7), (1e12, big)):
        cols = {**users, **{("server_rate", s): np.full(n, rate) for s in flat.server_ids},
                **{("server_burst", s): np.full(n, burst) for s in flat.server_ids},
                ("lb_rate",): np.full(n, rate), ("lb_burst",): np.full(n, burst)}
        spec = SweepSpec(flat, n, cols)
        assert twin_ratelimit.ratelimit_launch(flat, spec) and not twin_ratelimit.lean_launch(flat, spec)
        b = _run(flat, build, sweep=spec, **kw)
        for k in (*OUT, "band_rows", "lat_rows", "dist_rows", "occ"):
            if k == "throttled":
                assert not b[k].any()
            else:
                np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} {rate} {burst}")


def test_rows_of_one_stream_generate_the_same_whatever_their_limits():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    n = 4
    lam = _arrival_rate(payload)
    spec = SweepSpec(flat, n, {("users_mean",): np.full(n, 4.0 * float(flat.pod.users_mean)),
                               ("lb_rate",): [0.0, 0.2 * lam, 0.5 * lam, 2.0 * lam], ("lb_burst",): [1, 1, 5, 5]})
    r = twin_ratelimit.run(flat, seed=SEED, n=n, sweep=spec, streams=[8] * n)
    assert len(set(r["stats"]["generated"].tolist())) == 1
    assert len(set(r["sent"][:, flat.pod.gen_edge].tolist())) == 1
    lbt = r["throttled"][:, flat.n_servers]
    assert lbt[0] == 0 and lbt[1] >= lbt[2] > 0


@pytest.mark.parametrize("build", BUILDS)
def test_every_request_is_accounted_for(build):
    payload = load_scenario("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    n = 8
    rng = np.random.default_rng(11)
    spec = SweepSpec(flat, n, {**_rate_columns(flat, payload, n, rng, caps=True, deadlines=True),
                               ("users_mean",): rng.choice([1.0, 3.0], n) * float(flat.pod.users_mean)})
    r = _run(flat, build, seed=SEED, n=n, sweep=spec)
    st = r["stats"]
    gone = (st["completed"].astype(np.int64) + r["dropped"].sum(axis=1) + r["rejected"].sum(axis=1)
            + r["expired"].sum(axis=1) + r["throttled"].sum(axis=1))
    assert (gone <= st["generated"]).all()
    assert r["throttled"].sum() > 0


def test_a_launch_with_a_rate_limit_runs_the_full_lane_build():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    s0 = flat.server_ids[0]
    assert twin_ratelimit.lean_launch(flat) and not twin_ratelimit.ratelimit_launch(flat)
    set_rate_limits(flat, {s0: (0.0, 4)}, lb=(0.0, 2))
    assert twin_ratelimit.lean_launch(flat) and not twin_ratelimit.ratelimit_launch(flat)
    set_rate_limits(flat, {s0: (5.0, 1)})
    assert not twin_ratelimit.lean_launch(flat) and twin_ratelimit.ratelimit_launch(flat)
    set_rate_limits(flat, {s0: (0.0, 1)}, lb=(5.0, 1))
    assert not twin_ratelimit.lean_launch(flat) and twin_ratelimit.ratelimit_launch(flat)
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for sel in (("server_rate", s0), ("lb_rate",)):
        spec = SweepSpec(flat, 2, {sel: [0.0, 0.0]})
        assert not twin_ratelimit.lean_launch(flat, spec) and twin_ratelimit.ratelimit_launch(flat, spec)
    for sel in (("server_burst", s0), ("lb_burst",)):
        spec = SweepSpec(flat, 2, {sel: [1, 3]})
        assert not twin_ratelimit.lean_launch(flat, spec) and twin_ratelimit.ratelimit_launch(flat, spec)


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [-1, -0.5, np.nan, np.inf, True, "fast"])
def test_python_refuses_a_bad_rate_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for sel in (("server_rate", flat.server_ids[0]), ("lb_rate",)):
        with pytest.raises(ValueError, match="sweep row 1"):
            SweepSpec(flat, 3, {sel: [2, bad, 3]})
    with pytest.raises(ValueError, match="rate"):
        set_rate_limits(flat, {flat.server_ids[0]: (bad, 1)})


@pytest.mark.parametrize("bad", [0, -1, 1.5, 2.0 ** 31, np.nan, True, "many"])
def test_python_refuses_a_bad_burst_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for sel in (("server_burst", flat.server_ids[0]), ("lb_burst",)):
        with pytest.raises(ValueError, match="sweep row 1"):
            SweepSpec(flat, 3, {sel: [2, bad, 3]})


def test_python_refuses_an_unknown_server_and_lb_columns_without_an_lb():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for name in ("server_rate", "server_burst"):
        with pytest.raises(KeyError, match="nope"):
            SweepSpec(flat, 2, {(name, "nope"): [1, 2]})
    with pytest.raises(KeyError, match="nope"):
        set_rate_limits(flat, {"nope": (1.0, 1)})
    plain = flatten(load_scenario("c1_my_service.yml", 5))
    for name in ("lb_rate", "lb_burst"):
        with pytest.raises(ValueError, match="load balancer"):
            SweepSpec(plain, 2, {(name,): [1, 2]})
    with pytest.raises(ValueError, match="load balancer"):
        set_rate_limits(plain, None, lb=(1.0, 1))


@pytest.mark.parametrize("bad", [-1.0, -1e-300, np.nan, np.inf, -np.inf])
def test_c_refuses_a_bad_rate_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for field in (K.RATE_FIELDS["server_rate"], K.RATE_FIELDS["lb_rate"]):
        assert twin_ratelimit.sweep_fits(flat, [(field, 0)], [[0.0], [7.5]]) is None
        why = twin_ratelimit.sweep_fits(flat, [(field, 0)], [[1.0], [bad]])
        assert why is not None and "row 1" in why


@pytest.mark.parametrize("bad", [0.0, -1.0, 1.5, 2.0 ** 31, np.nan, np.inf])
def test_c_refuses_a_bad_burst_naming_the_row(bad):
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    for field in (K.RATE_FIELDS["server_burst"], K.RATE_FIELDS["lb_burst"]):
        assert twin_ratelimit.sweep_fits(flat, [(field, 0)], [[1.0], [2.0 ** 31 - 1]]) is None
        why = twin_ratelimit.sweep_fits(flat, [(field, 0)], [[1.0], [bad]])
        assert why is not None and "row 1" in why


def test_c_refuses_lb_columns_without_an_lb_and_bad_scenario_values():
    plain = flatten(load_scenario("c1_my_service.yml", 5))
    for field in (K.RATE_FIELDS["lb_rate"], K.RATE_FIELDS["lb_burst"]):
        assert "load balancer" in twin_ratelimit.sweep_fits(plain, [(field, 0)], [[1.0]])
    assert twin_ratelimit.validate(plain) is None
    plain.pod.lb_rate_limit = 3.0
    assert "load balancer" in twin_ratelimit.validate(plain)
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin_ratelimit.validate(flat) is None
    for bad in (-1.0, np.nan, np.inf):
        flat.pod.servers[1].rate_limit = bad
        assert "rate_limit" in twin_ratelimit.validate(flat)
        flat.pod.servers[1].rate_limit = 0.0
        flat.pod.lb_rate_limit = bad
        assert "lb_rate_limit" in twin_ratelimit.validate(flat)
        flat.pod.lb_rate_limit = 0.0
    flat.pod.servers[0].burst = -1
    assert "burst" in twin_ratelimit.validate(flat)
    flat.pod.servers[0].burst = 0
    flat.pod.lb_burst = -2
    assert "lb_burst" in twin_ratelimit.validate(flat)
    flat.pod.lb_burst = 0
    assert twin_ratelimit.validate(flat) is None


# ---- front end --------------------------------------------------------------------------------------------------------------
def test_payload_for_refuses_a_rate_row_and_payload_and_overload_gives_it():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    s0, s1 = flat.server_ids
    spec = SweepSpec(flat, 3, {("server_rate", s0): [0.0, 40.0, 0.0], ("server_burst", s0): [1, 2, 9],
                               ("lb_rate",): [0.0, 0.0, 90.0], ("users_mean",): [10.0, 20.0, 30.0]})
    assert spec.payload_for(payload, 0)["rqs_input"]["avg_active_users"]["mean"] == 10.0
    for i in (1, 2):
        with pytest.raises(ValueError, match="payload_and_overload"):
            spec.payload_for(payload, i)
        with pytest.raises(ValueError, match="payload_and_overload"):
            spec.payload_and_admission(payload, i)
    p, ov = spec.payload_and_overload(payload, 2)
    assert ov["rate_limit"] == {s0: (0.0, 9)} and ov["lb_rate_limit"] == (90.0, 1)
    assert ov["admission"] == {} and ov["deadline"] == {} and ov["client_timeout"] is None
    assert p["rqs_input"]["avg_active_users"]["mean"] == 30.0 and p["topology_graph"] == payload["topology_graph"]
    set_rate_limits(flat, {s1: (12.0, 4)}, lb=(50.0, 0))
    spec = SweepSpec(flat, 2, {("server_burst", s1): [2, 6]})
    assert spec.rate_limits_for(1) == ({s1: (12.0, 6)}, (50.0, 1))


def test_sweep_runner_front_end():
    from asyncflow_b200 import runner as R
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    s0 = flatten(payload).server_ids[0]
    sr = R.SweepRunner(payload, 3, {("server_rate", s0): [0.0, 20.0, 50.0], ("server_burst", s0): [1, 3, 5],
                                    ("lb_rate",): [100.0, 100.0, 0.0], ("lb_burst",): [10, 10, 1]},
                       streams=[4, 4, 6])
    p, ov = sr.payload_and_overload(2)
    assert ov["rate_limit"] == {s0: (50.0, 5)} and ov["lb_rate_limit"] == (0.0, 1)
    run = sr.replica_runner(2)
    assert run.rate_limit == {s0: (50.0, 5)} and run.lb_rate_limit == (0.0, 1) and run.replica == 6
    assert run.simulation_input == p
    n, ns = 3, sr.flat.n_servers
    res = SweepResults(sr.flat, np.zeros(n, K.STATS_DTYPE), np.zeros((n, sr.flat.n_edges), np.uint32),
                       np.zeros((n, sr.flat.n_edges), np.uint32), np.zeros((n, sr.flat.n_series), np.uint64),
                       np.zeros((n, sr.flat.n_series), np.uint32))
    assert res.server_throttled.shape == (n, ns) and res.lb_throttled.shape == (n,)
    res.server_throttled = np.arange(n * ns, dtype=np.uint32).reshape(n, ns)
    res.lb_throttled = np.array([5, 6, 7], dtype=np.uint32)
    res.rows = np.arange(n)
    t = res.take([2, 0])
    np.testing.assert_array_equal(t.server_throttled, res.server_throttled[[2, 0]])
    np.testing.assert_array_equal(t.lb_throttled, res.lb_throttled[[2, 0]])
    c = SweepResults.concatenate([res.take([0]), res.take([1, 2])])
    np.testing.assert_array_equal(c.server_throttled, res.server_throttled)
    np.testing.assert_array_equal(c.lb_throttled, res.lb_throttled)
    pytest.importorskip("pandas")
    df = sr.frame(res)
    assert df[f"server_rate:{s0}"].tolist() == [0.0, 20.0, 50.0] and df["lb_burst"].tolist() == [10, 10, 1]
    assert df["throttled"].tolist() == (res.server_throttled.sum(axis=1) + res.lb_throttled).tolist()


def test_the_example_and_the_tool_dry_run():
    import subprocess
    import sys
    for script in ("examples/sweep_rate_limit.py", "tools/bench_ratelimit.py"):
        r = subprocess.run([sys.executable, str(ROOT / script), "--dry-run"], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr
