"""Load-balancer rows (``("lb_covered", server)`` / ``("lb_algorithm",)`` sweep columns) on the CPU twin of both state
machines: every row equals the oracle run on ``SweepSpec.payload_for(row)`` -- the scenario without the LB's edges to
the uncovered servers -- an uncovered edge carries nothing, a row equal to the scenario changes no output byte, rows of
one stream see the same traffic whatever their fleet and policy, and every rule refuses a bad row by name."""

from __future__ import annotations

import copy
import ctypes as C
import zlib

import des_port
import fuzz
import numpy as np
import pytest
import twin
import twin_lb
import twin_streams
from helpers import SEED, load_scenario
from lb_rows import check_replica, lb_columns, lb_servers

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten

OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max")
FUZZ_SEEDS = [302, 322, 329]
CASES = [("c3_lb_two_servers.yml", 30), ("mixed_lc.yml", 20), ("c4_lb8_events.yml", 20), ("ev_spikes_outages.yml", None),
         ("c5_multihop32.yml", 4)] + [f"fuzz:{s}" for s in FUZZ_SEEDS]


def _payload(case):
    if isinstance(case, str) and case.startswith("fuzz:"):
        return fuzz.scenario(int(case[5:]))
    return load_scenario(*case)


def _columns(case, payload, flat, n: int, rng) -> dict:
    """Random fleets and algorithms, mixed with other swept columns; c4's outage and spike moved inside the horizon."""
    cols = lb_columns(payload, n, rng)
    cols[("users_mean",)] = rng.choice([0.5, 1.0, 1.5], n) * float(flat.pod.users_mean)
    if case[0] == "c4_lb8_events.yml":
        cols[("event_start", "ev-srv3-down")] = rng.choice([2.0, 6.0], n)
        cols[("event_end", "ev-srv3-down")] = rng.choice([9.0, 14.0], n)
        cols[("event_start", "ev-spike")] = np.full(n, 4.0)
        cols[("event_end", "ev-spike")] = np.full(n, 11.0)
    return cols


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("case", CASES, ids=str)
def test_rows_equal_the_oracle(case, engine):
    payload = _payload(case)
    flat = flatten(payload)
    n = 5
    rng = np.random.default_rng(zlib.crc32(str(case).encode()))
    spec = SweepSpec(flat, n, _columns(case, payload, flat, n, rng))
    streams = [7, 7, 3, 7, 11]                           # common random numbers across fleets and policies
    r = twin_streams.run(flat, seed=SEED, n=n, sweep=spec, streams=streams, trace=n, clock_cap=200000,
                         request_capacity=200000, engine=engine)
    assert twin_lb.cover_fits(flat, spec, 0, n, timeline=spec if spec.timelines is not None else None) is None
    for i in range(n):
        p = spec.payload_for(payload, i)
        st = r["stats"][i]
        k, nt = int(st["completed"]), int(st["n_ticks"])
        check_replica(des_port.simulate(p, seed=SEED, replica=streams[i]), flat, p, stats=st, sent=r["sent"][i],
                      dropped=r["dropped"][i], thr=r["thr"][i], clocks=r["trace_clocks"][i, :k],
                      series=r["trace_series"][i][:, :nt])


def test_the_reduced_payload_drops_the_edge_and_keeps_the_server():
    payload = load_scenario("ev_spikes_outages.yml")
    flat = flatten(payload)
    spec = SweepSpec(flat, 2, {("lb_covered", "srv-1"): [True, False], ("lb_algorithm",): ["round_robin", K.LB_LEAST_CONNECTIONS]})
    p0, p1 = spec.payload_for(payload, 0), spec.payload_for(payload, 1)
    assert p0["topology_graph"] == payload["topology_graph"]
    lb = p1["topology_graph"]["nodes"]["load_balancer"]
    assert lb["server_covered"] == ["srv-2", "srv-3"] and lb["algorithms"] == "least_connection"
    assert "lb-srv1" not in {e["id"] for e in p1["topology_graph"]["edges"]}
    assert {s["id"] for s in p1["topology_graph"]["nodes"]["servers"]} == set(flat.server_ids)
    assert p1["events"] == payload["events"]            # srv-1's outages stay: no-ops there
    # the row's timeline: srv-1's marks with lb_edge = -1, fire times as in the scenario
    red = flatten(p1)
    ou = spec.timelines.outages[1]
    mine = np.frombuffer(C.string_at(red.pod.outage_marks, ou.nbytes), dtype=ou.dtype)   # edges by id: indices shift
    assert np.array_equal(mine[["fire_time", "down"]], ou[["fire_time", "down"]])
    assert [red.edge_ids[e] if e >= 0 else None for e in mine["lb_edge"]] == [flat.edge_ids[e] if e >= 0 else None
                                                                              for e in ou["lb_edge"]]
    assert (ou["lb_edge"] != flat.edge_ids.index("lb-srv1")).all()
    assert np.array_equal(ou["fire_time"], spec.timelines.outages[0]["fire_time"])


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("case", [("c3_lb_two_servers.yml", 30), ("mixed_lc.yml", 20), ("ev_spikes_outages.yml", None)], ids=str)
def test_rows_equal_to_the_scenario_change_nothing(case, engine):
    payload = load_scenario(*case)
    flat = flatten(payload)
    n = 3
    users = {("users_mean",): [10.0, 20.0, 30.0]}
    cols = dict(users)
    cols.update({("lb_covered", s): np.ones(n) for s in lb_servers(payload)})
    cols[("lb_algorithm",)] = [payload["topology_graph"]["nodes"]["load_balancer"]["algorithms"]] * n
    same = SweepSpec(flat, n, cols)
    assert same.timelines is None
    a = twin.run(flat, seed=SEED, n=n, sweep=same, engine=engine)
    b = twin.run(flat, seed=SEED, n=n, sweep=SweepSpec(flat, n, users), engine=engine)
    for k in OUT:
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_one_stream_sees_the_same_traffic_in_every_fleet_and_policy(engine):
    payload = load_scenario("mixed_lc.yml", 20)
    flat = flatten(payload)
    n = 4
    cols = {("lb_covered", "srv-2"): [1, 0, 1, 0], ("lb_covered", "srv-3"): [1, 1, 0, 0],
            ("lb_algorithm",): ["round_robin", "least_connection", "least_connection", "round_robin"]}
    spec = SweepSpec(flat, n, cols)
    r = twin_streams.run(flat, seed=SEED, n=n, sweep=spec, streams=[5] * n, trace=n, clock_cap=200000, engine=engine)
    gen = r["stats"]["generated"]
    assert (gen == gen[0]).all() and gen[0] > 100
    starts = [set(r["trace_clocks"][i, :int(r["stats"][i]["completed"]), 0].tolist()) for i in range(n)]
    assert len(set.union(*starts)) <= int(gen[0])           # every completion started at one of the same arrivals
    assert len(set.intersection(*starts)) >= 0.8 * min(map(len, starts))
    assert len({r["sent"][i].tobytes() for i in range(n)}) == n     # and the fleets route them differently


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_sweepspec_refuses_bad_rows_by_name():
    c3 = load_scenario("c3_lb_two_servers.yml")
    f3 = flatten(c3)
    with pytest.raises(ValueError, match=r"sweep row 1: .*covers no server"):
        SweepSpec(f3, 2, {("lb_covered", "srv-1"): [1, 0], ("lb_covered", "srv-2"): [0, 0]})
    with pytest.raises(ValueError, match=r"sweep row 1: \('lb_covered', 'srv-1'\) = 2"):
        SweepSpec(f3, 2, {("lb_covered", "srv-1"): [1, 2]})
    with pytest.raises(ValueError, match=r"sweep row 0: \('lb_algorithm',\) = 'random'"):
        SweepSpec(f3, 2, {("lb_algorithm",): ["random", "round_robin"]})
    with pytest.raises(ValueError, match=r"sweep row 1: \('lb_algorithm',\) = 2"):
        SweepSpec(f3, 2, {("lb_algorithm",): [0, 2]})
    with pytest.raises(ValueError, match="no load balancer"):
        SweepSpec(flatten(load_scenario("c1_my_service.yml")), 2, {("lb_algorithm",): ["round_robin"] * 2})
    c5 = flatten(load_scenario("c5_multihop32.yml"))
    back = next(s for s in c5.server_ids if not s.startswith("fe-"))
    with pytest.raises(KeyError, match="does not cover"):
        SweepSpec(c5, 2, {("lb_covered", back): [1, 0]})
    spiked = copy.deepcopy(c3)
    spiked["events"] = [{"event_id": "sp", "target_id": "lb-srv1", "start": {"kind": "network_spike_start", "t_start": 1.0,
                         "spike_s": 0.01}, "end": {"kind": "network_spike_end", "t_end": 2.0}}]
    with pytest.raises(ValueError, match=r"sweep row 1: .*'sp' targets the load balancer's edge"):
        SweepSpec(flatten(spiked), 2, {("lb_covered", "srv-1"): [1, 0]})
    SweepSpec(flatten(spiked), 2, {("lb_covered", "srv-2"): [1, 0]})      # the other server may go
    ev = flatten(load_scenario("ev_spikes_outages.yml"))
    # srv-1 alone is covered in row 1, and goes down at t = 8 (no event time swept: the scenario's outages)
    with pytest.raises(ValueError, match=r"sweep row 1: .*every server behind the load balancer is down"):
        SweepSpec(ev, 2, {("lb_covered", "srv-2"): [1, 0], ("lb_covered", "srv-3"): [1, 0]})
    # ... and with a row's own outage times
    with pytest.raises(ValueError, match=r"sweep row 0: .*every server behind the load balancer is down"):
        SweepSpec(ev, 2, {("lb_covered", "srv-3"): [0, 1], ("event_start", "ev-f"): [10.0, 18.0],
                          ("event_end", "ev-f"): [12.0, 28.25]})


def _raw_sweep(cols: list[tuple[int, int]], values) -> tuple[K.AfSweep, tuple]:
    v = np.ascontiguousarray(values, dtype=np.float64)
    c = (K.AfSweepColumn * len(cols))(*[K.AfSweepColumn(f, i) for f, i in cols])
    sw = K.AfSweep()
    sw.n_columns, sw.n_rows = len(cols), v.shape[0]
    sw.columns = C.cast(c, C.POINTER(K.AfSweepColumn))
    sw.values = v.ctypes.data_as(C.POINTER(C.c_double))
    return sw, (c, v)


def _sweep_fits(flat, cols, values) -> str | None:
    sw, keep = _raw_sweep(cols, values)
    L = twin_lb.lib()
    ok = L.af_twin_lb_sweep_fits(C.byref(flat.pod), C.byref(sw))
    return None if ok else L.af_twin_lb_error().decode()


def test_the_engine_refuses_bad_columns_by_row():
    f3 = flatten(load_scenario("c3_lb_two_servers.yml"))
    cov, algo = K.LB_FIELDS["lb_covered"], K.LB_FIELDS["lb_algorithm"]
    assert _sweep_fits(f3, [(cov, 0), (algo, 0)], [[1, 0], [0, 1]]) is None
    assert "row 2 covers no edge" in _sweep_fits(f3, [(cov, 0), (cov, 1)], [[1, 0], [0, 1], [0, 0]])
    assert "row 0 column 0 (lb_covered): value 0.5" in _sweep_fits(f3, [(cov, 1)], [[0.5]])
    assert "row 1 column 1 (lb_algorithm): value 2" in _sweep_fits(f3, [(cov, 1), (algo, 0)], [[1, 0], [1, 2]])
    # the later of two columns over one position wins, as in the kernels
    assert "row 0 covers no edge" in _sweep_fits(f3, [(cov, 0), (cov, 1), (cov, 0)], [[1, 0, 0]])
    c1 = flatten(load_scenario("c1_my_service.yml"))
    assert "without one" in _sweep_fits(c1, [(algo, 0)], [[0]])


def test_af_run_refuses_rows_that_uncover_a_server_its_outage_marks_name():
    payload = load_scenario("ev_spikes_outages.yml")
    flat = flatten(payload)
    spec = SweepSpec(flat, 3, {("lb_covered", "srv-1"): [1, 0, 1]})
    assert spec.timelines is not None                  # srv-1 has outages: the rows carry timelines
    assert twin_lb.cover_fits(flat, spec, 0, 3, timeline=spec) is None
    why = twin_lb.cover_fits(flat, spec, 0, 3)         # the scenario's marks name srv-1's edge
    assert why is not None and "replica 1 uncovers load-balancer edge" in why and "scenario's timeline" in why
    assert twin_lb.cover_fits(flat, spec, 2, 3) is None          # replica 1 is not in the launch
    assert twin_lb.cover_fits(flat, spec, 5, 9, sweep_first=5) is not None   # rows addressed by replica id
    assert twin_lb.cover_fits(flat, spec, 0, 3, timeline=spec, timeline_first=1) is not None   # replica 1 reads row 0
    # a server without outages may be uncovered with the scenario's marks
    free = SweepSpec(flat, 2, {("lb_covered", "srv-3"): [1, 0]})
    assert free.timelines is None and twin_lb.cover_fits(flat, free, 0, 2) is None


def test_frame_shows_the_algorithm_names():
    pytest.importorskip("pandas")
    from asyncflow_b200 import SweepRunner
    payload = load_scenario("c3_lb_two_servers.yml", 10)
    runner = SweepRunner(payload, 2, {("lb_algorithm",): ["least_connection", "round_robin"], ("lb_covered", "srv-2"): [1, False]})
    from asyncflow_b200.results import SweepResults
    flat = runner.flat
    n = 2
    res = SweepResults(flat, np.zeros(n, dtype=K.STATS_DTYPE), np.zeros((n, flat.n_edges), np.uint32),
                       np.zeros((n, flat.n_edges), np.uint32), np.zeros((n, flat.n_series), np.uint64),
                       np.zeros((n, flat.n_series), np.uint32), None, None, 0)
    df = runner.frame(res)
    assert list(df["lb_algorithm"]) == ["least_connection", "round_robin"]
    assert list(df["lb_covered:srv-2"]) == [1.0, 0.0]
