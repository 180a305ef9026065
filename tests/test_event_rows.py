"""Per-replica event timelines (``("event_start"|"event_end", event_id)`` sweep columns, af_timeline_upload) on the CPU
twin of both state machines: every row equals the oracle run on ``SweepSpec.payload_for(row)``, the rows' fire times
are the oracle's, rows equal to the scenario's timeline change nothing, replicas without a row keep the scenario's,
every payload rule refuses a bad row by name, and the bands and occupancy of such a launch add up."""

from __future__ import annotations

import ctypes as C
import runpy
import sys
import time
import zlib

import band_ref
import des_port
import fuzz
import numpy as np
import pytest
import twin
import twin_rows
from event_rows import event_time_columns
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from twin_engine import TwinEngine

from asyncflow_b200 import _capi as K
from asyncflow_b200.flatten import SweepSpec, flatten

OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max")


def _fuzz_with_events() -> list[int]:
    return [s for s in range(100, 200) if {"sp1", "out1"} <= {e["event_id"] for e in fuzz.scenario(s).get("events") or []}][:4]


CASES = [("c4_lb8_events.yml", 20), ("ev_spikes_outages.yml", None)] + [f"fuzz:{s}" for s in _fuzz_with_events()]


def _payload(case):
    if isinstance(case, str) and case.startswith("fuzz:"):
        return fuzz.scenario(int(case[5:]))
    return load_scenario(*case)


def _check_rows(payload, flat, spec, r: dict, rows, first: int = 0) -> None:
    for i in rows:
        p = spec.payload_for(payload, i)
        o = des_port.simulate(p, seed=SEED, replica=first + i)
        st = r["stats"][i]
        k, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0
        assert_matches_oracle(o, flatten(p), stats=st, clocks=r["trace_clocks"][i, :k], sent=r["sent"][i],
                              dropped=r["dropped"][i], series=r["trace_series"][i][:, :nt], throughput=r["thr"][i])


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("amp", [False, True])
@pytest.mark.parametrize("case", CASES, ids=str)
def test_rows_equal_the_oracle(case, amp, engine):
    payload = _payload(case)
    flat = flatten(payload)
    n = 4
    rng = np.random.default_rng(zlib.crc32(f"{case}{amp}".encode()))
    spec = SweepSpec(flat, n, event_time_columns(flat, n, rng, spike_delta=amp))
    r = twin_rows.run(flat, seed=SEED, n=n, sweep=spec, trace=n, clock_cap=200000, request_capacity=200000, engine=engine)
    _check_rows(payload, flat, spec, r, range(n))


def test_an_outage_moved_across_the_spikes_reorders_the_marks():
    """ev_spikes_outages: srv-1's first outage moved to before, inside and after the others; the spikes' start and
    end swapped around each other."""
    payload = load_scenario("ev_spikes_outages.yml")
    flat = flatten(payload)
    start = np.array([0.0, 3.0, 20.0, 19.5])
    cols = {("event_start", "ev-e"): start, ("event_end", "ev-e"): start + np.array([5.0, 15.0, 8.0, 10.0]),
            ("event_start", "ev-a"): [12.0, 5.0, 25.0, 10.0], ("event_end", "ev-a"): [30.0, 9.0, 26.0, 20.0],
            ("spike_delta", "ev-b"): [0.5, 0.0, 0.25, 0.2]}
    spec = SweepSpec(flat, 4, cols)
    orders = {tuple(m) for m in spec.timelines.outage_mark} | {tuple(m) for m in spec.timelines.spike_mark}
    assert len(orders) > 2
    for engine in ("lane", "warp"):
        r = twin_rows.run(flat, seed=SEED, n=4, sweep=spec, trace=4, clock_cap=200000, request_capacity=200000,
                     engine=engine)
        _check_rows(payload, flat, spec, r, range(4))


def _oracle_fires(times) -> list[float]:
    """The oracle's clock at each mark of a sorted timeline (des_port's injection generators on its SimPy)."""
    import simpy
    env = simpy.Environment()
    out: list[float] = []

    def proc():
        last_t = float(env.now)
        for t in times:
            dt = t - last_t
            if dt > 0.0:
                yield env.timeout(dt)
            last_t = t
            out.append(env.now)
    env.process(proc())
    env.run()
    return out


def test_fire_times_of_non_representable_times_and_ties_are_the_oracles():
    payload = load_scenario("ev_spikes_outages.yml")
    flat = flatten(payload)
    third = 1.0 / 3.0
    cols = {("event_start", "ev-a"): [0.1, 0.3, third, 2.0], ("event_end", "ev-a"): [0.3, 0.7, 2 * third, 5.0],
            ("event_start", "ev-b"): [0.3, 0.1 + 0.2, third, 2.0], ("event_end", "ev-b"): [0.7, 0.9, 1.1, 5.5],
            ("event_start", "ev-e"): [0.1, 0.2, third, 5.0], ("event_end", "ev-e"): [0.3, 1.3, 0.7, 7.0],
            ("event_start", "ev-f"): [0.3, 1.3, 0.7, 7.0], ("event_end", "ev-f"): [1.7, 2.9, 1.9, 9.0]}
    spec = SweepSpec(flat, 4, cols)
    key = lambda m: (m[0], m[3] == "start", m[1], m[2])  # noqa: E731  (the reference's sort key)
    for i in range(4):
        p = spec.payload_for(payload, i)
        edges = {e["id"] for e in p["topology_graph"]["edges"]}
        spikes, outs = [], []
        for ev in p["events"]:
            marks = [(float(ev["start"]["t_start"]), ev["event_id"], ev["target_id"], "start"),
                     (float(ev["end"]["t_end"]), ev["event_id"], ev["target_id"], "end")]
            (spikes if ev["target_id"] in edges else outs).extend(marks)
        for table, marks in ((spec.timelines.spikes[i], spikes), (spec.timelines.outages[i], outs)):
            want = _oracle_fires([m[0] for m in sorted(marks, key=key)])
            assert [float(x) for x in table["fire_time"]] == want
        single = flatten(p)                     # the scenario path gives the same tables
        assert C.string_at(single.pod.spike_marks, spec.timelines.spikes[i].nbytes) == spec.timelines.spikes[i].tobytes()
        assert C.string_at(single.pod.outage_marks, spec.timelines.outages[i].nbytes) == spec.timelines.outages[i].tobytes()
    for engine in ("lane", "warp"):
        r = twin_rows.run(flat, seed=SEED, n=4, sweep=spec, trace=4, clock_cap=200000, request_capacity=200000,
                     engine=engine)
        _check_rows(payload, flat, spec, r, range(4))


def _same_as_scenario(flat, n: int) -> SweepSpec:
    cols = {}
    for e in flat.events:
        cols[("event_start", e.event_id)] = np.full(n, e.t_start)
        cols[("event_end", e.event_id)] = np.full(n, e.t_end)
    return SweepSpec(flat, n, cols)


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_rows_equal_to_the_scenario_change_nothing(engine):
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    n = 3
    a = twin_rows.run(flat, seed=SEED, n=n, replica_begin=5, engine=engine, trace=n, clock_cap=100000)
    b = twin_rows.run(flat, seed=SEED, n=n, replica_begin=5, engine=engine, trace=n, clock_cap=100000,
                 timeline=_same_as_scenario(flat, 8))
    for k in twin.OUTPUTS:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_replicas_outside_the_rows_run_the_scenarios_timeline(engine):
    payload = load_scenario("ev_spikes_outages.yml")
    flat = flatten(payload)
    n = 6
    spec = SweepSpec(flat, n, event_time_columns(flat, n, np.random.default_rng(3)))
    full = twin_rows.run(flat, seed=SEED, n=n, engine=engine, sweep=spec)
    none = twin_rows.run(flat, seed=SEED, n=n, engine=engine)
    part = twin_rows.run(flat, seed=SEED, n=n, engine=engine, timeline=spec, timeline_first=2, timeline_rows=2)
    for k in OUT:
        assert np.array_equal(part[k][2:4], full[k][2:4]), k
        assert np.array_equal(part[k][[0, 1, 4, 5]], none[k][[0, 1, 4, 5]]), k
    assert not np.array_equal(full["stats"], none["stats"])


# ---- validation ----------------------------------------------------------------------------------------------------
def _good(flat, n):
    return event_time_columns(flat, n, np.random.default_rng(11))


@pytest.mark.parametrize(("edit", "words"), [
    ({("event_start", "ev-a"): -1.0}, "0 <= t_start < t_end <= the horizon"),
    ({("event_end", "ev-c"): 41.0}, "0 <= t_start < t_end <= the horizon"),
    ({("event_start", "ev-f"): 12.0, ("event_end", "ev-f"): 12.0}, "0 <= t_start < t_end"),
    ({("event_start", "ev-g"): float("nan")}, "0 <= t_start"),
    ({("spike_delta", "ev-b"): -0.1}, "spike_s is finite and >= 0"),
])
def test_each_time_rule_refuses_a_bad_row_by_name(edit, words):
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    cols = _good(flat, 5)
    for sel, v in edit.items():
        col = np.array(cols.get(sel, np.full(5, 0.1)), dtype=float)
        col[3] = v
        cols[sel] = col
    with pytest.raises(ValueError, match="sweep row 3: event") as e:
        SweepSpec(flat, 5, cols)
    assert words in str(e.value)


def test_overlapping_outages_of_one_server_are_refused():
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    cols = _good(flat, 4)
    cols[("event_start", "ev-g")] = np.array(cols[("event_start", "ev-g")])
    cols[("event_end", "ev-e")] = np.array(cols[("event_end", "ev-e")])
    cols[("event_start", "ev-g")][2] = cols[("event_end", "ev-e")][2] - 0.01
    with pytest.raises(ValueError, match=r"sweep row 2: event 'ev-g'.*overlaps the outage 'ev-e'"):
        SweepSpec(flat, 4, cols)
    cols[("event_start", "ev-g")][2] = cols[("event_end", "ev-e")][2]          # back to back is fine
    SweepSpec(flat, 4, cols)


def test_every_server_down_is_refused():
    p = load_scenario("ev_spikes_outages.yml")
    p["events"].append({"event_id": "ev-h", "target_id": "srv-3", "start": {"kind": "server_down", "t_start": 1.0},
                        "end": {"kind": "server_up", "t_end": 2.0}})
    flat = flatten(p)
    cols = {("event_start", "ev-h"): [1.0, 11.0, 1.0], ("event_end", "ev-h"): [2.0, 12.0, 2.0],
            ("event_start", "ev-f"): [18.0, 10.0, 18.0], ("event_end", "ev-f"): [28.25, 20.0, 28.25]}
    with pytest.raises(ValueError, match="sweep row 1: event 'ev-h'.*every server is down"):
        SweepSpec(flat, 3, cols)


def test_an_empty_load_balancer_is_refused():
    """Servers chained behind the covered ones keep the reference's all-down rule quiet; flatten's own rule that the
    LB keeps an edge until the horizon applies to every row."""
    p = load_scenario("ev_spikes_outages.yml")
    p["events"] = [e for e in p["events"] if e["event_id"] in ("ev-e", "ev-f")]
    p["events"].append({"event_id": "ev-h", "target_id": "srv-3", "start": {"kind": "server_down", "t_start": 1.0},
                        "end": {"kind": "server_up", "t_end": 2.0}})
    p["topology_graph"]["nodes"]["servers"].append({"id": "srv-4", "server_resources": {"cpu_cores": 1, "ram_mb": 256},
                                                    "endpoints": [{"endpoint_name": "/a", "steps": [
                                                        {"kind": "initial_parsing", "step_operation": {"cpu_time": 0.001}}]}]})
    for e in p["topology_graph"]["edges"]:
        if e["source"] == "srv-3":
            e["target"] = "srv-4"
    p["topology_graph"]["edges"].append({"id": "srv4-client", "source": "srv-4", "target": "client-1",
                                         "latency": {"mean": 0.003, "distribution": "exponential"}})
    flat = flatten(p)
    cols = {("event_start", "ev-h"): [1.0, 8.5], ("event_end", "ev-h"): [2.0, 12.0],
            ("event_start", "ev-f"): [18.0, 10.0], ("event_end", "ev-f"): [28.25, 20.0]}
    with pytest.raises(ValueError, match="sweep row 1: event injection: at t=10s every server behind the load balancer"):
        SweepSpec(flat, 2, cols)


def test_unknown_events_are_refused():
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    with pytest.raises(KeyError):
        SweepSpec(flat, 2, {("event_start", "nope"): [1.0, 2.0]})
    with pytest.raises(KeyError, match="no spike event"):
        SweepSpec(flat, 2, {("event_start", "ev-a"): [1.0, 2.0], ("spike_delta", "ev-e"): [0.1, 0.1]})


def test_a_million_rows_validate_in_seconds():
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    n = 1_000_000
    cols = event_time_columns(flat, n, np.random.default_rng(2), spike_delta=True)
    t0 = time.perf_counter()
    spec = SweepSpec(flat, n, cols)
    assert time.perf_counter() - t0 < 30.0
    assert spec.timelines.spikes.shape == (n, 8) and spec.timelines.outages.shape == (n, 6)
    assert spec.n_columns == 0 and spec.timeline_row_bytes == 8 * 24 + 6 * 16


def _tl(spikes: np.ndarray, outages: np.ndarray):
    return K.AfTimeline(spikes.shape[0], spikes.ctypes.data_as(C.POINTER(K.AfSpikeMark)),
                        outages.ctypes.data_as(C.POINTER(K.AfOutageMark)))


class _Rows:
    """A stand-in for a SweepSpec that hands the twin hand-made timeline rows."""

    def __init__(self, spikes, outages):
        self.spikes, self.outages = np.ascontiguousarray(spikes), np.ascontiguousarray(outages)
        self.timelines = self

    def timeline_pod(self, first, count):
        return _tl(self.spikes, self.outages), None


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize(("bad", "words"), [
    ("edge", "timeline row 1: spike mark 2: edge 99 out of range"),
    ("spike_order", "timeline row 1: spike marks unsorted at mark 3"),
    ("outage_order", "timeline row 1: outage marks unsorted at mark 1"),
    ("lb_edge", "timeline row 1: outage mark 0: lb_edge 0 is neither -1 nor an edge of the load balancer"),
])
def test_the_c_checks_refuse_malformed_rows(engine, bad, words):
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    spec = _same_as_scenario(flat, 2)
    sp, ou = spec.timelines.spikes.copy(), spec.timelines.outages.copy()
    if bad == "edge":
        sp[1, 2]["edge"] = 99
    elif bad == "spike_order":
        sp[1, 3]["fire_time"] = sp[1, 2]["fire_time"] - 1.0
    elif bad == "outage_order":
        ou[1, 1]["fire_time"] = ou[1, 0]["fire_time"] - 1.0
    else:
        ou[1, 0]["lb_edge"] = 0
    with pytest.raises(RuntimeError, match=words):
        twin_rows.run(flat, seed=SEED, n=2, engine=engine, timeline=_Rows(sp, ou))


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_a_spike_delta_column_with_timeline_rows_is_refused(engine):
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    amp = SweepSpec(flat, 2, {("spike_delta", "ev-a"): [0.1, 0.2]})
    assert amp.timelines is None and amp.n_columns == 2
    with pytest.raises(RuntimeError, match="AF_FIELD_SPIKE_DELTA"):
        twin_rows.run(flat, seed=SEED, n=2, engine=engine, sweep=amp, timeline=_same_as_scenario(flat, 2))


def test_struct_size_matches_the_header():
    assert C.sizeof(K.AfTimeline) == twin_rows.lib().af_twin_rows_sizeof_timeline() == 24


# ---- bands and occupancy ---------------------------------------------------------------------------------------------
def test_bands_and_occupancy_with_timeline_rows():
    """Per-tick, latency and distribution bands and occupancy of a launch with timeline rows: both state machines agree,
    and the per-tick bands are the sums of the replicas' own traced series."""
    payload = load_scenario("ev_spikes_outages.yml", 20)
    for e in payload["events"]:
        e["start"]["t_start"], e["end"]["t_end"] = min(e["start"]["t_start"], 10.0), min(e["end"]["t_end"], 20.0)
    flat = flatten(payload)
    n = 6
    spec = SweepSpec(flat, n, event_time_columns(flat, n, np.random.default_rng(8), spike_delta=True))
    groups = np.array([0, 1, 0, 1, 1, 0], dtype=np.uint32)
    kw = dict(seed=SEED, n=n, sweep=spec, groups=groups, n_groups=2, sampled=True, window=2, series=[0, 3], f=24,
              request_capacity=4096, event_capacity=2048)
    lane = twin_rows.run_lane(flat, **kw)
    warp = twin_rows.run_warp(flat, **kw)
    for k in ("lat_rows", "occ", "stats", "samp_sum"):
        assert np.array_equal(lane[k], warp[k]), k
    for x, y in zip(band_ref.scan(flat, lane["band_rows"], 2), band_ref.scan(flat, warp["band_rows"], 2)):
        assert np.array_equal(x, y)
    T = twin.ticks(flat)
    assert np.array_equal(band_ref.dist_scan(lane["dist_rows"], 2, T), band_ref.dist_scan(warp["dist_rows"], 2, T))
    tr = twin_rows.run(flat, seed=SEED, n=n, sweep=spec, trace=n, clock_cap=100000)
    count, s, _ = band_ref.scan(flat, lane["band_rows"], 2)
    for g in range(2):
        mine = [i for i in range(n) if groups[i] == g]
        T = count.shape[1]
        want = sum(tr["trace_series"][i][:, :T].astype(np.uint64) for i in mine)
        assert np.array_equal(s[g], want)
    assert not np.array_equal(lane["occ"], twin_rows.run_lane(flat, **{**kw, "sweep": None})["occ"])


# ---- the example and the tool, dry-run on the twin-backed engine ----------------------------------------------------
class LatencyTwinEngine(TwinEngine):
    """TwinEngine with the sweep's timeline rows and latency bands (the lane state machine), for the example and the
    tool."""

    band_groups = None

    def upload_bands(self, groups, first_replica: int = 0, n_groups=None) -> None:
        self.band_groups = None if groups is None else np.asarray(groups, dtype=np.uint32)
        self.band_first, self.n_groups = int(first_replica), n_groups

    def configure_bands(self, *, sampled: bool = True, latency_window_s: int = 0) -> None:
        self.window = latency_window_s

    def run(self, seed, begin, end) -> None:
        with twin_rows.rows(self.flat, self.sweep, begin):          # the sweep's timeline rows, as upload_sweep's
            super().run(seed, begin, end)
        if self.band_groups is not None:
            out = twin_rows.run_lane(self.flat, seed=seed, n=end - begin, replica_begin=begin, sweep=self.sweep,
                                sweep_first=begin, groups=self.band_groups, n_groups=self.n_groups,
                                band_first=self.band_first, window=self.window)
            self._lat = twin.lat_split(out["lat_rows"], self.n_groups)

    def latency_bands(self):
        return self._lat


@pytest.fixture()
def twin_backed(monkeypatch):
    import asyncflow_b200
    import asyncflow_b200.runner as R
    monkeypatch.setattr(R, "Engine", LatencyTwinEngine)
    monkeypatch.setattr(asyncflow_b200, "Engine", LatencyTwinEngine)


def test_outage_duration_example(twin_backed, monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_outage_duration.py", "1"])
    runpy.run_path(str(ROOT / "examples" / "sweep_outage_duration.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "8 replicas in one launch" in out and "whole run, p95" in out and "down  60 s" in out


def test_bench_event_rows_tool(twin_backed, monkeypatch, capsys):
    import json
    monkeypatch.setattr(sys, "argv", ["bench_event_rows.py", "--replicas", "2", "--horizon", "30", "--reps", "1"])
    runpy.run_path(str(ROOT / "tools" / "bench_event_rows.py"), run_name="__main__")
    row = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert row["rows_identical"] is True and row["scenario"] > 0 and row["random"] > 0
