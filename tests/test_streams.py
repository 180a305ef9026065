"""Random streams (``af_streams_upload``, ``SweepRunner(streams=)``) on the CPU twin of both state machines: a replica
with a stream equals the oracle run with that stream as its replica id, bit for bit; an identity table changes no
output; rows that share a stream share their traffic; every path of ``SweepRunner`` keeps a row's stream; and
``SweepResults.paired`` does numpy's arithmetic and narrows the interval of a common-random-numbers comparison."""

from __future__ import annotations

import runpy
import sys

import band_ref
import des_port
import fuzz
import numpy as np
import pytest
import twin
import twin_streams
from event_rows import event_time_columns
from helpers import ROOT, SEED, assert_matches_oracle, load_scenario
from twin_engine import TwinEngine

from asyncflow_b200.flatten import SweepSpec, flatten
from asyncflow_b200.results import SweepResults
from asyncflow_b200.runner import SweepRunner

OUT = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max")
N = 6
FIRST = 1                                   # the table covers replicas 1 .. 4; replicas 0 and 5 draw as their own id
TABLE = np.array([7, 2**40 + 3, 7, 2**63 + 11], dtype=np.uint64)   # a repeat, streams >= 2^32 and >= 2^63


def stream_of(i: int) -> int:
    return int(TABLE[i - FIRST]) if FIRST <= i < FIRST + TABLE.size else i


def _named(name: str, horizon: int) -> tuple[dict, dict]:
    payload = load_scenario(name, horizon)
    flat = flatten(payload)
    rng = np.random.default_rng(11)
    servers = [s["id"] for s in payload["topology_graph"]["nodes"]["servers"]]
    cols = {("users_mean",): rng.uniform(0.5, 1.5, N) * flat.pod.users_mean,
            ("step_duration", servers[0], 0, 0): rng.choice([0.001, 0.002, 0.003], N)}
    if flat.events:
        cols.update(event_time_columns(flat, N, rng))
    return payload, cols


def _fuzz(seed: int) -> tuple[dict, dict]:
    payload = fuzz.scenario(seed)
    return payload, fuzz.sweep_columns(seed, payload, N)


CASES = {"c3_lb_two_servers": lambda: _named("c3_lb_two_servers.yml", 20),
         "c4_lb8_events": lambda: _named("c4_lb8_events.yml", 20),
         "mixed_lc": lambda: _named("mixed_lc.yml", 20),
         **{f"fuzz{s}": (lambda s=s: _fuzz(s)) for s in (300, 307, 316)}}


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("case", list(CASES))
def test_streams_equal_the_oracle(case, engine):
    payload, cols = CASES[case]()
    flat = flatten(payload)
    spec = SweepSpec(flat, N, cols)
    r = twin_streams.run(flat, seed=SEED, n=N, sweep=spec, trace=N, clock_cap=200000, request_capacity=200000,
                         engine=engine, streams=TABLE, stream_first=FIRST)
    for i in range(N):
        p = spec.payload_for(payload, i)
        o = des_port.simulate(p, seed=SEED, replica=stream_of(i))
        st = r["stats"][i]
        k, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0
        assert_matches_oracle(o, flatten(p), stats=st, clocks=r["trace_clocks"][i, :k], sent=r["sent"][i],
                              dropped=r["dropped"][i], series=r["trace_series"][i][:, :nt], throughput=r["thr"][i])


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_identity_table_changes_no_output(engine, lean):
    """Every output byte, with per-tick, latency and distribution bands and occupancy on."""
    name = "c3_lb_two_servers.yml" if lean else "c4_lb8_events.yml"
    payload, cols = _named(name, 20)
    flat = flatten(payload)
    begin = 5
    spec = SweepSpec(flat, N, cols)
    groups = np.array([0, 1, 0, 1, 1, 0], dtype=np.uint32)
    kw = dict(seed=SEED, n=N, replica_begin=begin, sweep=spec, sweep_first=begin, groups=groups, n_groups=2,
              band_first=begin, sampled=True, window=2, series=[0, 3], f=24, request_capacity=4096,
              event_capacity=2048, trace=2, clock_cap=50000)
    if engine == "lane":
        kw["lean"] = lean
        if lean:
            kw["trace"] = 0
            assert twin.lean_qualifies(flat)
    run = twin_streams.run_lane if engine == "lane" else twin_streams.run_warp
    none = run(flat, **kw)
    same = run(flat, **kw, streams=np.arange(begin, begin + N), stream_first=begin)
    for k in none:
        assert np.array_equal(none[k], same[k]), k
    other = run(flat, **kw, streams=np.arange(N) + 1000, stream_first=begin)
    assert not np.array_equal(none["stats"], other["stats"])


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_rows_that_share_a_stream_share_their_traffic(engine):
    payload = load_scenario("c3_lb_two_servers.yml", 20)
    flat = flatten(payload)
    # rows 0, 1: same parameters; rows 2, 3: the parsing steps of row 0 and a different one; all on stream 42
    cols = {("step_duration", "srv-1", 0, 0): [0.002, 0.002, 0.002, 0.0015],
            ("step_duration", "srv-2", 0, 0): [0.002, 0.002, 0.004, 0.0015],
            ("server_cpu_cores", "srv-2"): [1, 1, 2, 1]}
    spec = SweepSpec(flat, 4, cols)
    r = twin_streams.run(flat, seed=SEED, n=4, sweep=spec, engine=engine, streams=[42] * 4)
    for k in OUT:
        assert np.array_equal(r[k][0], r[k][1]), k
    upstream = [j for j, e in enumerate(payload["topology_graph"]["edges"]) if e["source"] in ("rqs-1", "client-1")]
    assert upstream == [0, 1]
    for i in (2, 3):
        assert r["stats"]["generated"][i] == r["stats"]["generated"][0]
        assert np.array_equal(r["sent"][i][upstream], r["sent"][0][upstream])
        assert np.array_equal(r["dropped"][i][upstream], r["dropped"][0][upstream])
        assert r["stats"]["lat_sum"][i] != r["stats"]["lat_sum"][0]


def test_a_warp_rerun_draws_from_the_replicas_stream():
    """af_run's second pass: the warp engine re-runs flagged replicas with their own streams, as a first-hand run."""
    payload, cols = _named("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    spec = SweepSpec(flat, N, cols)
    kw = dict(seed=SEED, n=N, sweep=spec, groups=np.zeros(N, dtype=np.uint32), sampled=True, f=24,
              streams=TABLE, stream_first=FIRST, request_capacity=4096, event_capacity=2048)
    lane = twin_streams.run_lane(flat, **kw, split="random", split_seed=3)
    warp = twin_streams.run_warp(flat, **kw)
    redo = np.arange(N, dtype=np.uint32)[::2]
    for k in ("stats", "sent", "occ"):
        lane[k][redo] = 0
    twin_streams.run_warp(flat, **kw, redo=redo, into=lane)
    for k in ("stats", "sent", "dropped", "samp_sum", "occ"):
        assert np.array_equal(lane[k][redo], warp[k][redo]), k


# ---- SweepRunner on the twin-backed engine ---------------------------------------------------------------------------
class StreamTwinEngine(TwinEngine):
    """TwinEngine with ``upload_streams``: its launches run on the twin with the stream table set."""

    streams = None
    stream_first = 0

    def upload_streams(self, streams, first_replica: int = 0) -> None:
        self.streams = None if streams is None else np.array(streams, dtype=np.uint64)
        self.stream_first = int(first_replica)
        self.calls.append(("upload_streams", int(first_replica), None if streams is None else len(streams)))

    def run(self, seed, begin, end) -> None:
        with twin_streams.rows(self.flat, streams=self.streams, stream_first=self.stream_first):
            super().run(seed, begin, end)


@pytest.fixture()
def twin_backed(monkeypatch):
    import asyncflow_b200
    import asyncflow_b200.runner as R
    monkeypatch.setattr(R, "Engine", StreamTwinEngine)
    monkeypatch.setattr(asyncflow_b200, "Engine", StreamTwinEngine)


def _c3_sweep(n: int, horizon: int = 10):
    payload = load_scenario("c3_lb_two_servers.yml", horizon)
    users = np.linspace(200.0, 1200.0, n)
    return payload, {("users_mean",): users}


def test_balance_deal_and_shards_keep_each_rows_stream(twin_backed):
    payload, cols = _c3_sweep(8)
    streams = np.array([3, 3, 2**35, 0, 9, 9, 1, 2**64 - 1], dtype=np.uint64)
    plain = SweepRunner(payload, 8, cols, streams=streams, request_capacity=20000).run()
    assert np.array_equal(plain.streams, streams)
    bal = SweepRunner(payload, 8, cols, streams=streams, balance=True, deal=2, request_capacity=20000)
    assert bal.order is not None and not np.array_equal(bal.replica_ids, np.arange(8))
    assert np.array_equal(bal.stream_ids, streams)
    full = bal.run()
    for k in ("stats", "edge_sent", "edge_dropped", "samp_sum", "samp_max"):
        assert np.array_equal(getattr(full, k), getattr(plain, k)), k
    assert np.array_equal(full.streams, streams)
    parts = [bal.run(0, 3), bal.run(3, 8)]                       # two shards, as distributed.run_sharded launches them
    cat = SweepResults.concatenate(parts)
    rows = np.concatenate([p.rows for p in parts])
    assert np.array_equal(cat.streams, streams[rows])
    for k in ("stats", "edge_sent", "samp_sum"):
        assert np.array_equal(getattr(cat, k), getattr(plain, k)[rows]), k
    # balancing without streams changes a row's draws (its replica id), with streams it does not
    unbal = SweepRunner(payload, 8, cols, balance=True, deal=2, request_capacity=20000).run()
    assert not np.array_equal(unbal.stats, plain.stats)


def test_replica_runner_exact_percentiles_and_frame_use_the_rows_stream(twin_backed):
    payload, cols = _c3_sweep(4)
    streams = [2**40 + 1, 5, 2**40 + 1, 77]
    sw = SweepRunner(payload, 4, cols, streams=streams, request_capacity=20000, balance=True)
    res = sw.run()
    assert [sw.replica_runner(i).replica for i in range(4)] == streams
    sw.exact_percentiles(res, [0, 3])
    for i in (0, 3):
        o = des_port.simulate(sw.payload_for(i), seed=sw.seed, replica=streams[i])
        lat = np.array([f - s for s, f in o["clocks"]])
        assert tuple(res.stats[["p50", "p95", "p99"]][i]) == tuple(np.percentile(lat, [50, 95, 99]))
        assert res.stats["completed"][i] == o["completed"]
    df = sw.frame(res)
    assert list(df["stream"]) == streams
    assert list(df["replica_id"]) == list(sw.replica_ids)
    plain = SweepRunner(payload, 4, cols, request_capacity=20000)
    assert np.array_equal(plain.stream_ids, plain.replica_ids)
    assert list(plain.frame(plain.run())["stream"]) == [0, 1, 2, 3]


def test_retry_overflow_reruns_with_the_rows_stream(twin_backed):
    payload, cols = _c3_sweep(4)
    streams = [2**50, 1, 2**50, 3]
    want = SweepRunner(payload, 4, cols, streams=streams, request_capacity=20000).run()
    sw = SweepRunner(payload, 4, cols, streams=streams, request_capacity=8, event_capacity=64)
    res = sw.run(retry_overflow=True)
    assert res.reran and not res.overflowed.any()
    for k in ("stats", "edge_sent", "samp_sum"):
        a, b = getattr(res, k), getattr(want, k)
        if k == "stats":
            a, b = a[["generated", "completed", "lat_sum", "lat_max", "n_events"]], b[["generated", "completed",
                                                                                        "lat_sum", "lat_max", "n_events"]]
        assert np.array_equal(a, b), k
    uploads = [c for c in sw._engine.calls if c[0] == "upload_streams"]
    assert len(uploads) > 1                                       # the launch and every re-run carry the table


@pytest.mark.parametrize("bad", [[-1, 0, 1, 2], [0, 1, 2, 2**64], [0.0, 1.0, 2.0, 3.0], [0, 1, 2], [True, 0, 1, 2],
                                 ["0", 1, 2, 3], [[0], [1], [2], [3]], [0, 1.5, 2, 3]], ids=str)
def test_refusals(bad):
    payload, cols = _c3_sweep(4)
    with pytest.raises(ValueError, match="streams"):
        SweepRunner(payload, 4, cols, streams=bad)


def test_accepted_stream_types():
    payload, cols = _c3_sweep(4)
    for good in ([0, 1, 2**64 - 1, 2**63], np.arange(4, dtype=np.int32), np.arange(4, dtype=np.uint64),
                 range(4)):
        sw = SweepRunner(payload, 4, cols, streams=good)
        assert sw.streams.dtype == np.uint64
        assert [int(x) for x in sw.stream_ids] == [int(x) for x in good]


# ---- paired differences ---------------------------------------------------------------------------------------------
def _results(x: np.ndarray) -> SweepResults:
    from asyncflow_b200 import _capi as K
    st = np.zeros(x.size, dtype=K.STATS_DTYPE)
    st["completed"] = 1
    st["lat_sum"] = x
    st["p95"] = 2 * x
    z = np.zeros((x.size, 1))
    return SweepResults(None, st, z, z, z, z)


def test_paired_arithmetic_matches_numpy():
    from statistics import NormalDist
    rng = np.random.default_rng(4)
    x = rng.normal(1.0, 0.3, 40)
    x[5] = np.nan
    res = _results(x)
    a, b = np.arange(0, 20), np.arange(20, 40)
    p = res.paired("mean", a, b, level=0.9)
    keep = np.isfinite(x[a]) & np.isfinite(x[b])
    xa, xb = x[a][keep], x[b][keep]
    d = xa - xb
    z = NormalDist().inv_cdf(0.95)
    n = d.size
    assert p["n"] == n == 19
    assert p["estimate"] == pytest.approx(d.mean(), rel=1e-15)
    assert p["half_width"] == pytest.approx(z * d.std(ddof=1) / np.sqrt(n), rel=1e-12)
    assert (p["lo"], p["hi"]) == (p["estimate"] - p["half_width"], p["estimate"] + p["half_width"])
    assert p["corr"] == pytest.approx(np.corrcoef(xa, xb)[0, 1], rel=1e-12)
    uh = z * np.sqrt((xa.var(ddof=1) + xb.var(ddof=1)) / n)
    assert p["unpaired_half_width"] == pytest.approx(uh, rel=1e-12)
    assert p["unpaired"][0] == pytest.approx(xa.mean() - xb.mean(), rel=1e-12)
    q = res.paired(2 * x, a, b, level=0.9)                        # an array: here the p95 column
    assert q["estimate"] == pytest.approx(res.paired("p95", a, b, level=0.9)["estimate"], rel=1e-15)
    assert q["estimate"] == pytest.approx(2 * p["estimate"], rel=1e-15)
    assert res.confidence_interval(2 * x) == res.confidence_interval("p95")
    with pytest.raises(ValueError):
        res.paired("mean", a, b[:3])
    with pytest.raises(ValueError):
        res.paired(x[:5], a, b)
    with pytest.raises(KeyError):
        res.paired("nope", a, b)
    assert np.isnan(res.paired("mean", [5], [6])["estimate"])
    one = res.paired("mean", [0], [1])
    assert one["n"] == 1 and one["half_width"] == 0.0 and np.isnan(one["corr"])


def test_paired_streams_narrow_the_interval_on_c3(twin_backed):
    """The measurement behind common random numbers (C3, 10 s, users_mean 1 500, both parsing steps 2 ms vs 1.5 ms,
    seed 7, 24 replicas per variant): shared streams give an interval of the mean latency difference at least twice
    narrower than independent ones."""
    payload = load_scenario("c3_lb_two_servers.yml", 10)
    payload["rqs_input"]["avg_active_users"]["mean"] = 1500
    R = 24
    variant = np.repeat([0, 1], R)
    dur = np.array([0.002, 0.0015])[variant]
    cols = {("step_duration", "srv-1", 0, 0): dur, ("step_duration", "srv-2", 0, 0): dur}
    sw = SweepRunner(payload, 2 * R, cols, seed=7, streams=np.tile(np.arange(R), 2), request_capacity=40000)
    res = sw.run()
    a, b = np.arange(R), np.arange(R, 2 * R)
    for what in ("mean", "p95"):
        p = res.paired(what, a, b)
        assert p["n"] == R and p["estimate"] > 0
        assert p["half_width"] <= 0.5 * p["unpaired_half_width"], (what, p)
        assert p["corr"] > 0.8
    indep = SweepRunner(payload, 2 * R, cols, seed=7, request_capacity=40000).run()
    assert indep.paired("mean", a, b)["corr"] < 0.5


# ---- the example and the tool ---------------------------------------------------------------------------------------
def test_paired_steps_example(twin_backed, monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", ["sweep_paired_steps.py", "--replicas", "3", "--horizon", "2"])
    runpy.run_path(str(ROOT / "examples" / "sweep_paired_steps.py"), run_name="__main__")
    out = capsys.readouterr().out
    assert "18 replicas in one launch" in out and "paired" in out and "unpaired" in out
    assert out.count("users ") == 6


def test_bench_streams_tool(monkeypatch, capsys):
    import json

    class Eng(StreamTwinEngine):
        def __init__(self, device: int = 0) -> None:
            super().__init__(device)
            self._ran = None

        def reduced_histogram(self):
            return self._r["hist"].astype(np.uint64).sum(axis=0)

    import asyncflow_b200.runner as R
    monkeypatch.setattr(R, "Engine", Eng)
    monkeypatch.setattr(sys, "argv", ["bench_streams.py", "--replicas", "3", "--horizon", "2", "--reps", "1"])
    runpy.run_path(str(ROOT / "tools" / "bench_streams.py"), run_name="__main__")
    row = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert row["identity_identical"] is True and row["none"] > 0 and row["shared"] > 0


def test_streams_with_bands_and_occupancy_lane_equals_warp():
    payload, cols = _named("c4_lb8_events.yml", 20)
    flat = flatten(payload)
    spec = SweepSpec(flat, N, cols)
    kw = dict(seed=SEED, n=N, sweep=spec, groups=np.array([0, 1, 0, 1, 1, 0], dtype=np.uint32), n_groups=2,
              sampled=True, window=2, series=[0, 3], f=24, request_capacity=4096, event_capacity=2048,
              streams=TABLE, stream_first=FIRST)
    lane = twin_streams.run_lane(flat, **kw)
    warp = twin_streams.run_warp(flat, **kw)
    for k in ("lat_rows", "occ", "stats", "samp_sum"):
        assert np.array_equal(lane[k], warp[k]), k
    for x, y in zip(band_ref.scan(flat, lane["band_rows"], 2), band_ref.scan(flat, warp["band_rows"], 2)):
        assert np.array_equal(x, y)
