"""GPU tier: whole launches in which lanes and warps run several replicas each, against the CPU twin, every replica and
every output.

In a launch that fits one wave, each lane runs at most one replica.  The cases here are sized from the device so that
lanes start their second and third replicas while the rest of their warp is mid-run (each with its own pool split, on
the lane's leftover shared-memory and global-tier state), the heaviest-first pull order spans several waves, warps
finish at different times, and the stitched re-run has more flagged replicas than warp slots.  Each case asserts the
launch shape it is meant to have.  Reference: the twin (tests/host_twin) over the same (seed, replicas, sweep rows),
which runs the replicas one after another.  Every replica's p50 / p95 / p99 must also be the bytes of the host
definition (afh::hist_percentile, results.hist_percentiles) on the device's own histogram."""

from __future__ import annotations

import des_port
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, assert_matches_oracle, load_scenario
from test_percentile_end_bins import LONG_KW, assert_percentiles, overload_payload

from asyncflow_b200 import Engine, SweepSpec, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.results import hist_percentiles

pytestmark = pytest.mark.gpu

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW
QS = ((50.0, "p50"), (95.0, "p95"), (99.0, "p99"))
#: the warp engine's default capacities, given to the pinned lane kernel too (it takes capacities as given)
CAPS = dict(event_capacity=2048, request_capacity=16384)
BEGIN = 1000
LANE_CASES = {"c1_my_service.yml": 3, "ev_spikes_outages.yml": 4, "tie_cpu_io.yml": 3, "mixed_lc.yml": 4,
              "c5_multihop32.yml": 3}
#: horizons of the warp-reuse case: the parity scenarios, shortened where a full run of hundreds of replicas is long
WARP_HORIZONS = {**PARITY_CASES, "c1_my_service.yml": 10, "c3_lb_two_servers.yml": 12, "c4_lb8_events.yml": 60,
                 "c5_multihop32.yml": 6}


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def light_heavy_rows(flat, n: int, seed: int) -> SweepSpec:
    """BEGIN + n rows (rows [BEGIN, BEGIN + n) describe replicas BEGIN, ...): users from 0.05 (replicas with 0, 1 or 2
    completions) to 400 interleaved at random, and an edge latency column, so that the pull order permutes heavily and
    consecutive replicas of a lane get different pool splits."""
    rng = np.random.default_rng(seed)
    m = BEGIN + n
    users = rng.choice([0.05, 0.3, 1.0, 4.0, 30.0, 120.0, 400.0], m)
    rtt = rng.choice([0.0005, 0.003, 0.02], m)
    return SweepSpec(flat, m, {("users_mean",): users, ("edge_mean", flat.edge_ids[1]): rtt})


def device_run(eng: Engine, flat, n: int, *, sweep=None, begin: int = BEGIN, rows: int | None = None, trace: int = 0,
               clock_cap: int = 0, **opts) -> dict:
    """Replicas [begin, begin + n); rows [begin, begin + rows) of ``sweep`` (default: one per replica) describe
    replicas begin, ..."""
    eng.upload(flat)
    eng.configure(trace_replicas=trace, trace_clock_capacity=clock_cap, **opts)
    if sweep is not None:
        eng.upload_sweep(sweep, begin, row_first=begin, row_count=n if rows is None else rows)
    else:
        eng.upload_sweep(None)
    eng.run(SEED, begin, begin + n)
    sent, dropped = eng.edge_counts()
    ssum, smax = eng.sampled()
    out = {"stats": eng.stats().copy(), "sent": sent, "dropped": dropped, "samp_sum": ssum, "samp_max": smax,
           "hist": eng.histograms(), "thr": eng.throughput(), "reduced": eng.reduced_histogram(),
           "passes": eng.last_run_passes()}
    if trace:
        out["clocks"] = [eng.trace_clocks(i) for i in range(trace)]
        out["series"] = [eng.trace_series(i) for i in range(trace)]
    return out


def twin_run(flat, n: int, *, sweep=None, begin: int = BEGIN, engine: str = "lane", **kw) -> dict:
    """The twin over what :func:`device_run` runs: every row of ``sweep`` from ``begin`` on."""
    return twin.run(flat, seed=SEED, replica_begin=begin, n=n, sweep=sweep, sweep_first=begin if sweep else 0,
                    engine=engine, **kw)


def assert_percentile_kernel(st: np.ndarray, hist: np.ndarray) -> None:
    """af_percentile_kernel == afh::hist_percentile == results.hist_percentiles on the device's histograms."""
    np.testing.assert_array_equal(hist.sum(axis=1, dtype=np.uint64), st["completed"])
    L = twin.lib()
    for q, key in QS:
        want = np.array([L.af_twin_hist_percentile(hist[i].ctypes.data, int(st["completed"][i]), q,
                                                   float(st["lat_min"][i]), float(st["lat_max"][i]))
                         for i in range(len(st))])
        bad = np.flatnonzero(st[key].view(np.uint64) != want.view(np.uint64))
        assert bad.size == 0, (key, bad[:8], st[key][bad[:8]], want[bad[:8]])
        np.testing.assert_array_equal(st[key], hist_percentiles(hist, q, lo=st["lat_min"], hi=st["lat_max"]), err_msg=key)


def assert_launch_equals_twin(dev: dict, ref: dict) -> None:
    assert not (dev["stats"]["flags"] & STOPS).any(), "device replicas stopped"
    assert not (ref["stats"]["flags"] & STOPS).any(), "twin replicas stopped"
    for k in ("stats", "sent", "dropped", "samp_sum", "samp_max", "hist", "thr"):
        a, b = dev[k], ref[k]
        assert a.shape == b.shape and a.dtype == b.dtype, k
        if a.tobytes() != b.tobytes():
            rows = np.flatnonzero((a.reshape(len(a), -1).view(np.uint8) != b.reshape(len(b), -1).view(np.uint8)).any(axis=1))
            pytest.fail(f"{k}: {rows.size} replicas differ from the twin, first local indices {rows[:8].tolist()}")
    assert dev["reduced"].tobytes() == ref["hist"].sum(axis=0, dtype=np.uint64).tobytes()
    assert_percentile_kernel(dev["stats"], dev["hist"])


@pytest.fixture(scope="module")
def eng():
    with Engine(0) as e:
        yield e
        e.set_mode("auto")


_refs: dict = {}


def lane_reference(name: str, n: int):
    if name not in _refs:
        flat = flatten(load_scenario(name, LANE_CASES[name]))
        spec = light_heavy_rows(flat, n, seed=len(name))
        _refs[name] = (flat, spec, twin_run(flat, n, sweep=spec, **CAPS))
    return _refs[name]


@pytest.mark.parametrize("mode", ["lane", "two_pass"])
@pytest.mark.parametrize("name", sorted(LANE_CASES))
def test_lanes_that_run_three_replicas_or_more_equal_the_twin(eng, name, mode):
    """One warp per SM (an explicit warps_per_block skips the whole-wave adjustment): every lane runs three replicas
    or four, the last warp ragged, rows from replica 1000 on."""
    sms = sm_count()
    lanes = sms * 32
    n = 3 * lanes + 17
    flat, spec, ref = lane_reference(name, n)
    eng.set_mode(mode)
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["lane_warps_per_sm"] == 1 and p["lane_replicas"] == n, p
    assert n >= 3 * sms * p["lane_warps_per_sm"] * 32
    if name == "c1_my_service.yml":
        assert p["lane_lean"] == 1, p
    if name == "ev_spikes_outages.yml":
        assert p["lane_lean"] == 0, p
    for k in (0, 1, 2):
        assert (ref["stats"]["completed"] == k).any(), f"no replica with {k} completions"
    assert_launch_equals_twin(dev, ref)


def test_the_default_shape_over_two_waves_equals_the_twin(eng):
    """AUTO with default options on the bench workload's rows: a little over one wave at the largest occupancy, so the
    policy takes two waves at a smaller one and most lanes run two replicas (lean build)."""
    import bench
    sms = sm_count()
    n = int(1.1 * sms * 12 * 32)
    flat = flatten(bench.workload(0, 2))
    ids = (np.arange(BEGIN + n, dtype=np.int64) * 7) % 100_000
    spec = SweepSpec(flat, BEGIN + n, bench._c3_cols(flat, ids, 100_000))
    eng.set_mode("auto")
    dev = device_run(eng, flat, n, sweep=spec)
    p = dev["passes"]
    lanes = sms * p["lane_warps_per_sm"] * 32
    assert p["lane_pass"] == 1 and p["lane_lean"] == 1 and n > lanes, p
    ref = twin_run(flat, n, sweep=spec)
    assert_launch_equals_twin(dev, ref)


def test_stitched_rerun_with_more_flagged_replicas_than_warp_slots_equals_the_twin(eng):
    """TWO_PASS, one lane warp and one re-run block (4 warps) per SM: overloaded rows overflow the lane pass's nominal
    pools, and the re-run pulls more of them than it has warps.  The caller's capacities hold every replica."""
    sms = sm_count()
    slots = 4 * sms
    n = 2 * slots
    flat = flatten(load_scenario("overload_single.yml", 8))
    rng = np.random.default_rng(3)
    spec = SweepSpec(flat, BEGIN + n, {("users_mean",): rng.choice([20.0, 500.0, 600.0], BEGIN + n, p=[0.2, 0.4, 0.4])})
    caps = dict(event_capacity=8192, request_capacity=1 << 15)
    eng.set_mode("two_pass")
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, blocks_per_sm=1, **caps)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["warp_pass"] == 1 and p["lane_replicas"] == n, p
    assert p["warp_replicas"] > slots, (p, slots)
    ref = twin_run(flat, n, sweep=spec, engine="warp", **caps)
    assert_launch_equals_twin(dev, ref)


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_warps_that_run_four_replicas_or_more_equal_the_twin(eng, name):
    """WARP mode, one warp per block and one block per SM: SMs warps for 4 x SMs + 7 replicas."""
    sms = sm_count()
    n = 4 * sms + 7
    payload = load_scenario(name, WARP_HORIZONS[name])
    flat = flatten(payload)
    eng.set_mode("warp")
    dev = device_run(eng, flat, n, warps_per_block=1, blocks_per_sm=1)
    p = dev["passes"]
    assert p["lane_pass"] == 0 and p["warp_pass"] == 1 and p["warp_replicas"] == n, p
    ref = twin_run(flat, n, engine="warp")
    assert_launch_equals_twin(dev, ref)
    if name not in ("c1_my_service.yml", "mixed_lc.yml", "chain_two_servers.yml"):
        return
    # a link that does not go through the twin: the replicas that generated most and least (pulled first and last by
    # the predicted-work order) and a few between, against the oracle
    gen = dev["stats"]["generated"].astype(np.int64)
    order = np.argsort(-gen, kind="stable")
    picks = sorted({int(order[0]), int(order[-1]), *(int(order[k]) for k in np.linspace(1, n - 2, 6).astype(int))})
    for i in picks:
        o = des_port.simulate(payload, seed=SEED, replica=BEGIN + i)
        assert_matches_oracle(o, flat, stats=dev["stats"][i], clocks=None, sent=dev["sent"][i], dropped=dev["dropped"][i],
                              throughput=dev["thr"][i], hist=dev["hist"][i])


def test_traced_launch_with_lane_reuse_equals_the_twin(eng):
    """Tracing (the full build of the lane kernel) on a launch whose lanes run three replicas or more: the 64 traced
    replicas' clocks and series equal the twin's."""
    sms = sm_count()
    n = 3 * sms * 32 + 17
    trace, cap = 64, 20_000
    flat, spec, _ = lane_reference("c1_my_service.yml", n)
    eng.set_mode("lane")
    dev = device_run(eng, flat, n, sweep=spec, trace=trace, clock_cap=cap, warps_per_block=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["lane_lean"] == 0 and p["lane_warps_per_sm"] == 1, p
    ref = twin_run(flat, n, sweep=spec, trace=trace, clock_cap=cap, **CAPS)
    assert_launch_equals_twin(dev, ref)
    for i in range(trace):
        m, nt = int(ref["stats"]["completed"][i]), int(ref["stats"]["n_ticks"][i])
        assert dev["clocks"][i].tobytes() == np.ascontiguousarray(ref["trace_clocks"][i, :m]).tobytes(), i
        assert dev["series"][i].tobytes() == np.ascontiguousarray(ref["trace_series"][i][:, :nt]).tobytes(), i


@pytest.mark.parametrize("mode", ["warp", "lane", "auto"])
def test_percentiles_past_the_last_bin_on_the_device(eng, mode):
    """The 9000 s overloaded replica: p50 / p95 / p99 within 1 % of numpy on its traced latencies, and the twin's
    bytes."""
    flat = flatten(overload_payload(9000, 8))
    eng.set_mode(mode)
    eng.upload(flat)
    eng.upload_sweep(None)
    eng.configure(trace_replicas=1, trace_clock_capacity=LONG_KW["clock_cap"], event_capacity=CAPS["event_capacity"],
                  request_capacity=LONG_KW["request_capacity"])
    eng.run(SEED, 0, 1)
    st, hist, clocks = eng.stats(), eng.histograms(), eng.trace_clocks(0)
    assert st[0]["flags"] == 0
    lat = clocks[:, 1] - clocks[:, 0]
    assert lat.max() > 4096.0
    assert_percentiles(st[0], hist[0], lat)
    ref = twin.run(flat, seed=SEED, n=1, trace=1, engine="warp", **LONG_KW)
    assert st.tobytes() == ref["stats"].tobytes()
    assert hist.tobytes() == ref["hist"].tobytes()
