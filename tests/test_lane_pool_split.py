"""CPU tier: the lane engine's shared-memory pool (af_lane.cuh) split PER REPLICA between heap entries and request
records, by each replica's own pending-events estimate (its sweep row's: aflh::row_events_estimates).  Whatever the
split, every replica equals the oracle bit for bit; the split itself follows the policy of afl::pool_events."""

from __future__ import annotations

import ctypes as C

import des_port
import numpy as np
import pytest
import split_twin
import twin
from helpers import PARITY_CASES, SEED, assert_matches_oracle, load_scenario

from asyncflow_b200 import SweepSpec, flatten


def _c3_rtt_spec(flat, rtt):
    rtt = np.asarray(rtt, dtype=np.float64)
    cols = {}
    for e in flat.edge_ids:
        cols[("edge_mean", e)] = rtt
        cols[("edge_sigma", e)] = 0.3 * rtt
    return SweepSpec(flat, len(rtt), cols)


def test_each_sweep_row_gets_the_split_of_its_own_load():
    """configs[2]'s shape at the bench budget (512 B of pool per lane at 12 warps/SM: 32 elements): a 1 ms row needs ~9
    pending events and keeps the even split (records fit), a 50 ms row needs ~34 and takes all but the 2-slot floor --
    and the split the launch reports (AfRunPasses) is the heaviest row's; the tests' launch-wide twin gives the sweep's
    maximum estimate the same split."""
    import bench
    payload = bench.workload(0, 6)
    flat = flatten(payload)
    spec = _c3_rtt_spec(flat, [0.001, 0.010, 0.025, 0.050])
    pool, reported, rows = split_twin.row_splits(flat, spec, 604)
    assert pool == 32
    needs = [r[0] for r in rows]
    assert needs == sorted(needs) and needs[0] <= 12 and needs[-1] >= 30, rows
    for need, ev, rq in rows:
        assert ev + rq == pool and 1 <= ev and 2 <= rq <= 32
        assert ev >= min(need, pool - 2)                  # never fewer events than needed while records hold more
        assert ev >= pool - (pool - 4) // 2               # never below the even split
    assert rows[0][1:] == (pool - (pool - 4) // 2, (pool - 4) // 2)
    assert rows[-1][1:] == (pool - 2, 2) and reported == rows[-1][1:]
    out = (C.c_int32 * 2)()
    sw, keep = spec.pod(0, None)
    assert twin.lib().af_twin_lane_split(C.byref(flat.pod), C.byref(sw), 604, 1, out) == 0
    del keep
    assert tuple(out) == rows[-1][1:]


def test_rows_with_very_different_splits_each_match_the_oracle():
    """One sweep, three rows that need very different splits of a small pool: a light row whose heap and records fit
    entirely, a heavy row that spills both tables to the global tier, and a 1-core server under load whose waiter FIFOs
    (CPU queue) run through shared-memory record slots."""
    payload = load_scenario("c1_my_service.yml", 4)
    flat = flatten(payload)
    users = np.array([5.0, 2000.0, 60.0])
    cores = np.array([1.0, 8.0, 1.0])
    spec = SweepSpec(flat, 3, {("users_mean",): users, ("server_cpu_cores", flat.server_ids[0]): cores})
    lane_bytes = 420
    r = split_twin.run(flat, lane_bytes=lane_bytes, split="rows", seed=SEED, n=3, sweep=spec, trace=3, clock_cap=100000,
                       request_capacity=200000)
    # the twin runs a warp of one lane: the same pool as 32 lanes of lane_bytes each
    _, _, rows = split_twin.row_splits(flat, spec, lane_bytes)
    st = r["stats"]
    for i in range(3):
        p = spec.payload_for(payload, i)
        o = des_port.simulate(p, seed=SEED, replica=i)
        m, nt = int(st[i]["completed"]), int(st[i]["n_ticks"])
        assert st[i]["flags"] == 0
        assert_matches_oracle(o, flatten(p), stats=st[i], clocks=r["trace_clocks"][i, :m], sent=r["sent"][i],
                              dropped=r["dropped"][i], series=r["trace_series"][i][:, :nt], throughput=r["thr"][i],
                              hist=r["hist"][i])
    (_, ev0, rq0), (_, ev1, rq1), (_, ev2, rq2) = rows
    assert st[0]["peak_events"] <= ev0 and st[0]["peak_requests"] <= rq0, (rows, st[0])
    assert st[1]["peak_events"] > ev1 and st[1]["peak_requests"] > rq1, (rows, st[1])
    assert st[2]["peak_requests"] <= rq2, (rows, st[2])
    assert r["samp_max"][2][0] > 0                          # requests did wait in app-1's ready queue


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_random_per_replica_splits_match_the_oracle(name):
    """Every replica of a launch on its own random split of the pool (2 .. pool - 1 record slots, the root still in
    shared memory), at budgets the CUDA engine runs: each replica equals the oracle."""
    payload = load_scenario(name, PARITY_CASES[name])
    flat = flatten(payload)
    r = split_twin.run(flat, lane_bytes=520, split="random", split_seed=7, seed=SEED, replica_begin=5, n=3, trace=3,
                       clock_cap=300000, request_capacity=400000, event_capacity=8192)
    for i in range(3):
        o = des_port.simulate(payload, seed=SEED, replica=5 + i)
        m, nt = int(r["stats"][i]["completed"]), int(r["stats"][i]["n_ticks"])
        assert r["stats"][i]["flags"] == 0
        assert_matches_oracle(o, flat, stats=r["stats"][i], clocks=r["trace_clocks"][i, :m], sent=r["sent"][i],
                              dropped=r["dropped"][i], series=r["trace_series"][i][:, :nt], throughput=r["thr"][i])
