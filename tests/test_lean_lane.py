"""CPU tier: the lean build of the lane engine's loop (run_lane<*, *, true>: no spikes, outages, traces, general edge
samplers or endpoint draws) gives the same outputs as the full build, bit for bit, on every launch that qualifies for it
(aflh::lean_launch) -- with per-replica pool splits, sweeps and both kinds of bands -- and the qualification rule
rejects each feature the lean loop leaves out."""

from __future__ import annotations

import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario
from twin import lean_qualifies as qualifies

from asyncflow_b200 import SweepSpec, flatten

#: scenarios -> whether they qualify as written; the others run as one_endpoint() makes them
SCENARIOS = {"c3_lb_two_servers.yml": True, "c1_my_service.yml": True, "chain_two_servers.yml": True,
             "tie_cpu_io.yml": False, "poisson_ties.yml": False, "overload_single.yml": False}
BANDS = ((False, False), (True, False), (False, True), (True, True))    # (per-tick bands, latency bands)


def one_endpoint(payload: dict) -> dict:
    """The scenario with each server's last endpoint only and every edge without a normal / exponential latency made
    exponential with the same mean: what the lean loop can run.  tie_cpu_io, poisson_ties and overload_single keep
    their one- and two-core servers under load -- CPU and RAM waiter queues, now-queue ties."""
    for s in payload["topology_graph"]["nodes"]["servers"]:
        s["endpoints"] = s["endpoints"][-1:]
    for e in payload["topology_graph"]["edges"]:
        if e["latency"].get("distribution") not in ("normal", "exponential"):
            e["latency"] = {"mean": e["latency"]["mean"], "distribution": "exponential"}
    return payload


def scenario(name: str) -> dict:
    h = PARITY_CASES.get(name)
    payload = load_scenario(name, min(h, 30) if h else None)
    return payload if SCENARIOS[name] else one_endpoint(payload)


def assert_lean_equals_full(flat, *, n: int, **kw) -> dict:
    """The thread-per-replica engine over replicas [0, n) in groups i % 3, lean and full."""
    kw.update(seed=SEED, n=n, groups=np.arange(n) % 3, n_groups=3, split_seed=7, lane_bytes=604)
    lean, full = twin.run_lane(flat, lean=True, **kw), twin.run_lane(flat, lean=False, **kw)
    for k, v in full.items():
        assert v.tobytes() == lean[k].tobytes(), (k, kw)
    return lean


@pytest.mark.parametrize("name", SCENARIOS)
def test_lean_loop_equals_full_loop(name):
    """Every scenario, every band combination, the scenario's split and random per-replica splits."""
    assert qualifies(flatten(load_scenario(name))) == SCENARIOS[name]
    flat = flatten(scenario(name))
    assert qualifies(flat)
    for sampled, lat in BANDS:
        for split in ("scenario", "random"):
            out = assert_lean_equals_full(flat, n=6, split=split, sampled=sampled, window=2 if lat else 0)
            assert out["stats"]["completed"].sum() > 0


def test_lean_loop_equals_full_loop_on_bench_sweep_rows():
    """configs[2]'s shape (normal-jitter edges) on rows of the bench's own RTT x jitter grid, each replica split by
    its row's estimate as af_run does, at the bench's per-lane budget (604 B at 12 warps/SM)."""
    import bench
    flat = flatten(bench.workload(0, 6))
    assert qualifies(flat)
    ids = np.linspace(0, 99_999, 24).astype(np.int64)
    spec = SweepSpec(flat, ids.size, bench._c3_cols(flat, ids, 100_000))
    for sampled, lat in BANDS:
        out = assert_lean_equals_full(flat, n=ids.size, sweep=spec, split="rows", sampled=sampled, window=1 if lat else 0)
        assert (out["stats"]["completed"] > 0).all()


def test_qualification_rejects_every_feature_the_lean_loop_leaves_out():
    """Spikes and outages, a lognormal (general-sampler) edge, traced replicas, servers with two endpoints."""
    flat = flatten(load_scenario("ev_spikes_outages.yml"))
    assert flat.pod.n_spike_marks > 0 or flat.pod.n_outage_marks > 0
    assert not qualifies(flat)
    payload = load_scenario("c1_my_service.yml", 10)
    assert qualifies(flatten(payload)) and not qualifies(flatten(payload), trace_replicas=1)
    payload["topology_graph"]["edges"][1]["latency"] = {"mean": 0.003, "distribution": "log_normal", "variance": 0.001}
    assert not qualifies(flatten(payload))
    for name in ("c5_multihop32.yml", "mixed_lc.yml"):
        flat = flatten(load_scenario(name))
        assert any(flat.pod.servers[i].n_endpoints > 1 for i in range(flat.pod.n_servers)), name
        assert not qualifies(flat), name
    assert not qualifies(flatten(load_scenario("c4_lb8_events.yml")))
