"""GPU tier: occupancy integrals (af_occupancy_configure / af_fetch_occupancy) on the device.  The rows must equal the
CPU twin's bit for bit on multi-wave launches in every pass structure, a stitched launch included; be the same in the
lean and the full build; leave every other output and every kind of band unchanged; add up across shards of one sweep;
and be patched by the retries of ``run(retry_overflow=True)``."""

from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest
import twin
from helpers import ROOT, SEED, load_scenario

from asyncflow_b200 import Engine, SweepRunner, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.engine import EngineError
from asyncflow_b200.results import SweepResults

pytestmark = pytest.mark.gpu

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW
F = 32


def _c3(horizon: int = 10):
    return flatten(load_scenario("c3_lb_two_servers.yml", horizon))


def _sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def launch(flat, n, *, mode="auto", occ=True, f=F, rq=0, ev=0, groups=None, G=1, sampled=True, window=0, series=None,
           trace=0):
    eng = Engine(0)
    eng.upload(flat)
    eng.set_mode(mode)
    eng.configure(request_capacity=rq, event_capacity=ev, throughput=True, trace_replicas=trace,
                  trace_clock_capacity=20000 if trace else 0)
    eng.configure_occupancy(occ, f)
    if groups is not None:
        eng.configure_bands(sampled=sampled, latency_window_s=window)
        eng.configure_dist_bands(series)
        eng.upload_bands(np.asarray(groups, dtype=np.uint32), 0, G)
    eng.run(SEED, 0, n)
    return eng


def outputs(eng: Engine) -> dict:
    st = eng.stats().copy()
    sent, dropped = eng.edge_counts()
    ssum, smax = eng.sampled()
    return {"stats": st.tobytes(), "sent": sent.tobytes(), "dropped": dropped.tobytes(), "ssum": ssum.tobytes(),
            "smax": smax.tobytes(), "thr": eng.throughput().tobytes(), "hist": eng.histograms().tobytes()}


def twin_rows(flat, ids) -> np.ndarray:
    return np.stack([twin.run_lane(flat, seed=SEED, n=1, replica_begin=int(i), f=F)["occ"][0] for i in ids])


@pytest.mark.parametrize("mode", ["auto", "lane", "warp", "two_pass"])
def test_rows_equal_the_twin_on_a_multiwave_launch(mode):
    flat = _c3()
    n = _sm_count() * 12 * 32 + 1500                   # more than one wave of the thread-per-replica pass
    eng = launch(flat, n, mode=mode)
    occ, f = eng.occupancy()
    passes = eng.last_run_passes()
    assert f == F and occ.shape == (n, twin.occ_cols(flat))
    assert (eng.stats()["flags"] & STOPS == 0).all()
    if mode != "warp":
        assert passes["lane_pass"] == 1 and n > _sm_count() * passes["lane_warps_per_sm"] * 32, passes
    ids = np.unique(np.concatenate([np.arange(8), np.linspace(0, n - 1, 24).astype(np.int64), np.arange(n - 8, n)]))
    assert occ[ids].tobytes() == twin_rows(flat, ids).tobytes()
    assert occ.all(axis=0)[[1, 2, 3, 4]].all()          # server 0: cpu_wait, cpu, io, ram_mb


def test_a_stitched_launch_gives_the_warp_pass_rows():
    flat = flatten(load_scenario("overload_single.yml"))
    n = 2000
    two = launch(flat, n, mode="two_pass")
    passes = two.last_run_passes()
    warp = launch(flat, n, mode="warp")
    assert passes["warp_replicas"] >= 1, passes
    assert two.occupancy()[0].tobytes() == warp.occupancy()[0].tobytes()
    ids = np.flatnonzero(np.arange(n) % 400 == 0)
    rows = np.stack([twin.run_warp(flat, seed=SEED, n=1, replica_begin=int(i), f=F)["occ"][0] for i in ids])
    assert two.occupancy()[0][ids].tobytes() == rows.tobytes()


BAND_KINDS = [None, dict(sampled=True), dict(sampled=False, window=2), dict(sampled=False, series=[0, 3]),
              dict(sampled=True, window=2, series=[0, 1, 2, 3])]


@pytest.mark.parametrize("bands", BAND_KINDS, ids=lambda b: "none" if b is None else "+".join(k for k in sorted(b) if b[k]))
@pytest.mark.parametrize("mode", ["two_pass", "warp"])
def test_on_equals_off_for_every_other_output(bands, mode):
    flat = _c3()
    n, G = 4096, 3
    kw = {} if bands is None else dict(groups=np.arange(n) % G, G=G, **bands)
    on, off = launch(flat, n, mode=mode, **kw), launch(flat, n, mode=mode, occ=False, **kw)
    assert on.occupancy()[0].any()
    assert outputs(on) == outputs(off)
    if bands is not None:
        if bands.get("sampled"):
            assert all(a.tobytes() == b.tobytes() for a, b in zip(on.bands(), off.bands()))
        if bands.get("window"):
            assert all(a.tobytes() == b.tobytes() for a, b in zip(on.latency_bands(), off.latency_bands()))
        if bands.get("series"):
            assert on.dist_bands().tobytes() == off.dist_bands().tobytes()
    with pytest.raises(EngineError, match="no occupancy"):
        off.occupancy()


def test_lean_and_full_builds_agree(monkeypatch):
    flat = _c3()
    n = 4096
    a = launch(flat, n, mode="two_pass")
    monkeypatch.setenv("ASYNCFLOW_B200_LANE_FULL", "1")
    b = launch(flat, n, mode="two_pass")
    assert a.last_run_passes()["lane_lean"] == 1 and b.last_run_passes()["lane_lean"] == 0
    assert a.occupancy()[0].tobytes() == b.occupancy()[0].tobytes()


def test_a_bound_that_does_not_fit_is_refused():
    flat = flatten(load_scenario("c1_my_service.yml", 86_400))
    eng = Engine(0)
    eng.upload(flat)
    eng.configure(request_capacity=(1 << 20) - 1)
    eng.configure_occupancy(True, 28)
    with pytest.raises(EngineError, match=r"B = 1048575 .* H = 86400 s .* f = 28"):
        eng.run(SEED, 0, 4)
    with pytest.raises(EngineError, match="7 fraction bits"):
        eng.configure_occupancy(True, 7)


def test_two_shards_equal_one_launch_over_a_ram_sweep():
    payload = load_scenario("c3_lb_two_servers.yml", 10)
    flat = flatten(payload)
    n = 4000
    ram = np.where(np.arange(n) < n // 2, 1024.0, 1 << 22)       # the shards' largest ram_mb differ
    sweep = {("server_ram_mb", flat.server_ids[0]): ram}
    r = SweepRunner(payload, n, sweep, occupancy=True, pinned=False)
    whole = r.run()
    parts = SweepResults.concatenate([r.run(0, n // 2), r.run(n // 2, n)])
    assert whole.occ_frac_bits == parts.occ_frac_bits == r.occ_frac_bits
    assert whole.occupancy.tobytes() == parts.occupancy.tobytes()
    b = whole.breakdown()
    assert b["raw"] == parts.breakdown()["raw"] and abs(np.nansum(b["share"]) - 1.0) < 1e-9
    r.close()


def test_retry_overflow_patches_the_rows():
    payload = load_scenario("overload_single.yml")
    n = 256
    small = SweepRunner(payload, n, occupancy=True, request_capacity=64, event_capacity=64, pinned=False)
    first = small.run()
    assert first.overflowed.any()
    res = small.run(retry_overflow=True)
    big = SweepRunner(payload, n, occupancy=True, pinned=False).run()
    assert not res.overflowed.any() and not big.overflowed.any()
    assert res.occ_frac_bits == big.occ_frac_bits
    assert res.occupancy.tobytes() == big.occupancy.tobytes()
    assert (first.occupancy[first.overflowed] != res.occupancy[first.overflowed]).any()
    small.close()


def test_the_example_runs():
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    r = subprocess.run([sys.executable, str(ROOT / "examples" / "sweep_time_breakdown.py"), "--replicas", "256",
                        "--horizon", "20"], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "cpu_wait" in r.stdout and "users_mean" in r.stdout
