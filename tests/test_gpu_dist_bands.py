"""GPU tier: per-tick distribution bands (af_dist_bands_configure / af_fetch_dist_bands) on the device.  The rows must be
the histogram of the device's own traced series over each group's replicas in every pass structure, a stitched launch
included; equal the CPU twin; be the same in the lean and the full build; leave every other output unchanged; and add
up across shards."""

from __future__ import annotations

import band_ref
import numpy as np
import pytest
import twin
from helpers import ROOT, SEED, load_scenario

from asyncflow_b200 import Engine, SweepRunner, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.engine import EngineError
from asyncflow_b200.results import SweepResults, gauge_bin_edges

pytestmark = pytest.mark.gpu

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW


def _bins(values: np.ndarray, B: int) -> np.ndarray:
    return np.minimum(np.searchsorted(gauge_bin_edges(B + 1), values, side="right") - 1, B - 1)


def traced_hist(eng: Engine, n: int, series, groups, G: int, B: int, upto=None) -> np.ndarray:
    """[G, n_dist, T, B] histogram of the traced replicas' series (replica i counts ticks < upto[i])."""
    T = None
    out = None
    for i in range(n):
        ser = eng.trace_series(i)
        if out is None:
            T = ser.shape[1]
            out = np.zeros((G, len(series), T, B), dtype=np.uint32)
        k = T if upto is None else min(int(upto[i]), T)
        for s, j in enumerate(series):
            out[groups[i], s, np.arange(k), _bins(ser[j, :k], B)] += 1
    return out


def launch(flat, n, series, groups, G, *, mode="auto", dist=True, sampled=True, window=0, trace=True, rq=0, ev=0):
    eng = Engine(0)
    eng.upload(flat)
    eng.set_mode(mode)
    eng.configure(trace_replicas=n if trace else 0, trace_clock_capacity=20000 if trace else 0, request_capacity=rq,
                  event_capacity=ev, throughput=True)
    eng.configure_bands(sampled=sampled, latency_window_s=window)
    eng.configure_dist_bands(series if dist else None)
    eng.upload_bands(np.asarray(groups, dtype=np.uint32), 0, G)
    eng.run(SEED, 0, n)
    return eng


def outputs(eng: Engine) -> dict:
    st = eng.stats().copy()
    sent, dropped = eng.edge_counts()
    ssum, smax = eng.sampled()
    return {"stats": st.tobytes(), "sent": sent.tobytes(), "dropped": dropped.tobytes(), "ssum": ssum.tobytes(),
            "smax": smax.tobytes(), "thr": eng.throughput().tobytes(), "hist": eng.histograms().tobytes()}


def _c3():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    series = [0, 3, 2, 3 * flat.n_servers]          # ready queues of both servers, ram of server 0, an edge
    return flat, series


@pytest.mark.parametrize("mode", ["auto", "lane", "warp", "two_pass"])
def test_rows_are_the_histogram_of_the_traced_series(mode):
    flat, series = _c3()
    n, G = 96, 3
    groups = np.arange(n) % G
    eng = launch(flat, n, series, groups, G, mode=mode)
    d = eng.dist_bands()
    st = eng.stats()
    assert (st["flags"] & STOPS == 0).all()
    assert d.shape[:2] == (G, len(series))
    np.testing.assert_array_equal(d, traced_hist(eng, n, series, groups, G, d.shape[3]))
    assert (d.sum(axis=3) == n // G).all()
    if mode == "two_pass":                          # the twin, both state machines
        tw = twin.run_lane(flat, seed=SEED, n=n, series=series, groups=groups, n_groups=G)
        np.testing.assert_array_equal(d, band_ref.dist_scan(tw["dist_rows"], G, d.shape[2]))


def test_a_stitched_launch_counts_each_replica_once():
    flat = flatten(load_scenario("overload_single.yml"))
    series = [0, 1, 2]
    n, G = 64, 2
    groups = np.arange(n) % G
    eng = launch(flat, n, series, groups, G, mode="two_pass", trace=False)
    passes = eng.last_run_passes()
    d = eng.dist_bands()
    ref = launch(flat, n, series, groups, G, mode="warp", trace=False)
    np.testing.assert_array_equal(d, ref.dist_bands())
    assert passes["warp_replicas"] >= 1, passes


def test_lean_and_full_builds_agree(monkeypatch):
    flat, series = _c3()
    n, G = 2000, 2
    groups = np.arange(n) % G
    a = launch(flat, n, series, groups, G, mode="two_pass", trace=False)
    lean = a.last_run_passes()["lane_lean"]
    monkeypatch.setenv("ASYNCFLOW_B200_LANE_FULL", "1")
    b = launch(flat, n, series, groups, G, mode="two_pass", trace=False)
    assert lean == 1 and b.last_run_passes()["lane_lean"] == 0
    np.testing.assert_array_equal(a.dist_bands(), b.dist_bands())


@pytest.mark.parametrize("sampled,window", [(True, 0), (False, 0), (True, 2), (False, 2)])
def test_other_outputs_do_not_change(sampled, window):
    flat, series = _c3()
    n, G = 3000, 4
    groups = np.arange(n) % G
    on = launch(flat, n, series, groups, G, sampled=sampled, window=window, trace=False)
    off = launch(flat, n, series, groups, G, sampled=sampled, window=window, dist=False, trace=False)
    assert outputs(on) == outputs(off)
    if sampled:
        for a, b in zip(on.bands(), off.bands()):
            np.testing.assert_array_equal(a, b)
        cnt, s, _ = on.bands()
        d = on.dist_bands()
        np.testing.assert_array_equal(d.sum(axis=3)[:, 0], cnt)
        edges = gauge_bin_edges(d.shape[3]).astype(np.uint64)
        small = d[:, 0][..., 64:].sum(axis=-1) == 0                       # series 0 stays below 64: sums are exact
        np.testing.assert_array_equal((d[:, 0].astype(np.uint64) * edges).sum(axis=-1)[small], s[:, series[0]][small])
    if window:
        for a, b in zip(on.latency_bands(), off.latency_bands()):
            np.testing.assert_array_equal(a, b)


def test_two_shards_concatenated_equal_one_launch():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    keys = [("ready_queue_len", "srv-1"), ("ready_queue_len", "srv-2")]
    flat = flatten(payload)
    if not set(k[1] for k in keys) <= set(flat.server_ids):
        keys = [("ready_queue_len", s) for s in flat.server_ids[:2]]
    users = np.repeat([20.0, 60.0, 120.0], 200)
    runner = SweepRunner(payload, users.size, {("users_mean",): users}, seed=SEED, bands=np.repeat([0, 1, 2], 200),
                         dist_series=keys)
    whole = runner.run()
    parts = SweepResults.concatenate([runner.run(0, 250), runner.run(250, users.size)])
    np.testing.assert_array_equal(whole.dist_hist, parts.dist_hist)
    g = whole.group_dist(*keys[0], at_least=1)
    assert g["q"].shape == (3, 5, whole.dist_hist.shape[2]) and np.isfinite(g["q"]).all()
    assert (np.diff(np.nanmean(g["q"][:, 2], axis=1)) >= 0).all()          # more users, longer queues
    runner.close()


def test_shards_with_different_swept_ram_concatenate_to_one_launch():
    """Each launch sizes its bins by its own rows' largest ram_mb: the shards differ in bin count, and concatenate pads
    them to the whole sweep's."""
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    srv = flat.server_ids[0]
    ram = np.repeat([4096.0, 8192.0, 65536.0, 131072.0], 150)
    runner = SweepRunner(payload, ram.size, {("server_ram_mb", srv): ram}, seed=SEED, bands=np.repeat([0, 1, 2, 3], 150),
                         dist_series=[("ram_in_use", srv), ("ready_queue_len", srv)])
    whole = runner.run()
    a, b = runner.run(0, 300), runner.run(300, ram.size)
    assert a.dist_hist.shape[-1] < b.dist_hist.shape[-1] == whole.dist_hist.shape[-1]
    np.testing.assert_array_equal(SweepResults.concatenate([a, b]).dist_hist, whole.dist_hist)
    runner.close()


def test_bad_series_and_oversized_rows_are_refused():
    flat, series = _c3()
    with Engine(0) as eng:
        eng.upload(flat)
        for bad in ([flat.n_series], [-1], [0, 0]):
            with pytest.raises(EngineError, match="distribution bands"):
                eng.configure_dist_bands(bad)
        eng.configure(request_capacity=(1 << 20) - 1)
        eng.configure_dist_bands(list(range(flat.n_series)))
        with pytest.raises(EngineError, match="GB of rows"):
            eng.upload_bands(np.arange(2_000_000, dtype=np.uint32) % 200_000, 0, 200_000)


def test_example_runs(monkeypatch, capsys):
    import runpy
    import sys
    monkeypatch.setattr(sys, "argv", ["sweep_outage_dist.py", "20"])
    runpy.run_path(str(ROOT / "examples" / "sweep_outage_dist.py"), run_name="__main__")
    assert "P(queue" in capsys.readouterr().out
