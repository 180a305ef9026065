"""CPU tier: per-tick distribution bands (af_dist_bands_configure / af_fetch_dist_bands).  Both state machines, driven
with their difference rows by the CPU twin (tests/twin.py), must give per group, tick and value bin exactly the
histogram of the oracle's sampled series over the group's replicas: first-hand, stitched (a replica the
thread-per-replica pass stops and the warp-per-replica pass re-runs from its stop tick), truncated (a stopped replica
that is not re-run, its zeros included), with every other output unchanged; and the host side must read quantiles,
extremes and exceedance off the counts as numpy reads them off the values."""

from __future__ import annotations

import band_ref
import des_port
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario, oracle_series_matrix

from asyncflow_b200 import flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.distributed import BAND_FIELDS
from asyncflow_b200.results import SweepResults, gauge_bin_edges

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW


def bins_of(values: np.ndarray, B: int) -> np.ndarray:
    return np.minimum(np.searchsorted(gauge_bin_edges(B + 1), values, side="right") - 1, B - 1)


def oracle_matrix(payload, flat, replica: int) -> np.ndarray:
    o = des_port.simulate(payload, seed=SEED, replica=replica)
    m = oracle_series_matrix(o, flat)
    T = twin.ticks(flat)
    return m if m.shape[1] == T else np.zeros((flat.n_series, T), dtype=np.uint32)


def expected(mats, series, groups, G: int, T: int, B: int, upto=None) -> np.ndarray:
    """[G, n_dist, T, B]: the histogram of the series matrices; replica i counts ticks < upto[i] (default: all)."""
    out = np.zeros((G, len(series), T, B), dtype=np.uint32)
    for i, (m, g) in enumerate(zip(mats, groups)):
        k = T if upto is None else min(int(upto[i]), T)
        for s, j in enumerate(series):
            out[g, s, np.arange(k), bins_of(m[j, :k], B)] += 1
    return out


def got(out, G: int, T: int) -> np.ndarray:
    return band_ref.dist_scan(out["dist_rows"], G, T)


def test_gauge_bin_mirror_matches_the_c_function():
    B = twin.gauge_bin(0xFFFFFFFF) + 1
    edges = gauge_bin_edges(B + 1)
    assert list(edges[:64]) == list(range(64)) and (np.diff(edges) > 0).all()
    assert (np.diff(edges)[64:] <= edges[64:-1] / 16).all()                   # at most 1/16 of the lower edge wide
    vals = np.unique(np.concatenate([np.arange(300), edges[:-1] - 1, edges[:-1], edges[:-1] + 1,
                                     np.random.default_rng(1).integers(0, 2 ** 32, 2000)]))
    vals = vals[(vals >= 0) & (vals < 2 ** 32)]
    want = np.array([twin.gauge_bin(int(v)) for v in vals])
    np.testing.assert_array_equal(bins_of(vals, B), want)


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_rows_equal_the_oracle_histogram(name, engine):
    payload = load_scenario(name, PARITY_CASES[name])
    flat = flatten(payload)
    n, begin = 4, 2
    groups = np.array([1, 0, 1, 0], dtype=np.uint32)
    series = [j for j in range(flat.n_series) if j % 2 == 0] or [0]
    run = twin.run_lane if engine == "lane" else twin.run_warp
    out = run(flat, seed=SEED, n=n, replica_begin=begin, series=series, groups=groups, n_groups=2, band_first=begin)
    assert (out["stats"]["flags"] & STOPS == 0).all()
    T, B = twin.ticks(flat), out["dist_rows"].shape[3]
    mats = [oracle_matrix(payload, flat, begin + i) for i in range(n)]
    np.testing.assert_array_equal(got(out, 2, T), expected(mats, series, groups, 2, T, B))


def _overloaded():
    payload = load_scenario("overload_single.yml")
    return payload, flatten(payload)


def test_a_stitched_replica_counts_once_and_equals_the_oracle():
    payload, flat = _overloaded()
    n, series = 6, [0, 1, 2]
    groups = np.array([0, 1, 2, 0, 1, 2], dtype=np.uint32)
    kw = dict(seed=SEED, n=n, series=series, groups=groups, n_groups=3, bin_capacity=16384)
    lane = twin.run_lane(flat, event_capacity=24, request_capacity=12, lane_bytes=520, **kw)
    flagged = np.flatnonzero(lane["stats"]["flags"] & STOPS)
    assert flagged.size >= 1 and all(0 < int(lane["band_from"][i]) < twin.ticks(flat) for i in flagged)
    out = twin.run_warp(flat, redo=flagged, into=lane, **kw)
    T, B = twin.ticks(flat), out["dist_rows"].shape[3]
    mats = [oracle_matrix(payload, flat, i) for i in range(n)]
    np.testing.assert_array_equal(got(out, 3, T), expected(mats, series, groups, 3, T, B))


def test_a_truncated_replica_contributes_its_ticks_before_the_stop_zeros_included():
    payload, flat = _overloaded()
    n, T = 6, twin.ticks(flat)
    series = [0, 1, 2]
    groups = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint32)
    out = twin.run_lane(flat, seed=SEED, n=n, series=series, groups=groups, n_groups=2, event_capacity=24,
                      request_capacity=12, lane_bytes=520)
    stopped = (out["stats"]["flags"] & STOPS) != 0
    assert stopped.any()
    upto = np.where(stopped, out["band_from"], T).astype(np.int64)
    B = out["dist_rows"].shape[3]
    mats = [oracle_matrix(payload, flat, i) for i in range(n)]
    g = got(out, 2, T)
    np.testing.assert_array_equal(g, expected(mats, series, groups, 2, T, B, upto))
    # a stopped replica holding 0 in some series leaves bin 0 at its stop tick (the v = 0 case band_stop skips)
    zero_at_stop = [i for i in np.flatnonzero(stopped) for j in series if mats[i][j, int(upto[i]) - 1] == 0]
    assert zero_at_stop, "no stopped replica holds a 0: the case is not exercised"
    assert (g.sum(axis=3)[:, :, -1] == np.bincount(groups[~stopped], minlength=2)[:, None]).all()


def test_cross_checks_with_the_sampled_bands():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    series = list(range(flat.n_series))
    groups = np.array([0, 1, 1, 0, 0], dtype=np.uint32)
    for run in (twin.run_lane, twin.run_warp):
        out = run(flat, seed=SEED, n=5, series=series, groups=groups, n_groups=2, sampled=True)
        T = twin.ticks(flat)
        d = got(out, 2, T)
        cnt, s, _ = band_ref.scan(flat, out["band_rows"], 2)
        np.testing.assert_array_equal(d.sum(axis=3), np.repeat(cnt[:, None, :], len(series), axis=1))
        edges = gauge_bin_edges(d.shape[3]).astype(np.uint64)
        small = d[..., 64:].sum(axis=-1) == 0
        assert small.any()
        np.testing.assert_array_equal((d.astype(np.uint64) * edges).sum(axis=-1)[small], s[small])


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("sampled,window", [(False, 0), (True, 0), (False, 3), (True, 3)])
def test_every_other_output_is_unchanged(sampled, window, lean):
    payload, flat = _overloaded()
    kw = dict(seed=SEED, n=5, replica_begin=1, groups=np.array([0, 1, 0, 1, 0], dtype=np.uint32), n_groups=2,
              band_first=1, event_capacity=24, request_capacity=12, lane_bytes=520, sampled=sampled, window=window,
              lean=lean)
    if not lean:
        kw.update(trace=3, clock_cap=5000)
    on = twin.run_lane(flat, series=[0, 2], **kw)
    off = twin.run_lane(flat, series=[], **kw)
    assert (on["stats"]["flags"] & STOPS).any() and on["dist_rows"].any()
    for k in (*twin.OUTPUTS, "band_rows", "band_from", "lat_rows", "lat_from"):
        if k == "band_from" and not sampled:
            continue                                        # (written by the distribution bands alone when on)
        assert on[k].tobytes() == off[k].tobytes(), k
    wkw = {k: v for k, v in kw.items() if k not in ("lane_bytes", "lean")}
    w_on, w_off = twin.run_warp(flat, series=[0, 2], **wkw), twin.run_warp(flat, series=[], **wkw)
    for k in (*twin.OUTPUTS, "band_rows", "lat_rows"):
        assert w_on[k].tobytes() == w_off[k].tobytes(), k


def test_lean_and_full_builds_give_the_same_rows():
    payload = load_scenario("c3_lb_two_servers.yml", 30)
    flat = flatten(payload)
    kw = dict(seed=SEED, n=6, series=[0, 3, 4], groups=np.array([0, 1, 2, 0, 1, 2], dtype=np.uint32), n_groups=3)
    a, b = twin.run_lane(flat, lean=True, **kw), twin.run_lane(flat, lean=False, **kw)
    assert a["dist_rows"].tobytes() == b["dist_rows"].tobytes()


def test_bad_series_and_oversized_rows_are_refused():
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    assert twin.dist_fits(flat, [0, 3], 10)[0]
    for bad, why in (([flat.n_series], "out of range"), ([-1], "out of range"), ([0, 0], "listed twice")):
        ok, _, _, msg = twin.dist_fits(flat, bad, 1)
        assert not ok and "distribution bands" in msg and why in msg
    ok, T, B, msg = twin.dist_fits(flat, list(range(flat.n_series)), 100_000, mem_total=80 << 30, request_capacity=(1 << 20) - 1)
    assert not ok and "GB of rows" in msg and "request capacity" in msg
    payload = load_scenario("c1_my_service.yml", 86_400)
    payload["sim_settings"]["sample_period_s"] = 0.001
    ok, _, _, msg = twin.dist_fits(flatten(payload), [0], 1)
    assert not ok and "ticks or more" in msg
    payload = load_scenario("c1_my_service.yml", 10)
    payload["sim_settings"]["enabled_sample_metrics"] = ["edge_concurrent_connection"]
    ok, _, _, msg = twin.dist_fits(flatten(payload), [0], 1)
    assert not ok and "not sampled" in msg


# ---- host side ----------------------------------------------------------------------------------------------------
def _results(values: np.ndarray, B: int) -> SweepResults:
    """SweepResults with one group whose replicas hold values[r, k] of ready_queue_len on server 0."""
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    S = flat.n_series
    res = SweepResults(flat, np.zeros(0, dtype=K.STATS_DTYPE), np.zeros((0, flat.n_edges)), np.zeros((0, flat.n_edges)),
                       np.zeros((0, S)), np.zeros((0, S)))
    R, T = values.shape
    h = np.zeros((1, 1, T, B), dtype=np.uint32)
    for k in range(T):
        np.add.at(h[0, 0, k], bins_of(values[:, k], B), 1)
    res.dist_series = [("ready_queue_len", flat.server_ids[0])]
    res.dist_hist = h
    return res


def test_group_dist_equals_numpy_on_the_values():
    rng = np.random.default_rng(7)
    B = twin.gauge_bin(1 << 20) + 1
    for R in (1, 2, 7, 20, 101):
        small = rng.integers(0, 64, (R, 9))
        big = rng.integers(0, 1 << 20, (R, 9))
        qs = (0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0)
        for vals in (small, big):
            res = _results(vals, B)
            d = res.group_dist("ready_queue_len", res.flat.server_ids[0], q=qs, at_least=4)
            lower = gauge_bin_edges(B)
            by_bin = lambda x: lower[bins_of(np.asarray(x), B)]   # noqa: E731
            want_q = np.stack([np.quantile(vals, q, axis=0, method="inverted_cdf") for q in qs])
            np.testing.assert_array_equal(d["q"][0], by_bin(want_q))
            np.testing.assert_array_equal(d["min"][0], by_bin(vals.min(axis=0)))
            np.testing.assert_array_equal(d["max"][0], by_bin(vals.max(axis=0)))
            np.testing.assert_array_equal(d["p_at_least"][0], (vals >= 4).mean(axis=0))
            np.testing.assert_array_equal(d["n"][0], np.full(9, R))
            if vals is small:
                np.testing.assert_array_equal(d["q"][0], want_q)
    res = _results(small, B)
    edge = int(gauge_bin_edges(80)[70])
    assert np.isfinite(res.group_dist("ready_queue_len", res.flat.server_ids[0], at_least=edge)["p_at_least"]).all()
    with pytest.raises(ValueError, match=f"{edge} and {int(gauge_bin_edges(80)[71])}"):
        res.group_dist("ready_queue_len", res.flat.server_ids[0], at_least=edge + 1)


def test_group_dist_is_nan_where_no_replica_contributes():
    res = _results(np.array([[1, 2, 3]]), 70)
    res.dist_hist[0, 0, 2] = 0
    d = res.group_dist("ready_queue_len", res.flat.server_ids[0], at_least=2)
    assert np.isnan(d["q"][0, :, 2]).all() and np.isnan(d["min"][0, 2]) and np.isnan(d["p_at_least"][0, 2])
    assert d["max"][0, 1] == 2 and d["n"][0, 2] == 0


def test_concatenate_and_take_carry_the_rows():
    a, b = _results(np.array([[1, 2], [3, 4]]), 70), _results(np.array([[5, 6]]), 70)
    c = SweepResults.concatenate([a, b])
    np.testing.assert_array_equal(c.dist_hist, a.dist_hist + b.dist_hist)
    assert c.dist_series == a.dist_series and c.take(np.arange(0)).dist_hist is c.dist_hist
    assert "dist_hist" in BAND_FIELDS


def test_shards_with_different_swept_ram_size_their_bins_differently():
    """A launch sizes its bins by its own rows' largest ram_mb: two shards of one sweep can differ in bin count."""
    from asyncflow_b200 import SweepSpec
    flat = flatten(load_scenario("c3_lb_two_servers.yml", 30))
    ram = [4096.0, 8192.0, 65536.0, 131072.0]
    col = ("server_ram_mb", flat.server_ids[0])
    bins = [twin.dist_fits(flat, [2], 2, request_capacity=16384, sweep=SweepSpec(flat, len(v), {col: v}))[2]
            for v in (ram[:2], ram[2:], ram)]
    assert bins[0] < bins[1] == bins[2]


def test_concatenate_pads_shards_with_fewer_bins_and_checks_the_series():
    a, b = _results(np.array([[1, 2], [70, 4]]), 80), _results(np.array([[5, 200]]), 120)
    c = SweepResults.concatenate([a, b])
    assert c.dist_hist.shape[-1] == 120 and c.dist_hist[..., 80:].sum() == b.dist_hist[..., 80:].sum()
    whole = _results(np.array([[1, 2], [70, 4], [5, 200]]), 120)
    np.testing.assert_array_equal(c.dist_hist, whole.dist_hist)
    d = c.group_dist("ready_queue_len", c.flat.server_ids[0], q=(0.5,))
    np.testing.assert_array_equal(d["max"][0], gauge_bin_edges(120)[[twin.gauge_bin(70), twin.gauge_bin(200)]])
    b.dist_series = [("ready_queue_len", b.flat.server_ids[-1] + "-other")]
    with pytest.raises(ValueError, match="different series"):
        SweepResults.concatenate([a, b])


def _gloo_worker(rank, port, q):
    import torch.distributed as dist

    from asyncflow_b200.distributed import all_reduce_bands
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=2)
    try:
        r = all_reduce_bands(_gloo_part(rank))
        q.put((rank, (r.dist_hist, r.group_size)))
    finally:
        dist.destroy_process_group()


def _gloo_part(rank: int) -> SweepResults:
    """Rank 0's shard sees values below 64 only (fewer bins), rank 1's up to 5 000 (more bins); both carry group sizes."""
    rng = np.random.default_rng(3 + rank)
    vals = rng.integers(0, 64 if rank == 0 else 5000, (7, 4))
    r = _results(vals, twin.gauge_bin(int(vals.max())) + 1 + 3 * rank)
    r.group_size = rng.integers(0, 1000, size=1).astype(np.int64)
    return r


def test_all_reduce_bands_pads_and_sums_the_distribution_rows_on_gloo():
    import socket

    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = SweepResults.concatenate([_gloo_part(r) for r in range(2)])
    assert _gloo_part(0).dist_hist.shape[-1] < want.dist_hist.shape[-1]
    for rank in (0, 1):
        hist, size = got[rank]
        assert hist.dtype == np.uint32 and np.array_equal(hist, want.dist_hist), rank
        assert np.array_equal(size, want.group_size), rank


def test_sweep_runner_needs_groups_for_dist_series():
    from asyncflow_b200 import SweepRunner
    payload = load_scenario("c1_my_service.yml", 5)
    flat = flatten(payload)
    with pytest.raises(ValueError, match="needs groups"):
        SweepRunner(payload, 2, dist_series=[("ready_queue_len", flat.server_ids[0])], pinned=False)
