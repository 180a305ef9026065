"""CPU tier: per-window latency bands, through the CPU twin of both engines (tests/twin.py).

The rows equal the oracle's clocks binned by finish window and latency bin, fixed-point sums included, in both state
machines; a replica the thread-per-replica pass stops and the warp-per-replica pass re-runs from ``lat_from`` counts
once, in full, even when the flag was raised in an iteration that completed requests after it; a replica that stays
stopped contributes exactly its completions before the stop; no other output changes; the window and row-size checks
refuse what they should; the shared percentile helper keeps ``GlobalSummary``'s numbers; and ``all_reduce_bands``
sums shards as ``concatenate`` does."""

from __future__ import annotations

import math
import socket

import band_ref
import des_port
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario

from asyncflow_b200 import SweepResults, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.results import hist_percentiles

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW | K.FLAG_LB_EMPTY
REDO = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW      # what af_run's second pass re-runs


def oracle_clocks(payload, replica: int, seed: int = SEED) -> np.ndarray:
    return np.asarray(des_port.simulate(payload, seed=seed, replica=replica)["clocks"], dtype=np.float64).reshape(-1, 2)


def expected(flat, clocks: list[np.ndarray], groups, n_groups: int, w: int, upto=None) -> np.ndarray:
    rows = twin.lat_rows(flat, n_groups, w)
    for i, (c, g) in enumerate(zip(clocks, groups)):
        band_ref.bin_clocks(rows, int(g), c if upto is None else c[:int(upto[i])], w, int(flat.horizon_s))
    return rows


def assert_rows(got: np.ndarray, want: np.ndarray, n_groups: int) -> None:
    assert got.dtype == want.dtype == np.uint64
    assert np.array_equal(got[:n_groups], want[:n_groups])


def _widths(horizon: int) -> list[int]:
    d = next((k for k in (5, 4, 3, 2) if horizon % k == 0 and k < horizon), 1)
    nd = next(k for k in (7, 3, 4, 6, 11) if horizon % k != 0)
    return [1, d, nd]


def test_fixed_point_and_bins_match_the_python_definition():
    rng = np.random.default_rng(1)
    lats = np.concatenate([rng.exponential(0.05, 2000), [0.0, 2.0 ** -33, 3 * 2.0 ** -33, 1.0, 4096.5, 1e-9]])
    for lat in lats:
        assert twin.lib().af_twin_fixed32(float(lat)) == round(float(lat) * 4294967296.0)
        assert twin.lib().af_twin_hist_bin(float(lat)) == band_ref.hist_bin(float(lat))


@pytest.mark.parametrize("engine", ["lane", "warp"])
@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_latency_rows_equal_the_oracle_clocks_binned(name, engine):
    payload = load_scenario(name, PARITY_CASES[name])
    flat = flatten(payload)
    n, begin = 4, 2
    groups = np.array([1, 0, 1, 0], dtype=np.uint32)
    clocks = [oracle_clocks(payload, begin + i) for i in range(n)]
    run = twin.run_lane if engine == "lane" else twin.run_warp
    for w in _widths(int(flat.horizon_s)):
        out = run(flat, seed=SEED, n=n, replica_begin=begin, groups=groups, n_groups=2, band_first=begin, window=w)
        assert (out["stats"]["flags"] & STOPS == 0).all()
        assert sum(len(c) for c in clocks) == int(out["stats"]["completed"].sum())
        assert_rows(out["lat_rows"], expected(flat, clocks, groups, 2, w), 2)


def _overloaded():
    payload = load_scenario("overload_single.yml")
    return payload, flatten(payload)


# Small event pools: the generator phase of an iteration raises the event-overflow flag, and the event the same
# iteration then pops can complete a request (replica 23 of these 24 does).
SMALL = dict(event_capacity=12, request_capacity=64, lane_bytes=1816)
N_SMALL = 24


def test_flagged_replicas_rerun_from_lat_from_give_the_first_hand_rows():
    payload, flat = _overloaded()
    n, seed = N_SMALL, SEED
    groups = (np.arange(n) % 3).astype(np.uint32)
    for w in (1, 7):
        lane = twin.run_lane(flat, seed=seed, n=n, groups=groups, n_groups=3, window=w, sampled=True, **SMALL)
        st = lane["stats"]
        flagged = np.flatnonzero(st["flags"] & REDO)
        assert flagged.size >= 1
        assert ((lane["lat_from"][flagged] < st["completed"][flagged])).any(), "no completion after a flag"
        out = twin.run_warp(flat, seed=seed, n=n, groups=groups, n_groups=3, window=w, sampled=True, redo=flagged, into=lane)
        assert (out["stats"]["flags"] & STOPS == 0).all()
        full = twin.run_warp(flat, seed=seed, n=n, groups=groups, n_groups=3, window=w, sampled=True)
        assert_rows(out["lat_rows"], full["lat_rows"], 3)
        assert np.array_equal(band_ref.scan(flat, out["band_rows"], 3)[1], band_ref.scan(flat, full["band_rows"], 3)[1])
        clocks = [oracle_clocks(payload, i, seed) for i in range(n)]
        assert_rows(out["lat_rows"], expected(flat, clocks, groups, 3, w), 3)


def test_a_stopped_replica_contributes_exactly_its_completions_before_the_stop():
    payload, flat = _overloaded()
    n, seed = N_SMALL, SEED
    groups = (np.arange(n) // 12).astype(np.uint32)
    out = twin.run_lane(flat, seed=seed, n=n, groups=groups, n_groups=2, window=1, **SMALL)
    st = out["stats"]
    stopped = (st["flags"] & STOPS) != 0
    assert stopped.any()
    upto = np.where(stopped, out["lat_from"], st["completed"]).astype(np.int64)
    assert (upto <= st["completed"]).all() and (upto[stopped] < st["completed"][stopped]).any()
    clocks = [oracle_clocks(payload, i, seed) for i in range(n)]
    assert all(len(c) >= u for c, u in zip(clocks, upto))
    assert_rows(out["lat_rows"], expected(flat, clocks, groups, 2, 1, upto), 2)


@pytest.mark.parametrize("engine", ["lane", "warp"])
def test_latency_bands_change_no_other_output(engine):
    payload, flat = _overloaded()
    run = twin.run_lane if engine == "lane" else twin.run_warp
    kw = dict(seed=SEED, n=5, replica_begin=1, groups=np.array([0, 1, 0, 1, 0], dtype=np.uint32), n_groups=2,
              band_first=1, trace=3, clock_cap=5000, event_capacity=24, request_capacity=12)
    if engine == "lane":
        kw["lane_bytes"] = 520
    off = run(flat, window=0, **kw)
    for sampled in (False, True):
        on = run(flat, window=3, sampled=sampled, **kw)
        assert (on["stats"]["flags"] & STOPS).any()
        for k in twin.OUTPUTS:
            assert on[k].tobytes() == off[k].tobytes(), k
        assert on["lat_rows"].any() and not off["lat_rows"].any()
        if sampled:       # and the per-tick bands are those of a run without latency bands
            ref = run(flat, window=0, sampled=True, **kw)
            assert on["band_rows"].tobytes() == ref["band_rows"].tobytes()


def test_window_and_row_size_checks():
    ok, why = twin.lat_fits(0, 60, 4, 1 << 40)
    assert not ok and "window of 0 s" in why
    ok, why = twin.lat_fits(-3, 60, 4, 1 << 40)
    assert not ok and "window of -3 s" in why
    assert twin.lat_fits(1, 60, 1000, 80 << 30)[0]             # 1 001 x 60 x 4 098 x 8 B = 1.97 GB
    ok, why = twin.lat_fits(1, 60, 1000, 1 << 30)
    assert not ok and "1000 groups x 60 windows of 1 s need 1.97 GB of rows, more than the device's 1.07 GB" in why
    ok, why = twin.lat_fits(1, 86_400, 1_000_000, 80 << 30)
    assert not ok and "86400 windows" in why
    assert twin.lat_fits(7, 60, 3, 2 << 20)[0]                  # 4 x 9 windows x 4 098 x 8 B = 1.18 MB


def _old_global_percentile(histogram: np.ndarray, q: float) -> float:
    """GlobalSummary.percentile as it was before it called hist_percentiles."""
    n = int(histogram.sum())
    if n == 0:
        return float("nan")
    cum = np.cumsum(histogram)
    base = (1023 + K.AF_HIST_MIN_EXP) << K.AF_HIST_SUB_BITS

    def order_stat(rank: int) -> float:
        b = int(np.searchsorted(cum, rank, side="right"))
        before = int(cum[b - 1]) if b else 0
        lo, hi = (np.array([(b + base) << (52 - K.AF_HIST_SUB_BITS),
                            (b + 1 + base) << (52 - K.AF_HIST_SUB_BITS)], dtype=np.uint64).view(np.float64))
        frac = ((rank - before) + 0.5) / float(histogram[b])
        return float(lo + frac * (hi - lo))

    pos = q / 100.0 * (n - 1)
    lo = int(np.floor(pos))
    frac = pos - lo
    a = order_stat(lo)
    return a if frac == 0.0 or lo + 1 >= n else a + frac * (order_stat(lo + 1) - a)


def test_percentile_helper_equals_the_global_summary_arithmetic():
    from asyncflow_b200.distributed import GlobalSummary
    rng = np.random.default_rng(7)
    hs = np.zeros((40, K.AF_HIST_BINS), dtype=np.int64)
    for i in range(40):
        k = int(rng.integers(0, 6))
        if k:
            idx = rng.integers(2000, 2600, size=k * 50)
            np.add.at(hs[i], idx, rng.integers(1, 4, size=idx.size))
    hs[3] = 0
    hs[5, 2222] = 1
    for q in (0.0, 50.0, 95.0, 99.0, 100.0, 37.3):
        got = hist_percentiles(hs, q)
        for i in range(40):
            want = _old_global_percentile(hs[i], q)
            assert (math.isnan(want) and math.isnan(got[i])) or got[i] == want, (i, q)
            gs = GlobalSummary(hs[i], 0, 0, 0, 0, 0, 0.0, 0.0, 0.0, [])
            g = gs.percentile(q)
            assert (math.isnan(want) and math.isnan(g)) or g == want


def _results(rng, G=3, W=5, S=2, T=6) -> SweepResults:
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    n = 1
    r = SweepResults(flat, np.zeros(n, dtype=K.STATS_DTYPE), np.zeros((n, flat.n_edges), np.uint32),
                     np.zeros((n, flat.n_edges), np.uint32), np.zeros((n, flat.n_series), np.uint64),
                     np.zeros((n, flat.n_series), np.uint32))
    u64 = lambda *s: rng.integers(0, 2 ** 63, size=s, dtype=np.uint64) * np.uint64(2) + np.uint64(1)  # noqa: E731
    r.band_count = rng.integers(0, 2 ** 32, size=(G, T), dtype=np.uint32)
    r.band_sum, r.band_sumsq = u64(G, S, T), u64(G, S, T)
    r.lat_window_s = 1
    r.lat_hist = u64(G, W, K.AF_HIST_BINS)
    r.lat_sum_hi, r.lat_sum_lo = u64(G, W), u64(G, W)
    r.group_size = rng.integers(0, 1000, size=G).astype(np.int64)
    return r


def _gloo_worker(rank, port, parts_seed, q):
    import torch.distributed as dist
    from asyncflow_b200.distributed import all_reduce_bands
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=2)
    try:
        r = all_reduce_bands(_results(np.random.default_rng(parts_seed + rank)))
        q.put((rank, {k: getattr(r, k) for k in ("band_count", "band_sum", "band_sumsq", "lat_hist", "lat_sum_hi",
                                                   "lat_sum_lo", "group_size")}))
    finally:
        dist.destroy_process_group()


def test_all_reduce_bands_equals_concatenate_on_gloo():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, port, 11, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = SweepResults.concatenate([_results(np.random.default_rng(11 + r)) for r in range(2)])
    for rank in (0, 1):
        for k, v in got[rank].items():
            w = getattr(want, k)
            assert v.dtype == w.dtype and np.array_equal(v, w), (rank, k)


def test_group_latency_statistics():
    rng = np.random.default_rng(3)
    flat = flatten(load_scenario("c1_my_service.yml", 5))
    r = SweepResults(flat, np.zeros(1, dtype=K.STATS_DTYPE), np.zeros((1, flat.n_edges), np.uint32),
                     np.zeros((1, flat.n_edges), np.uint32), np.zeros((1, flat.n_series), np.uint64),
                     np.zeros((1, flat.n_series), np.uint32))
    lats = [rng.exponential(0.02, 500) + 0.001 for _ in range(4)]                 # group g, windows of 2 s over 5 s
    fins = [rng.uniform(0.0, 5.0, 500) for _ in range(4)]
    rows = np.zeros((2, 3, twin.LAT_ROW), dtype=np.uint64)
    for g in range(2):
        for j in (2 * g, 2 * g + 1):
            band_ref.bin_clocks(rows, g, np.stack([fins[j] - lats[j], fins[j]], axis=1), 2, 5)
    r.lat_window_s, r.group_size = 2, np.array([2, 2])
    r.lat_hist, r.lat_sum_hi, r.lat_sum_lo = rows[:, :, :K.AF_HIST_BINS], rows[:, :, -2], rows[:, :, -1]
    out = r.group_latency()
    assert np.array_equal(out["t"], [2.0, 4.0, 5.0])
    for g in range(2):
        lat = np.concatenate([lats[2 * g], lats[2 * g + 1]])
        fin = np.concatenate([fins[2 * g], fins[2 * g + 1]])
        lat = np.concatenate([fins[2 * g], fins[2 * g + 1]]) - (fin - lat)            # the latencies as binned
        k = (np.maximum(np.ceil(fin) - 1, 0) // 2).astype(int)
        for w in range(3):
            sel = lat[k == w]
            assert out["n"][g, w] == sel.size
            assert abs(out["mean"][g, w] - sel.mean()) <= 2.0 ** -30
            assert out["rps"][g, w] == sel.size / ((2.0 if w < 2 else 1.0) * 2)
            assert abs(out["p95"][g, w] / np.percentile(sel, 95) - 1) < 0.01
        assert out["total"]["n"][g] == lat.size and abs(out["total"]["mean"][g] - lat.mean()) <= 2.0 ** -30
        assert out["total"]["rps"][g] == lat.size / (5.0 * 2)

