"""CPU tier: occupancy integrals (af_occupancy_configure / af_fetch_occupancy).  Both state machines, driven by
the CPU twin (tests/twin.py), must give per replica and column exactly the sum of delta x fixed(H - t) over the
oracle's own ledger of the same state changes; that sum must lie within the rounding bound of the exact rational
integral, telescope to the requests' own start / end times, and leave every other output unchanged; and the host side
must read request-seconds, time averages and breakdowns off the rows."""

from __future__ import annotations

from fractions import Fraction

import band_ref
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario

from asyncflow_b200 import SweepRunner, SweepSpec, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.results import GAUGE_STATE, SweepResults, occ_frac_bits, occupancy_columns

STOPS = K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW
F = 32


def _case(name: str):
    payload = load_scenario(name, PARITY_CASES[name])
    return payload, flatten(payload)


def test_fixed_point_is_round_to_nearest_even_on_both_sides():
    rng = np.random.default_rng(5)
    rests = [0.0, 0.5, 1.5, 2.5, 3.0, 1e-9, 0.1, 59.999999, 3600.0] + list(rng.uniform(0, 4000, 200))
    for f in (8, 20, 27, 32):
        for r in rests:
            assert twin.occ_fixed(r, f) == band_ref.fixed(r, f), (r, f)
    assert band_ref.fixed(2.5, 0) == 2 and band_ref.fixed(3.5, 0) == 4                       # ties to even


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_rows_equal_the_oracle_ledger_and_telescope(name):
    payload, flat = _case(name)
    H, n, begin = flat.horizon_s, 2, 1
    lane = twin.run_lane(flat, seed=SEED, n=n, replica_begin=begin, f=F)
    warp = twin.run_warp(flat, seed=SEED, n=n, replica_begin=begin, f=F)
    assert (lane["stats"]["flags"] & STOPS == 0).all() and (warp["stats"]["flags"] & STOPS == 0).all()
    C = twin.occ_cols(flat)
    ram_mb = [5 * s + 4 for s in range(flat.n_servers)]
    for i in range(n):
        o, ledger, reqs = band_ref.oracle_ledger(payload, flat, seed=SEED, replica=begin + i)
        assert len(reqs) == o["generated"] == int(lane["stats"]["generated"][i])
        want = band_ref.ledger_rows(ledger, C, float(H), F)
        assert lane["occ"][i].tobytes() == want.tobytes(), name
        assert warp["occ"][i].tobytes() == want.tobytes(), name
        # within (unit changes / 2) x 2^-f of the exact integral of the oracle's f64 clocks
        for c in range(C):
            entries = [(t, d) for t, cc, d in ledger if cc == c]
            exact = sum((d * (Fraction(H) - Fraction(t)) for t, d in entries), Fraction(0)) * 2 ** F
            assert abs(Fraction(int(want[c])) - exact) <= Fraction(sum(abs(d) for _, d in entries), 2), (name, c)
        # every non-zero-time stretch of a request's life is in exactly one column (RAM MB aside)
        tele = 0
        for start, end in reqs:
            tele += band_ref.fixed(H - start, F) - (0 if end is None else band_ref.fixed(H - end, F))
        total = sum(int(want[c]) for c in range(C) if c not in ram_mb)
        assert total & band_ref.MASK64 == tele & band_ref.MASK64, name


def test_every_state_is_exercised_and_requests_drop_and_stay_in_flight():
    seen = set()
    dropped = in_flight = False
    for name in sorted(PARITY_CASES):
        payload, flat = _case(name)
        out = twin.run_lane(flat, seed=SEED, n=2, f=F)
        for (_, state), v in zip(occupancy_columns(flat), out["occ"].any(axis=0)):
            if v:
                seen.add(state)
        dropped |= bool(out["dropped"].any())
        st = out["stats"]
        in_flight |= bool((st["generated"] > st["completed"] + out["dropped"].sum(axis=1)).any())
    assert seen == {"ram_wait", "cpu_wait", "cpu", "io", "ram_mb", "transit"}, seen
    assert dropped and in_flight


def test_lean_and_full_builds_give_the_same_rows():
    _, flat = _case("c3_lb_two_servers.yml")
    a = twin.run_lane(flat, seed=SEED, n=6, f=F, lean=True)
    b = twin.run_lane(flat, seed=SEED, n=6, f=F, lean=False)
    assert a["occ"].any() and a["occ"].tobytes() == b["occ"].tobytes()


def _overloaded():
    payload = load_scenario("overload_single.yml")
    return payload, flatten(payload)


BAND_KINDS = [dict(), dict(sampled=True), dict(window=3), dict(series=[0, 2]),
              dict(sampled=True, window=3, series=[0, 1, 2])]


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("bands", BAND_KINDS, ids=lambda b: "+".join(sorted(b)) or "none")
def test_every_other_output_is_unchanged(bands, lean):
    _, flat = _overloaded()
    kw = dict(seed=SEED, n=5, replica_begin=1, groups=np.array([0, 1, 0, 1, 0], dtype=np.uint32), n_groups=2,
              band_first=1, event_capacity=24, request_capacity=12, **bands)
    if not lean:
        kw.update(trace=3, clock_cap=5000)
    on = twin.run_lane(flat, f=F, lean=lean, lane_bytes=520, **kw)
    off = twin.run_lane(flat, f=0, lean=lean, lane_bytes=520, **kw)
    assert (on["stats"]["flags"] & STOPS).any() and on["occ"].any() and not off["occ"].any()
    for k in (*twin.OUTPUTS, "band_rows", "band_from", "lat_rows", "lat_from", "dist_rows"):
        assert on[k].tobytes() == off[k].tobytes(), k
    w_on, w_off = twin.run_warp(flat, f=F, **kw), twin.run_warp(flat, f=0, **kw)
    assert w_on["occ"].any()
    for k in (*twin.OUTPUTS, "band_rows", "lat_rows", "dist_rows"):
        assert w_on[k].tobytes() == w_off[k].tobytes(), k


def test_a_stitched_replica_equals_a_first_hand_warp_run():
    payload, flat = _overloaded()
    n = 6
    kw = dict(seed=SEED, n=n, f=F, groups=np.zeros(n, dtype=np.uint32), n_groups=1, sampled=True, window=2)
    lane = twin.run_lane(flat, event_capacity=24, request_capacity=12, lane_bytes=520, **kw)
    flagged = np.flatnonzero(lane["stats"]["flags"] & STOPS)
    assert flagged.size >= 1
    partial = lane["occ"].copy()
    out = twin.run_warp(flat, redo=flagged, into=lane, **kw)
    first = twin.run_warp(flat, **kw)
    assert out["occ"].tobytes() == first["occ"].tobytes()
    assert (out["occ"][flagged] != partial[flagged]).any()
    for i in flagged[:2]:
        _, ledger, _ = band_ref.oracle_ledger(payload, flat, seed=SEED, replica=int(i))
        assert out["occ"][i].tobytes() == band_ref.ledger_rows(ledger, twin.occ_cols(flat), float(flat.horizon_s), F).tobytes()


def test_the_bound_check_and_the_choice_of_f():
    payload = load_scenario("c1_my_service.yml", 86_400)
    flat = flatten(payload)
    H, rq = flat.horizon_s, (1 << 20) - 1
    f = twin.frac_bits(rq, H)
    assert f == occ_frac_bits(rq, H) == 27
    assert twin.occ_fits(flat, f, request_capacity=rq)[0]
    ok, why = twin.occ_fits(flat, f + 1, request_capacity=rq)
    assert not ok and f"B = {rq}" in why and f"H = {H} s" in why and f"f = {f + 1}" in why and f"f <= {f}" in why
    assert "request capacity" in why
    ok, why = twin.occ_fits(flatten(load_scenario("c1_my_service.yml", 10)), 7)
    assert not ok and "7 fraction bits" in why
    # swept RAM above the request capacity sets the bound
    col = ("server_ram_mb", flat.server_ids[0])
    sweep = SweepSpec(flat, 2, {col: [4096.0, float(1 << 24)]})
    ok, why = twin.occ_fits(flat, twin.frac_bits(rq, H), request_capacity=rq, sweep=sweep)
    assert not ok and "swept ram_mb 16777216" in why
    assert twin.occ_fits(flat, twin.frac_bits(1 << 24, H), request_capacity=rq, sweep=sweep)[0]
    # the edge of fitting: B x H x 2^f <= 2^64 - 1, in C and in Python
    for h in (1, 60, 3600, 86_400, 1 << 30):
        for f in (8, 20, 31, 32):
            b = ((1 << 64) - 1) // (h << f)
            for bb, want in ((b, f), (b + 1, f - 1)):
                got = twin.frac_bits(bb, h)
                assert got == occ_frac_bits(bb, h), (bb, h)
                if f < 32:
                    assert got == want, (bb, h, f)
                else:
                    assert got == (32 if bb == b else min(32, want)), (bb, h)
    assert twin.frac_bits(1 << 40, 1 << 30) == occ_frac_bits(1 << 40, 1 << 30) == -1


def test_sweep_runner_picks_one_scale_for_the_whole_sweep():
    payload = load_scenario("c1_my_service.yml", 86_400)
    flat = flatten(payload)
    r = SweepRunner(payload, 4, occupancy=True, pinned=False)
    assert r.occ_frac_bits == twin.frac_bits((1 << 20) - 1, 86_400)
    col = ("server_ram_mb", flat.server_ids[0])
    r = SweepRunner(payload, 4, {col: [1024, 2048, 1 << 26, 4096]}, occupancy=True, pinned=False)
    assert r.occ_frac_bits == twin.frac_bits(1 << 26, 86_400) < 27
    payload = load_scenario("c1_my_service.yml", 1 << 30)
    with pytest.raises(ValueError, match="fraction bits"):
        SweepRunner(payload, 2, {col: [1024, (1 << 31) - 1]}, occupancy=True, pinned=False)
    assert SweepRunner(load_scenario("c1_my_service.yml", 5), 2, pinned=False).occ_frac_bits == 0


# ---- host side ----------------------------------------------------------------------------------------------------
def _results(flat, out: dict, f: int) -> SweepResults:
    res = SweepResults(flat, out["stats"], out["sent"], out["dropped"], out["samp_sum"], out["samp_max"])
    res.occupancy, res.occ_frac_bits = out["occ"], f
    return res


def test_time_in_time_average_and_breakdown():
    payload, flat = _case("c3_lb_two_servers.yml")
    out = twin.run_lane(flat, seed=SEED, n=4, f=F)
    res = _results(flat, out, F)
    H = float(flat.horizon_s)
    assert res.occ_columns == occupancy_columns(flat) and len(res.occ_columns) == twin.occ_cols(flat)
    s0, e0 = flat.server_ids[0], flat.edge_ids[0]
    for j, (ent, st) in enumerate(res.occ_columns):
        np.testing.assert_array_equal(res.time_in(st, ent), out["occ"][:, j].astype(np.float64) / 2.0 ** F)
    for key, st in GAUGE_STATE.items():
        ent = e0 if st == "transit" else s0
        np.testing.assert_array_equal(res.time_average(key, ent), res.time_in(st, ent) / H)
    # the exact time average is close to the tick-sampled mean of the same gauge (100 Hz ticks here)
    j = res.series_index("ready_queue_len", s0)
    assert np.allclose(res.time_average("ready_queue_len", s0), res.sampled_mean()[:, j], rtol=0.1, atol=0.05)
    sel = np.array([0, 2])
    b = res.breakdown(sel)
    raw = [sum(int(v) for v in out["occ"][sel, j]) for j in range(twin.occ_cols(flat))]
    assert b["raw"] == raw and b["entity"][0] == s0 and b["state"][:5] == ["ram_wait", "cpu_wait", "cpu", "io", "ram_mb"]
    np.testing.assert_array_equal(b["seconds"], np.array([x / 2 ** F for x in raw]))
    req = np.array([st != "ram_mb" for st in b["state"]])
    assert np.isnan(b["share"][~req]).all() and abs(np.nansum(b["share"]) - 1.0) < 1e-12
    gen = float(out["stats"]["generated"][sel].sum())
    np.testing.assert_allclose(b["per_request"], b["seconds"] / gen, rtol=0, atol=0)
    with pytest.raises(KeyError):
        res.time_in("cpu", e0)
    with pytest.raises(ValueError, match="occupancy=True"):
        SweepResults(flat, out["stats"], out["sent"], out["dropped"], out["samp_sum"], out["samp_max"]).time_in("cpu", s0)


def test_breakdown_sums_exactly_beyond_2_64():
    _, flat = _case("c1_my_service.yml")
    occ = np.full((5, twin.occ_cols(flat)), (1 << 64) - 1, dtype=np.uint64)
    stats = np.zeros(5, dtype=K.STATS_DTYPE)
    stats["generated"] = 1
    res = SweepResults(flat, stats, np.zeros((5, flat.n_edges)), np.zeros((5, flat.n_edges)),
                       np.zeros((5, flat.n_series)), np.zeros((5, flat.n_series)))
    res.occupancy, res.occ_frac_bits = occ, 8
    assert res.breakdown()["raw"][0] == 5 * ((1 << 64) - 1)


def test_take_and_concatenate_carry_the_rows():
    _, flat = _case("c1_my_service.yml")
    a = _results(flat, twin.run_lane(flat, seed=SEED, n=3, f=F), F)
    b = _results(flat, twin.run_lane(flat, seed=SEED, n=2, replica_begin=3, f=F), F)
    c = SweepResults.concatenate([a, b])
    whole = twin.run_lane(flat, seed=SEED, n=5, f=F)
    assert c.occupancy.tobytes() == whole["occ"].tobytes() and c.occ_frac_bits == F
    t = c.take(np.array([4, 0]))
    np.testing.assert_array_equal(t.occupancy, whole["occ"][[4, 0]])
    assert t.occ_frac_bits == F
    b.occ_frac_bits = F - 1
    with pytest.raises(ValueError, match="different fixed-point scales"):
        SweepResults.concatenate([a, b])
