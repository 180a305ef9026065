"""CPU tier: the inputs and references tests/test_gpu_fuzz.py relies on, checked without a device, so that a failure
there points at the device and not at the reference.

The random sweeps cover every sweep field, the aliased launches share a slot between columns whose bases differ, the
warp-engine seeds reach multi-slot pools and simultaneous finishes, the big topologies reach the global tiers, the
stitched case has replicas the lane pass stops, and every occupancy state is non-zero; and the twin equals the oracle on
the replicas the GPU file compares with the oracle that the CPU tier does not already cover (sweep replicas from row
1000 on, replicas past a sweep's last row, the accumulating outputs' own groups)."""

from __future__ import annotations

import des_port
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, assert_matches_oracle
from test_gpu_fuzz import (ALIAS_SEEDS, BIG_SEEDS, CAPS, COVER, G, MULTI_SLOT_SHARE, N_ACC, OWN, STITCH_SEED,
                           SWEEP_SEEDS, TIE_SEEDS, TRACE, WARP_EV_SMEM, WARP_RQ_SMEM, WARP_SEEDS, acc_case, acc_groups,
                           acc_twin, added_alias_shares_a_slot, assert_own_groups_equal_oracle, big_reference,
                           occ_bits, stitched_replicas, sweep_case, swept_fields, twin_views, warp_seed_coverage,
                           warp_seed_reference)
from test_gpu_multiwave import BEGIN, twin_run

from asyncflow_b200 import _capi as K
from asyncflow_b200 import flatten
from asyncflow_b200.results import occupancy_columns

#: the launch size of the GPU file's sweep and alias cases on a 132-SM H100 (4 x SMs + 7)
N_H100 = 4 * 132 + 7


def test_the_sweeps_cover_every_field_and_aliased_columns_with_different_bases():
    assert swept_fields(SWEEP_SEEDS) == set(K.FIELDS), set(K.FIELDS) - swept_fields(SWEEP_SEEDS)
    assert all(added_alias_shares_a_slot(seed, N_H100 // 2) for seed in ALIAS_SEEDS)


def test_the_warp_seeds_reach_multi_slot_pools_and_ties():
    share, ties = warp_seed_coverage([(s, warp_seed_reference(s, COVER)[2]) for s in WARP_SEEDS])
    assert share >= MULTI_SLOT_SHARE and ties >= TIE_SEEDS, (share, ties)


@pytest.mark.parametrize("seed", BIG_SEEDS)
def test_big_topologies_reach_the_warp_engines_global_tiers(seed):
    st = big_reference(seed, 48)[2]["stats"]
    assert (st["peak_events"] > WARP_EV_SMEM).any() and (st["peak_requests"] > WARP_RQ_SMEM).any()


def test_the_stitched_case_has_replicas_the_lane_pass_stops():
    _, flat, spec = sweep_case(STITCH_SEED, COVER)
    assert stitched_replicas(flat, spec, COVER).size >= 1


def test_every_occupancy_state_is_nonzero_in_the_twin():
    seen = set()
    for case in sorted(PARITY_CASES) + [f"sweep-{s}" for s in SWEEP_SEEDS[:6]]:
        _, flat, spec = acc_case(case)
        f = occ_bits(flat, spec, CAPS["request_capacity"])
        occ = acc_twin(flat, spec, N_ACC, acc_groups(N_ACC), f, CAPS)["occ"]
        seen |= {st for (_, st), v in zip(occupancy_columns(flat), occ.any(axis=0)) if v}
    assert seen == {"ram_wait", "cpu_wait", "cpu", "io", "ram_mb", "transit"}, seen


@pytest.mark.parametrize("seed", SWEEP_SEEDS)
def test_twin_equals_oracle_on_the_traced_sweep_replicas(seed):
    payload, _, spec = sweep_case(seed, TRACE)
    r = twin_run(flatten(payload), TRACE, sweep=spec, trace=TRACE, clock_cap=100_000, **CAPS)
    for i in range(TRACE):
        p = spec.payload_for(payload, BEGIN + i)
        st = r["stats"][i]
        k, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0
        assert_matches_oracle(des_port.simulate(p, seed=SEED, replica=BEGIN + i), flatten(p), stats=st,
                              clocks=r["trace_clocks"][i, :k], sent=r["sent"][i], dropped=r["dropped"][i],
                              series=r["trace_series"][i][:, :nt], throughput=r["thr"][i], hist=r["hist"][i])


@pytest.mark.parametrize("seed", ALIAS_SEEDS)
def test_twin_equals_oracle_past_the_sweeps_last_row(seed):
    """Rows for half the launch and an aliased pair: the replicas past the last row run the scenario as written."""
    m = N_H100 // 2
    payload, flat, spec = sweep_case(seed, m, alias=True)
    ids = (m, m + 5, N_H100 - 1)
    for engine in ("lane", "warp"):
        r = twin_run(flat, N_H100, sweep=spec, engine=engine, **CAPS)
        for i in ids:
            assert_matches_oracle(des_port.simulate(payload, seed=SEED, replica=BEGIN + i), flat, stats=r["stats"][i],
                                  clocks=None, sent=r["sent"][i], dropped=r["dropped"][i], throughput=r["thr"][i],
                                  hist=r["hist"][i])


@pytest.mark.parametrize("case", [f"sweep-{s}" for s in SWEEP_SEEDS] + sorted(PARITY_CASES))
def test_twin_accumulating_outputs_of_the_own_groups_equal_the_oracle(case):
    payload, flat, spec = acc_case(case)
    f = occ_bits(flat, spec, CAPS["request_capacity"])
    tw = acc_twin(flat, spec, N_ACC, acc_groups(N_ACC), f, CAPS)
    assert not (tw["stats"]["flags"] != 0).any()
    assert_own_groups_equal_oracle(twin_views(flat, tw), payload, flat, spec, range(OWN), f)
    assert tw["band_rows"].shape[0] == G + OWN + 1


def test_twin_stitched_replicas_equal_the_oracle():
    """The stitched case's flagged replicas, re-run by the warp state machine from where the lane one stopped."""
    payload, flat, spec = sweep_case(STITCH_SEED, COVER)
    flagged = stitched_replicas(flat, spec, COVER)
    groups = acc_groups(COVER, own=flagged[:OWN])
    f = occ_bits(flat, spec, CAPS["request_capacity"])
    lane = acc_twin(flat, spec, COVER, groups, f, dict(event_capacity=512, request_capacity=2048),
                    bin_capacity=CAPS["request_capacity"])     # bins as af_run sizes them: by the caller's capacity
    assert np.array_equal(np.flatnonzero(lane["stats"]["flags"]), flagged)
    out = acc_twin(flat, spec, COVER, groups, f, CAPS, run=twin.run_warp, redo=flagged, into=lane)
    assert not out["stats"]["flags"].any()
    assert_own_groups_equal_oracle(twin_views(flat, out), payload, flat, spec, flagged[:OWN], f)


@pytest.mark.parametrize("case", ["sweep-326", "sweep-327"])
def test_stitched_replicas_give_their_first_hand_rows_in_every_group(case):
    """One group per replica: a replica the lane pass stops (nominal pools) and the warp pass re-runs from its stop tick
    gives the first-hand run's rows.  Several of these replicas overflow in the generator phase, whose timeout would
    fall before the next event: the lane pass must stop them at the ticks already taken, not after the ticks up to that
    event, which miss the lost arrival."""
    _, flat, spec = acc_case(case)
    n = N_ACC
    kw = dict(seed=SEED, n=n, replica_begin=BEGIN, sweep=spec, sweep_first=BEGIN, groups=np.arange(n, dtype=np.uint32),
              n_groups=n, band_first=BEGIN, sampled=True, window=2, series=[0, 2, 3 * flat.n_servers],
              f=occ_bits(flat, spec, CAPS["request_capacity"]), bin_capacity=CAPS["request_capacity"])
    lane = twin.run_lane(flat, event_capacity=512, request_capacity=2048, **kw)
    flagged = np.flatnonzero(lane["stats"]["flags"])
    assert flagged.size >= 5
    out = twin.run_warp(flat, redo=flagged, into=lane, **CAPS, **kw)
    full = twin.run_lane(flat, **CAPS, **kw)
    for k in ("band_rows", "lat_rows", "dist_rows", "occ", "stats", "samp_sum", "hist"):
        assert out[k].tobytes() == full[k].tobytes(), k
