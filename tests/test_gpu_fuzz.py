"""GPU tier: the random campaigns of the CPU tier (tests/fuzz.py) on the device, against the CPU twin and the oracle.

The twin runs the engines' state machines with a warp of one lane, so it never runs the code under ``AF_DEVICE_CODE``:
the event pool's arg-min over 32 lanes (``pool_scan``: ``w_min`` / ``w_ballot``, the between-lane tie-break on the push
sequence, ``more`` from two ballots; ``pool_top``, ``pool_find_hole``), the RED atomics and af_run's own launch set-up
(which sweep columns may share a slot).  Here whole launches of random scenarios, random sweeps of every sweep field and
C5-shaped big topologies run on the device in every pass structure, with lanes and warps running several replicas, and
must equal the twin byte for byte; selected replicas must equal the oracle directly (clocks and sampled series
included).  Then the four accumulating outputs (per-tick, latency and distribution bands, occupancy integrals) run
together on the random sweeps and every parity scenario, against the twin and, replica by replica, the oracle-side
references.  tests/test_fuzz_device_inputs.py checks on the CPU that the references and the coverage claims hold."""

from __future__ import annotations

import band_ref
import des_port
import fuzz
import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, assert_matches_oracle, load_scenario
from test_bands import expected as band_expected
from test_bands import oracle_matrix
from test_dist_bands import expected as dist_expected
from test_gpu_multiwave import BEGIN, CAPS, WARP_HORIZONS, assert_launch_equals_twin, device_run, sm_count, twin_run
from test_latency_bands import expected as lat_expected

from asyncflow_b200 import Engine, SweepSpec, flatten
from asyncflow_b200 import _capi as K
from asyncflow_b200.results import occ_frac_bits, occupancy_columns

pytestmark = pytest.mark.gpu

#: the CPU tier's random-sweep seeds (test_fuzz_parity), then a block of fresh ones
SWEEP_SEEDS = [*range(300, 330), *range(600, 603)]
#: rows of every random sweep: the generator's choices of fields depend on the row count, so it is fixed, not sized by
#: the device (a launch uses the first rows it needs)
SWEEP_ROWS = 12_000
#: sweeps run again on lanes that take two replicas or more, and sweeps with an aliased pair of step columns run past
#: their last row
REUSE_SEEDS = [300, 322, 602]
ALIAS_SEEDS = [301, 308, 315, 329]
#: the CPU tier's random-scenario seeds, on the warp engine
WARP_SEEDS = list(range(100, 170))
BIG_SEEDS = list(range(16))
BIG_CAPS = dict(event_capacity=8192, request_capacity=400_000)
TRACE, CLOCK_CAP = 3, 100_000
#: local replicas [0, COVER) of each warp-seed launch: the ones the coverage claims are made on
COVER = 256
#: the warp engine's shared-memory tiers (afh::DEFAULT_EV_SMEM, DEFAULT_RQ_SMEM): 2 pool slots per lane
WARP_EV_SMEM = WARP_RQ_SMEM = 64
SLOT_FIELDS = ("edge_mean", "edge_sigma", "edge_dropout", "step_duration", "endpoint_ram", "spike_delta")


# ---- inputs (no device) -----------------------------------------------------------------------------------------------
def _step_base(payload: dict, sel: tuple) -> float:
    srv = next(s for s in payload["topology_graph"]["nodes"]["servers"] if s["id"] == sel[1])
    (v,) = srv["endpoints"][sel[2]]["steps"][sel[3]]["step_operation"].values()
    return float(v)


def alias_pair(payload: dict) -> tuple[tuple, tuple] | None:
    """Two step-duration selectors of the scenario whose base durations differ (the first such pair), or None."""
    steps = [("step_duration", s["id"], j, k) for s in payload["topology_graph"]["nodes"]["servers"]
             for j, ep in enumerate(s["endpoints"]) for k, st in enumerate(ep["steps"]) if st["kind"] != "ram"]
    for i, a in enumerate(steps):
        for b in steps[i + 1:]:
            if _step_base(payload, a) != _step_base(payload, b):
                return a, b
    return None


def sweep_case(seed: int, rows: int = SWEEP_ROWS, *, alias: bool = False):
    """(payload, flat, spec): ``fuzz.sweep_columns`` over BEGIN + rows rows.  ``alias``: the second step of
    :func:`alias_pair` takes the first one's column (one is drawn when the generator did not sweep it), so the two
    columns are equal in every row while their base durations differ."""
    payload = fuzz.scenario(seed)
    flat = flatten(payload)
    cols = fuzz.sweep_columns(seed, payload, BEGIN + SWEEP_ROWS)
    if alias:
        a, b = alias_pair(payload)
        if a not in cols:
            cols[a] = list(np.random.default_rng(seed).choice(fuzz.DUR, BEGIN + SWEEP_ROWS))
        cols[b] = list(cols[a])
    cols = {sel: np.asarray(v, dtype=np.float64)[:BEGIN + rows] for sel, v in cols.items()}
    return payload, flat, SweepSpec(flat, BEGIN + rows, cols)


def column_aliases(values: np.ndarray) -> list[int]:
    """aflh::column_aliases restated: alias[c] = the first earlier unaliased column equal to column c in every row."""
    alias = [-1] * values.shape[1]
    for c in range(1, values.shape[1]):
        for a in range(c):
            if alias[a] < 0 and np.array_equal(values[:, c], values[:, a]):
                alias[c] = a
                break
    return alias


def aliased_slot_columns(spec: SweepSpec, first: int, count: int) -> list[tuple[int, int]]:
    """(column, the column whose slot it shares) of the looked-up columns, when rows [first, first + count) are
    uploaded and every replica of the launch has a row."""
    names = {v: k for k, v in K.FIELDS.items()}
    alias = column_aliases(spec.values[first:first + count])
    return [(c, a) for c, a in enumerate(alias) if a >= 0 and names[spec.columns[c][0]] in SLOT_FIELDS]


def added_alias_shares_a_slot(seed: int, rows: int) -> bool:
    """Whether the step columns :func:`sweep_case` made equal share a slot over rows [BEGIN, BEGIN + rows), with
    different base durations."""
    payload, flat, spec = sweep_case(seed, rows, alias=True)
    a, b = alias_pair(payload)
    ca, cb = (spec.columns.index((K.FIELDS["step_duration"], flat.step_index[s[1:]])) for s in (a, b))
    return (cb, ca) in aliased_slot_columns(spec, BEGIN, rows) and _step_base(payload, a) != _step_base(payload, b)


def swept_fields(seeds) -> set[str]:
    return {sel[0] for s in seeds for sel, _ in sweep_case(s, 1)[2].selectors}


def finish_ties(clocks) -> int:
    """Completions of an oracle replica that finish at an instant another completion also finishes at."""
    f = np.asarray(clocks, dtype=np.float64).reshape(-1, 2)[:, 1]
    _, counts = np.unique(f, return_counts=True)
    return int(counts[counts > 1].sum())


# ---- references, cached per module (the twin over a launch is what most of this file's time goes to) ---------------
_refs: dict = {}


def cached(key, make):
    if key not in _refs:
        _refs[key] = make()
    return _refs[key]


def warp_seed_reference(seed: int, n: int):
    payload = fuzz.scenario(seed)
    flat = flatten(payload)
    return payload, flat, cached(("warp", seed, n), lambda: twin_run(flat, n, begin=seed, **CAPS))


def big_reference(seed: int, n: int):
    payload = fuzz.big_scenario(seed)
    flat = flatten(payload)
    return payload, flat, cached(("big", seed, n), lambda: twin_run(flat, n, begin=seed, **BIG_CAPS))


def assert_traced_equal_oracle(dev: dict, payload: dict, flat, spec, local_ids, *, begin: int = BEGIN) -> None:
    for i in local_ids:
        p = payload if spec is None else spec.payload_for(payload, begin + i)
        o = des_port.simulate(p, seed=SEED, replica=begin + i)
        assert_matches_oracle(o, flatten(p), stats=dev["stats"][i], clocks=dev["clocks"][i], sent=dev["sent"][i],
                              dropped=dev["dropped"][i], series=dev["series"][i], throughput=dev["thr"][i],
                              hist=dev["hist"][i])


# ---- accumulating outputs ----------------------------------------------------------------------------------------------
#: groups: the first OWN local replicas of a launch each have a group of their own (G, G + 1, ...), checked against the
#: oracle; every other replica i is in group i % G, checked against the twin
G, OWN, N_ACC, WINDOW = 4, 3, 64, 2


def acc_groups(n: int, own=range(OWN)) -> np.ndarray:
    g = (np.arange(n) % G).astype(np.uint32)
    for k, i in enumerate(own):
        g[i] = G + k
    return g


def dist_series(flat) -> list[int]:
    """A few sampled series: server 0's ready queue and RAM in use, the first edge's connections."""
    return [0, 2, 3 * flat.n_servers]


def occ_bits(flat, spec, request_capacity: int) -> int:
    ram = [float(flat.pod.servers[i].ram_mb) for i in range(flat.n_servers)]
    if spec is not None:
        names = {v: k for k, v in K.FIELDS.items()}
        ram += [float(spec.values[:, c].max()) for c, (f, _) in enumerate(spec.columns) if names[f] == "server_ram_mb"]
    return occ_frac_bits(max(request_capacity, int(max(ram))), int(flat.horizon_s))


def acc_twin(flat, spec, n: int, groups, f: int, caps: dict, *, run=None, **kw) -> dict:
    """The twin with all four accumulating outputs on: per-tick bands, latency bands, distribution bands, occupancy."""
    run = run or twin.run_lane
    return run(flat, seed=SEED, n=n, replica_begin=BEGIN, sweep=spec, sweep_first=BEGIN if spec is not None else 0,
               groups=groups, n_groups=G + OWN, band_first=BEGIN, sampled=True, window=WINDOW,
               series=dist_series(flat), f=f, **caps, **kw)


def twin_views(flat, tw: dict) -> dict:
    """The twin's difference rows as the device's fetches return them."""
    n_groups = G + OWN
    T = tw["dist_rows"].shape[2] - 1
    return {"bands": band_ref.scan(flat, tw["band_rows"], n_groups), "lat": twin.lat_split(tw["lat_rows"], n_groups),
            "dist": band_ref.dist_scan(tw["dist_rows"], n_groups, T), "occ": tw["occ"]}


def assert_views_equal(got: dict, want: dict) -> None:
    for kind in ("bands", "lat"):
        for k, (a, b) in enumerate(zip(got[kind], want[kind])):
            assert a.dtype == b.dtype and a.shape == b.shape, (kind, k, a.shape, b.shape)
            if not np.array_equal(a, b):
                groups = np.flatnonzero((a != b).reshape(len(a), -1).any(axis=1))
                pytest.fail(f"{kind}[{k}]: groups {groups.tolist()} differ")
    for kind in ("dist", "occ"):
        a, b = got[kind], want[kind]
        assert a.dtype == b.dtype and a.shape == b.shape, (kind, a.shape, b.shape)
        if not np.array_equal(a, b):
            rows = np.flatnonzero((a != b).reshape(len(a), -1).any(axis=1))
            pytest.fail(f"{kind}: rows {rows[:8].tolist()} differ")


def own_groups_oracle(payload: dict, flat, spec, own, f: int) -> tuple[list, list, list]:
    """(occupancy rows, series matrices, clocks) of the oracle's replicas BEGIN + own[k]."""
    occs, mats, clocks = [], [], []
    for i in own:
        p = payload if spec is None else spec.payload_for(payload, BEGIN + i)
        o, ledger, _ = band_ref.oracle_ledger(p, flat, seed=SEED, replica=BEGIN + i)
        occs.append(band_ref.ledger_rows(ledger, twin.occ_cols(flat), float(flat.horizon_s), f))
        mats.append(oracle_matrix(p, flat, BEGIN + i))
        clocks.append(np.asarray(o["clocks"], dtype=np.float64).reshape(-1, 2))
    return occs, mats, clocks


def assert_own_groups_equal_oracle(views: dict, payload: dict, flat, spec, own, f: int, key=None) -> None:
    """Group G + k holds local replica own[k] alone: its per-tick band sums, latency rows and distribution rows, and
    that replica's occupancy row, against the oracle-side definitions (test_bands, test_latency_bands, test_dist_bands,
    band_ref's ledger).  ``key``: cache the oracle's side under it."""
    n_groups, T = G + OWN, twin.ticks(flat)
    make = lambda: own_groups_oracle(payload, flat, spec, own, f)  # noqa: E731
    occs, mats, clocks = make() if key is None else cached(("oracle",) + key, make)
    for i, occ in zip(own, occs):
        assert views["occ"][i].tobytes() == occ.tobytes(), ("occupancy", i)
    ks = list(range(len(own)))
    want = band_expected(flat, mats, ks, len(own))
    for name, a, b in zip(("count", "sum", "sumsq"), views["bands"], want):
        assert np.array_equal(a[G:G + len(own)], b), ("bands", name)
    lat = twin.lat_split(lat_expected(flat, clocks, ks, len(own), WINDOW), len(own))
    for name, a, b in zip(("hist", "sum_hi", "sum_lo"), views["lat"], lat):
        assert np.array_equal(a[G:G + len(own)], b), ("latency", name)
    d = views["dist"]
    want_d = dist_expected([m.astype(np.uint32) for m in mats], dist_series(flat), ks, len(own), T, d.shape[3])
    assert np.array_equal(d[G:G + len(own)], want_d), "distribution"
    assert d.shape[:3] == (n_groups, len(dist_series(flat)), T)


def acc_device(flat, spec, n: int, groups, f: int, mode: str, caps: dict) -> tuple[dict, dict]:
    """One launch with all four accumulating outputs on, on an engine of its own: (outputs, views)."""
    with Engine(0) as eng:
        eng.upload(flat)
        eng.set_mode(mode)
        eng.configure(warps_per_block=1, **caps)
        if spec is not None:
            eng.upload_sweep(spec, BEGIN, row_first=BEGIN, row_count=n)
        eng.configure_bands(sampled=True, latency_window_s=WINDOW)
        eng.configure_dist_bands(dist_series(flat))
        eng.configure_occupancy(True, f)
        eng.upload_bands(groups, BEGIN, G + OWN)
        eng.run(SEED, BEGIN, BEGIN + n)
        sent, dropped = eng.edge_counts()
        ssum, smax = eng.sampled()
        occ, f_dev = eng.occupancy()
        assert f_dev == f
        out = {"stats": eng.stats().copy(), "sent": sent, "dropped": dropped, "samp_sum": ssum, "samp_max": smax,
               "hist": eng.histograms(), "thr": eng.throughput(), "reduced": eng.reduced_histogram(),
               "passes": eng.last_run_passes()}
        views = {"bands": eng.bands(), "lat": eng.latency_bands(), "dist": eng.dist_bands(), "occ": occ}
    return out, views


def acc_case(case: str):
    """(payload, flat, spec) of an accumulating-output case: ``sweep-<seed>`` or a parity scenario (on the multiwave
    file's horizons: the oracle's ledger of a 250 s C4 replica alone takes a minute)."""
    if case.startswith("sweep-"):
        return sweep_case(int(case[6:]), N_ACC)
    payload = load_scenario(case, WARP_HORIZONS[case])
    return payload, flatten(payload), None


# ---- the tests ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    with Engine(0) as e:
        yield e


def test_the_sweep_parametrisation_covers_every_field_and_an_aliased_pair():
    """If the generator stops sweeping a field, or no launch shares a slot between columns with different bases, this
    fails rather than the campaign silently shrinking."""
    assert swept_fields(SWEEP_SEEDS) == set(K.FIELDS), set(K.FIELDS) - swept_fields(SWEEP_SEEDS)
    m = (4 * sm_count() + 7) // 2
    assert all(added_alias_shares_a_slot(seed, m) for seed in ALIAS_SEEDS)


@pytest.mark.parametrize("mode", ["lane", "warp", "two_pass", "auto"])
@pytest.mark.parametrize("seed", SWEEP_SEEDS)
def test_random_sweeps_equal_the_twin_and_the_oracle(eng, seed, mode):
    """4 x SMs + 7 replicas of a random sweep, one warp per block: in WARP and AUTO (too few replicas for lanes) one
    block per SM, so every warp runs four replicas or more; LANE and TWO_PASS on the lanes the launch needs (TWO_PASS
    re-runs the replicas that outgrow the lane pass's nominal pools).  The first replicas are traced."""
    sms = sm_count()
    n = 4 * sms + 7
    payload, flat, spec = sweep_case(seed)
    ref = cached(("sweep", seed, n), lambda: twin_run(flat, n, sweep=spec, **CAPS))
    eng.set_mode(mode)
    shape = dict(warps_per_block=1, blocks_per_sm=1 if mode in ("warp", "auto") else 0)
    dev = device_run(eng, flat, n, sweep=spec, trace=TRACE, clock_cap=CLOCK_CAP, **shape, **CAPS)
    p = dev["passes"]
    if mode in ("warp", "auto"):
        assert p["lane_pass"] == 0 and p["warp_pass"] == 1 and p["warp_replicas"] == n, p
    else:
        assert p["lane_pass"] == 1 and p["lane_replicas"] == n, p
    assert_launch_equals_twin(dev, ref)
    assert_traced_equal_oracle(dev, payload, flat, spec, range(TRACE))


@pytest.mark.parametrize("mode", ["lane", "two_pass"])
@pytest.mark.parametrize("seed", REUSE_SEEDS)
def test_random_sweeps_on_lanes_that_run_two_replicas_or_more(eng, seed, mode):
    """One warp per SM and lanes x 1.5 replicas: half the lanes or more start a second replica on their leftover
    state, each with its own row's pool split (and slots shared between equal columns, spike marks)."""
    sms = sm_count()
    lanes = sms * 32
    n = lanes + lanes // 2 + 17
    payload, flat, spec = sweep_case(seed)
    assert n <= SWEEP_ROWS
    ref = cached(("sweep", seed, n), lambda: twin_run(flat, n, sweep=spec, **CAPS))
    eng.set_mode(mode)
    dev = device_run(eng, flat, n, sweep=spec, warps_per_block=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 1 and p["lane_warps_per_sm"] == 1 and p["lane_replicas"] == n > lanes, p
    assert_launch_equals_twin(dev, ref)


@pytest.mark.parametrize("mode", ["lane", "two_pass", "warp"])
@pytest.mark.parametrize("seed", ALIAS_SEEDS)
def test_a_launch_past_the_sweeps_last_row_takes_each_columns_base(eng, seed, mode):
    """Rows for the first half of the launch only, two step columns equal in every row over different base durations:
    the replicas past the last row take each column's own base, so af_run must not let the columns share a slot."""
    sms = sm_count()
    n = 4 * sms + 7
    m = n // 2
    payload, flat, spec = sweep_case(seed, m, alias=True)
    assert aliased_slot_columns(spec, BEGIN, m)                       # the columns would share a slot with rows for all
    ref = cached(("past", seed, n), lambda: twin_run(flat, n, sweep=spec, **CAPS))
    eng.set_mode(mode)
    shape = dict(warps_per_block=1, blocks_per_sm=1 if mode == "warp" else 0)
    dev = device_run(eng, flat, n, sweep=spec, rows=m, trace=TRACE, clock_cap=CLOCK_CAP, **shape, **CAPS)
    assert dev["passes"]["lane_pass" if mode != "warp" else "warp_pass"] == 1
    assert_launch_equals_twin(dev, ref)
    assert_traced_equal_oracle(dev, payload, flat, spec, range(TRACE))
    for i in (m, m + 5, n - 1):                                      # past the last row: the scenario as written
        o = des_port.simulate(payload, seed=SEED, replica=BEGIN + i)
        assert_matches_oracle(o, flat, stats=dev["stats"][i], clocks=None, sent=dev["sent"][i], dropped=dev["dropped"][i],
                              throughput=dev["thr"][i], hist=dev["hist"][i])


@pytest.mark.parametrize("seed", WARP_SEEDS)
def test_random_scenarios_on_warps_that_run_several_replicas(eng, seed):
    """WARP mode, one warp per block and one block per SM, replicas [seed, seed + 2 x SMs + 7): every warp runs two
    replicas or three through the device's pool scan.  Replica ``seed`` (traced) against the oracle directly."""
    sms = sm_count()
    n = 2 * sms + 7
    assert n >= COVER
    payload, flat, ref = warp_seed_reference(seed, n)
    eng.set_mode("warp")
    dev = device_run(eng, flat, n, begin=seed, trace=1, clock_cap=CLOCK_CAP, warps_per_block=1, blocks_per_sm=1, **CAPS)
    p = dev["passes"]
    assert p["lane_pass"] == 0 and p["warp_replicas"] == n, p
    assert_launch_equals_twin(dev, ref)
    assert_traced_equal_oracle(dev, payload, flat, None, [0], begin=seed)


#: stated shares: replicas of the warp-seed launches whose pool held more events than its shared-memory slots, and
#: seeds whose oracle replica finishes two requests at one instant
MULTI_SLOT_SHARE, TIE_SEEDS = 0.5, 8


def warp_seed_coverage(refs) -> tuple[float, int]:
    """(share of replicas with peak_events > 64, seeds with finish ties in the oracle's replica ``seed``) over
    ``refs`` = [(seed, twin outputs of replicas [seed, seed + >= COVER))]."""
    peaks = np.concatenate([r["stats"]["peak_events"][:COVER] for _, r in refs])
    ties = sum(finish_ties(des_port.simulate(fuzz.scenario(s), seed=SEED, replica=s)["clocks"]) > 0 for s, _ in refs)
    return float((peaks > WARP_EV_SMEM).mean()), int(ties)


def test_the_warp_seeds_reach_multi_slot_pools_and_ties():
    n = 2 * sm_count() + 7
    share, ties = warp_seed_coverage([(s, warp_seed_reference(s, n)[2]) for s in WARP_SEEDS])
    assert share >= MULTI_SLOT_SHARE and ties >= TIE_SEEDS, (share, ties)


@pytest.mark.parametrize("mode", ["warp", "two_pass"])
@pytest.mark.parametrize("seed", BIG_SEEDS)
def test_big_topologies_equal_the_twin_and_the_oracle(eng, seed, mode):
    """C5-shaped, overloaded: replicas [seed, seed + 48) with the CPU tier's capacities, one warp per block and SM.
    Their pools reach the warp engine's spill regions; in TWO_PASS, the replicas that outgrow the lane pass's nominal
    global tiers (half the seeds) are re-run on warps."""
    n = 48
    payload, flat, ref = big_reference(seed, n)
    eng.set_mode(mode)
    dev = device_run(eng, flat, n, begin=seed, trace=1, clock_cap=200_000, warps_per_block=1, blocks_per_sm=1, **BIG_CAPS)
    p = dev["passes"]
    st = dev["stats"]
    assert (st["peak_events"] > WARP_EV_SMEM).any() and (st["peak_requests"] > WARP_RQ_SMEM).any()
    if mode == "warp":
        assert p["lane_pass"] == 0, p
    else:
        lane = twin.run_lane(flat, seed=SEED, n=n, replica_begin=seed, **NOMINAL)
        assert p["lane_pass"] == 1 and p["lane_replicas"] == n, p
        assert p["warp_replicas"] == int((lane["stats"]["flags"] != 0).sum()), p
        if p["warp_replicas"]:     # the lane pass filled its shared and global tiers (nominal capacities) and stopped
            assert ((st["peak_events"] > NOMINAL["event_capacity"]) | (st["peak_requests"] > NOMINAL["request_capacity"])).any()
    assert_launch_equals_twin(dev, ref)
    assert_traced_equal_oracle(dev, payload, flat, None, [0], begin=seed)


ACC_CASES = [f"sweep-{s}" for s in SWEEP_SEEDS[:30:3]] + ["sweep-326"] + sorted(PARITY_CASES)


@pytest.mark.parametrize("mode", ["lane", "warp", "two_pass"])
@pytest.mark.parametrize("case", ACC_CASES)
def test_every_accumulating_output_equals_the_twin_and_the_oracle(case, mode):
    """Per-tick bands, latency bands, distribution bands and occupancy, all on, over 64 replicas.  In TWO_PASS, sweeps
    326 and 327 have replicas whose generator timeout overflows the lane pass's pool ticks before their next event:
    they must stop at the ticks taken so far, or the re-run from there leaves those ticks wrong."""
    payload, flat, spec = acc_case(case)
    groups = acc_groups(N_ACC)
    f = occ_bits(flat, spec, CAPS["request_capacity"])
    tw = cached(("acc", case), lambda: acc_twin(flat, spec, N_ACC, groups, f, CAPS))
    dev, views = acc_device(flat, spec, N_ACC, groups, f, mode, CAPS)
    assert_launch_equals_twin(dev, tw)
    assert_views_equal(views, twin_views(flat, tw))
    assert_own_groups_equal_oracle(views, payload, flat, spec, range(OWN), f, key=(case,))


#: a random sweep whose heaviest replicas outgrow the lane pass's nominal pools (afl::LANE_EVENT_CAPACITY = 512 events)
STITCH_SEED, NOMINAL = 320, dict(event_capacity=512, request_capacity=2048)


def stitched_replicas(flat, spec, n: int) -> np.ndarray:
    """Local replicas the lane pass flags at its nominal capacities (what TWO_PASS re-runs on warps)."""
    lane = twin.run_lane(flat, seed=SEED, n=n, replica_begin=BEGIN, sweep=spec, sweep_first=BEGIN, **NOMINAL)
    return np.flatnonzero(lane["stats"]["flags"] & (K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW))


def test_stitched_fuzz_replicas_give_their_first_hand_rows():
    """TWO_PASS on a random sweep: the lane pass stops the replicas that outgrow its nominal pools and the warp pass
    re-runs them from where their bands stopped; every output equals the twin's first-hand run, and the stitched
    replicas' own groups and occupancy rows equal the oracle's."""
    n = 4 * sm_count() + 7
    payload, flat, spec = sweep_case(STITCH_SEED, n)
    flagged = stitched_replicas(flat, spec, n)
    assert flagged.size >= 1
    groups = acc_groups(n, own=flagged[:OWN])
    f = occ_bits(flat, spec, CAPS["request_capacity"])
    dev, views = acc_device(flat, spec, n, groups, f, "two_pass", CAPS)
    assert dev["passes"]["warp_replicas"] == flagged.size, dev["passes"]
    tw = acc_twin(flat, spec, n, groups, f, CAPS)
    assert_launch_equals_twin(dev, tw)
    assert_views_equal(views, twin_views(flat, tw))
    assert_own_groups_equal_oracle(views, payload, flat, spec, flagged[:OWN], f)


def test_every_occupancy_state_is_nonzero_on_the_device():
    """Over the parity scenarios and a few random sweeps, on the lane and the warp engine: RAM waits, CPU waits, cores
    held, I/O, RAM in use and edge transit each integrate to a non-zero value somewhere."""
    states = {"lane": set(), "warp": set()}
    for case in sorted(PARITY_CASES) + [f"sweep-{s}" for s in SWEEP_SEEDS[:6]]:
        _, flat, spec = acc_case(case)
        f = occ_bits(flat, spec, CAPS["request_capacity"])
        for mode, seen in states.items():
            _, views = acc_device(flat, spec, N_ACC, acc_groups(N_ACC), f, mode, CAPS)
            seen |= {st for (_, st), v in zip(occupancy_columns(flat), views["occ"].any(axis=0)) if v}
    for seen in states.values():
        assert seen == {"ram_wait", "cpu_wait", "cpu", "io", "ram_mb", "transit"}, states
