"""CPU tier: af_run hands replicas to lanes in a pull order (heaviest first by predicted work), not in id order.  A
replica's random numbers are keyed by its replica id and its outputs by its local index, so the order in which a lane
pulls them must not change one bit of any output: the state a replica leaves in the lane's shared memory and global
tier is reset when the next one starts, whichever that is.  Runs the CPU twin's lane engine (tests/twin.py)."""

from __future__ import annotations

import numpy as np
import pytest
import twin
from helpers import PARITY_CASES, SEED, load_scenario

from asyncflow_b200 import SweepSpec, flatten


def _run(flat, **kw) -> dict:
    return twin.run_lane(flat, **{"seed": SEED, "lane_bytes": 520, "event_capacity": 8192, "request_capacity": 400000, **kw})


def _assert_same(got, ref):
    assert list(got) == list(ref)
    for k in ref:
        assert got[k].tobytes() == ref[k].tobytes(), k


@pytest.mark.parametrize("name", sorted(PARITY_CASES))
def test_random_pull_order_changes_no_output(name):
    flat = flatten(load_scenario(name, PARITY_CASES[name]))
    n = 5
    kw = dict(n=n, replica_begin=3, trace=2, clock_cap=300000)
    ref = _run(flat, **kw)
    _assert_same(_run(flat, order=np.random.default_rng(11).permutation(n), **kw), ref)


def test_pull_order_across_sweep_rows_with_different_splits():
    """Heavy and light rows of one sweep interleaved in the pull (each on its own split of the pool, some spilling both
    tables to the global tier): reversed order, same outputs."""
    flat = flatten(load_scenario("c1_my_service.yml", 4))
    users = np.array([5.0, 2000.0, 60.0, 900.0])
    spec = SweepSpec(flat, len(users), {("users_mean",): users})
    kw = dict(n=len(users), sweep=spec, trace=4, clock_cap=100000, lane_bytes=420, request_capacity=200000)
    ref = _run(flat, **kw)
    assert (ref["stats"]["flags"] == 0).all()
    assert ref["stats"]["completed"].min() > 0
    _assert_same(_run(flat, order=np.arange(len(users))[::-1], **kw), ref)
