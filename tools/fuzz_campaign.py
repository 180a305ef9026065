"""Offline fuzz campaign: engine state machine (CPU twin) vs the oracle on many random scenarios.

    python tools/fuzz_campaign.py --first 1000 --count 2000 --jobs 8

Test tooling (uses oracle/ and tests/host_twin); prints the failing seeds, exits non-zero on any.
"""
from __future__ import annotations

import argparse
import multiprocessing as mp
import sys
import traceback
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (ROOT, ROOT / "tests", ROOT / "oracle", ROOT / "oracle" / "simpy_shim"):
    sys.path.insert(0, str(p))


ENGINE = "lane"
BIG = False
LAYOUTS = False


def layout_for(seed: int) -> dict:
    """A per-seed shared-memory layout for the lane engine: the budget of one lane (the CUDA engine runs 600-1800 B per
    lane, depending on the occupancy it picks), and a random split of the lane's pool for every replica (2 .. pool - 1
    record slots: af_run splits each replica by its own estimated load)."""
    if not LAYOUTS or ENGINE != "lane":
        return {}
    import random
    r = random.Random(seed * 7919 + 13)
    return {"lane_bytes": r.choice([1, 300, 420, 520, 604, 648, 660, 900, 1200, 1816]),     # 1: the smallest the scenario fits in
            "split": "random", "split_seed": seed}


def one(seed: int):
    import des_port
    import fuzz
    import twin
    from helpers import SEED, assert_matches_oracle

    from asyncflow_b200.flatten import flatten
    try:
        payload = fuzz.big_scenario(seed) if BIG else fuzz.scenario(seed)
        flat = flatten(payload)
        o = des_port.simulate(payload, seed=SEED, replica=seed)
        kw = dict(seed=SEED, replica_begin=seed, n=1, trace=1, clock_cap=200000, request_capacity=400000,
                  event_capacity=8192)
        layout = layout_for(seed)
        if layout:          # tests/split_twin.py: the lane state machine with a split of its pool per replica
            import split_twin
            r = split_twin.run(flat, **kw, **layout)
        else:
            r = twin.run(flat, engine=ENGINE, **kw)
        st = r["stats"][0]
        n, nt = int(st["completed"]), int(st["n_ticks"])
        assert st["flags"] == 0, f"flags {int(st['flags'])}"
        assert_matches_oracle(o, flat, stats=st, clocks=r["trace_clocks"][0, :n], sent=r["sent"][0],
                              dropped=r["dropped"][0], series=r["trace_series"][0][:, :nt], throughput=r["thr"][0])
        return seed, None, n
    except BaseException:
        return seed, traceback.format_exc(limit=3), 0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--first", type=int, default=1000)
    ap.add_argument("--count", type=int, default=500)
    ap.add_argument("--jobs", type=int, default=8)
    ap.add_argument("--engine", default="lane", choices=["lane", "warp"], help="which state machine of tests/twin.py")
    ap.add_argument("--big", action="store_true", help="C5-shaped topologies (fuzz.big_scenario)")
    ap.add_argument("--layouts", action="store_true",
                    help="lane engine: a random per-lane shared-memory budget per seed, a random split of the pool per replica (both tiers of every table)")
    a = ap.parse_args()
    global ENGINE, BIG, LAYOUTS
    ENGINE, BIG, LAYOUTS = a.engine, a.big, a.layouts
    import twin
    twin.build()
    if LAYOUTS and ENGINE == "lane":
        import split_twin
        split_twin.lib()                # built once, before the workers fork
    bad = []
    total = 0
    with mp.get_context("fork").Pool(a.jobs) as pool:
        for i, (seed, err, n) in enumerate(pool.imap_unordered(one, range(a.first, a.first + a.count), chunksize=4)):
            total += n
            if err:
                bad.append(seed)
                print(f"seed {seed} FAILED\n{err}", flush=True)
            if (i + 1) % 100 == 0:
                print(f"{i + 1}/{a.count} scenarios, {total} completions compared, {len(bad)} failures", flush=True)
    print(f"done: {a.count} scenarios, {total} completions compared bit for bit, failures: {bad}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
