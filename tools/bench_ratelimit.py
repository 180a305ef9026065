"""A rate-limit grid as one launch against one launch per value, and what a rate limit costs the launch.

The grid: C3 (two servers behind a load balancer) at ``--users``, rates ``--rates`` (requests per second, 0: none) with
burst ``--burst`` placed at the load balancer (the whole rate) or on each server (half of it each) x ``--reps``
repetitions, repetition k on stream k.  ``one launch``: one ``SweepRunner`` over every row with ``("lb_rate",)`` /
``("lb_burst",)`` and ``("server_rate"|"server_burst", server)`` columns (the full lane build).  ``per value``: one
scenario per (rate, placement) (``flatten.set_rate_limits``), each its own ``SweepRunner`` of ``--reps`` rows.
``no limit``: the one launch's rows without the rate-limit columns, which run the lean lane build: the cost baseline.
The first two give every row the same outputs (checked: stats and throttle counts).  Prints completions/s over the
device time of each way's launches (CUDA events), the median of ``--rounds`` alternating rounds, and the GPU's name and
power limit read in the same call.

    python tools/bench_ratelimit.py [--reps 10000] [--users 400] [--horizon 30] [--rounds 3] [--dry-run]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from asyncflow_b200 import SweepRunner, SweepSpec, flatten  # noqa: E402
from asyncflow_b200.flatten import set_rate_limits  # noqa: E402

PLACEMENTS = ("lb", "servers")


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (x.strip() for x in out.split(",", 1))
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10000)
    ap.add_argument("--users", type=float, default=400.0)
    ap.add_argument("--rates", type=float, nargs="+", default=[0.0, 200.0, 400.0, 800.0])
    ap.add_argument("--burst", type=int, default=20)
    ap.add_argument("--horizon", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dry-run", action="store_true", help="build every launch's rows; run nothing")
    a = ap.parse_args()
    payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
    payload["sim_settings"]["total_simulation_time"] = a.horizon
    payload["rqs_input"]["avg_active_users"]["mean"] = a.users
    flat = flatten(payload)
    rates = np.asarray(a.rates, dtype=float)
    C, P, R = len(rates), len(PLACEMENTS), a.reps
    ri, pi, rep = (g.ravel() for g in np.meshgrid(np.arange(C), np.arange(P), np.arange(R), indexing="ij"))
    at_lb = pi == 0
    cols = {("lb_rate",): np.where(at_lb, rates[ri], 0.0), ("lb_burst",): np.full(len(rep), a.burst)}
    cols.update({("server_rate", s): np.where(at_lb, 0.0, rates[ri] / flat.n_servers) for s in flat.server_ids})
    cols.update({("server_burst", s): np.full(len(rep), a.burst) for s in flat.server_ids})
    per_value = []
    for c in range(C):
        for p in range(P):
            f = flatten(payload)
            if p == 0:
                set_rate_limits(f, None, lb=(float(rates[c]), a.burst))
            else:
                set_rate_limits(f, {s: (float(rates[c]) / f.n_servers, a.burst) for s in f.server_ids})
            per_value.append(((ri == c) & (pi == p), f))
    if a.dry_run:
        SweepSpec(flat, len(rep), cols)
        print(f"{len(rep)} rows ({C} rates x {P} placements x {R}); one launch, {C * P} launches per value, one "
              "launch without")
        return
    ways = {"one_launch": [SweepRunner(flat, len(rep), cols, seed=3, streams=rep)],
            "per_value": [SweepRunner(f, R, None, seed=3, streams=np.arange(R)) for _, f in per_value],
            "no_limit": [SweepRunner(flatten(payload), len(rep), None, seed=3, streams=rep)]}

    def run(key):
        out, dev = [], 0.0
        for r in ways[key]:
            out.append(r.run())
            dev += r.last_ms[0] / 1e3
        return out, dev

    for key in ways:                        # warm-up: engines, allocations
        run(key)
    dev: dict = {k: [] for k in ways}
    last: dict = {}
    order = list(ways)
    for k in range(a.rounds):               # alternate, direction flipped every round
        for key in (order if k % 2 == 0 else order[::-1]):
            last[key], d = run(key)
            dev[key].append(d)
    one = last["one_launch"][0]
    same = True
    for (mask, _), r in zip(per_value, last["per_value"]):
        rows = np.flatnonzero(mask)
        for fld in ("generated", "completed", "n_events", "lat_sum", "lat_max"):
            same = same and np.array_equal(one.stats[fld][rows], r.stats[fld])
        same = same and np.array_equal(one.server_throttled[rows], r.server_throttled)
        same = same and np.array_equal(one.lb_throttled[rows], r.lb_throttled)
    info = gpu_info()
    lean = {key: bool(ways[key][0].engine().last_run_passes()["lane_lean"]) for key in ("one_launch", "no_limit")}
    gen = max(1, int(one.stats["generated"].sum()))
    out = {"replicas": int(len(rep)), "rates": a.rates, "burst": a.burst, "horizon": a.horizon, "users": a.users,
           "throttled_fraction": float((one.server_throttled.sum() + one.lb_throttled.sum()) / gen),
           "identical": bool(same), "lean": lean, **info}
    for key in ways:
        done = float(sum(r.stats["completed"].sum() for r in last[key]))
        out[key + "_device_s"] = float(np.median(dev[key]))
        out[key + "_completions_per_s"] = done / float(np.median(dev[key]))
        out[key + "_events_per_s"] = float(sum(r.stats["n_events"].sum() for r in last[key])) / float(np.median(dev[key]))
    print(f"{len(rep)} replicas ({C} rates x {P} placements x {R}), horizon {a.horizon} s, users {a.users:g}; "
          f"{info['gpu']}, power limit {info['power_limit']}; outputs of one launch and per-value launches identical: "
          f"{same}; lean lane build: {lean}")
    for key in ways:
        print(f"  {key:<12s} {out[key + '_device_s'] * 1e3:9.2f} ms device, {out[key + '_completions_per_s']:.4g} "
              f"completions/s, {out[key + '_events_per_s']:.4g} events/s")
    print(json.dumps(out))
    for rs in ways.values():
        for r in rs:
            r.close()


if __name__ == "__main__":
    main()
