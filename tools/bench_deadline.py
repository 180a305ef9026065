"""A request-deadline grid as one launch against one launch per deadline, and what a deadline costs the launch.

The grid: C3 (two servers behind a load balancer) at ``--users``, deadlines ``--deadlines`` (seconds, 0: none) on both
servers with the client timeout ``--timeout`` x ``--reps`` repetitions, repetition k on stream k.  ``one launch``: one
``SweepRunner`` over every row with ``("server_deadline", server)`` and ``("client_timeout",)`` columns (the full lane
build).  ``per deadline``: one scenario per deadline (``flatten.set_deadlines``), each its own ``SweepRunner`` of
``--reps`` rows.  ``no deadline``: the one launch's rows without the deadline columns, which run the lean lane build:
the cost baseline.  The first two give every row the same outputs (checked: stats, expiry and late counts).  Prints
completions/s over the device time of each way's launches (CUDA events), the median of ``--rounds`` alternating rounds,
and the GPU's name and power limit read in the same call.

    python tools/bench_deadline.py [--reps 20000] [--users 400] [--horizon 30] [--rounds 3] [--dry-run]
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
from asyncflow_b200.flatten import set_deadlines  # noqa: E402


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
    ap.add_argument("--reps", type=int, default=20000)
    ap.add_argument("--users", type=float, default=400.0)
    ap.add_argument("--deadlines", type=float, nargs="+", default=[0.0, 0.01, 0.02, 0.05, 0.1])
    ap.add_argument("--timeout", type=float, default=0.05)
    ap.add_argument("--horizon", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dry-run", action="store_true", help="build every launch's rows; run nothing")
    a = ap.parse_args()
    payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
    payload["sim_settings"]["total_simulation_time"] = a.horizon
    payload["rqs_input"]["avg_active_users"]["mean"] = a.users
    flat = flatten(payload)
    C, R = len(a.deadlines), a.reps
    lim, rep = (g.ravel() for g in np.meshgrid(np.arange(C), np.arange(R), indexing="ij"))
    cols = {("server_deadline", s): np.asarray(a.deadlines, dtype=float)[lim] for s in flat.server_ids}
    cols[("client_timeout",)] = np.full(len(rep), a.timeout)
    per_deadline = []
    for d in a.deadlines:
        f = flatten(payload)
        set_deadlines(f, dict.fromkeys(f.server_ids, d), client_timeout=a.timeout)
        per_deadline.append(f)
    if a.dry_run:
        SweepSpec(flat, len(rep), cols)
        print(f"{len(rep)} rows ({C} deadlines x {R}); one launch, {C} launches per deadline, one launch without")
        return
    ways = {"one_launch": [SweepRunner(flat, len(rep), cols, seed=3, streams=rep)],
            "per_deadline": [SweepRunner(f, R, None, seed=3, streams=np.arange(R)) for f in per_deadline],
            "no_deadline": [SweepRunner(flatten(payload), len(rep), None, seed=3, streams=rep)]}

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
    for c, r in enumerate(last["per_deadline"]):
        rows = np.flatnonzero(lim == c)
        for fld in ("generated", "completed", "n_events", "lat_sum", "lat_max"):
            same = same and np.array_equal(one.stats[fld][rows], r.stats[fld])
        same = same and np.array_equal(one.server_expired[rows], r.server_expired)
        same = same and np.array_equal(one.late[rows], r.late)
    info = gpu_info()
    lean = {key: bool(ways[key][0].engine().last_run_passes()["lane_lean"]) for key in ("one_launch", "no_deadline")}
    out = {"replicas": int(len(rep)), "deadlines": a.deadlines, "timeout": a.timeout, "horizon": a.horizon,
           "users": a.users, "expired_fraction": float(one.server_expired.sum() / max(1, one.stats["generated"].sum())),
           "late_fraction": float(one.late.sum() / max(1, one.stats["completed"].sum())), "identical": bool(same),
           "lean": lean, **info}
    for key in ways:
        done = float(sum(r.stats["completed"].sum() for r in last[key]))
        out[key + "_device_s"] = float(np.median(dev[key]))
        out[key + "_completions_per_s"] = done / float(np.median(dev[key]))
        out[key + "_events_per_s"] = float(sum(r.stats["n_events"].sum() for r in last[key])) / float(np.median(dev[key]))
    print(f"{len(rep)} replicas ({C} deadlines x {R}), horizon {a.horizon} s, users {a.users:g}; {info['gpu']}, "
          f"power limit {info['power_limit']}; outputs of one launch and per-deadline launches identical: {same}; "
          f"lean lane build: {lean}")
    for key in ways:
        print(f"  {key:<12s} {out[key + '_device_s'] * 1e3:9.2f} ms device, {out[key + '_completions_per_s']:.4g} "
              f"completions/s, {out[key + '_events_per_s']:.4g} events/s")
    print(json.dumps(out))
    for rs in ways.values():
        for r in rs:
            r.close()


if __name__ == "__main__":
    main()
