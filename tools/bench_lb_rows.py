"""A fleet-size x algorithm study as one launch against the F x A launches it takes without load-balancer rows.

The grid: C4 (eight servers behind a load balancer; its injected spike and outage left out), fleets 1..8 (the first k
of the load balancer's servers) x {round_robin, least_connection} x ``--reps`` repetitions at ``--users``, repetition k
on stream k.  ``one launch``: one ``SweepRunner`` over every row, with ``("lb_covered", server)`` and ``("lb_algorithm",)``
columns.  ``F x A launches``: one scenario per fleet and algorithm (the reduced payload of ``SweepSpec.payload_for``),
each its own ``SweepRunner`` of ``--reps`` rows.  Both give every row the same outputs (checked: stats and the sent
counts of the edges the fleet keeps).  Prints, for each way, the completions/s over the device time of its launches
(CUDA events) and over the wall clock of the whole study (``run()`` to results, engines already built), and the GPU's
name and power limit.

    python tools/bench_lb_rows.py [--reps 2000] [--users 1600] [--horizon 30] [--rounds 3]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from asyncflow_b200 import SweepRunner, flatten  # noqa: E402
from asyncflow_b200.flatten import SweepSpec  # noqa: E402

ALGOS = ("round_robin", "least_connection")


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
    ap.add_argument("--reps", type=int, default=2000)
    ap.add_argument("--users", type=float, default=1600.0)
    ap.add_argument("--horizon", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c4_lb8_events.yml").read_text())
    payload["sim_settings"]["total_simulation_time"] = a.horizon
    payload["rqs_input"]["avg_active_users"]["mean"] = a.users
    payload.pop("events", None)
    flat = flatten(payload)
    servers = payload["topology_graph"]["nodes"]["load_balancer"]["server_covered"]
    F, A, R = len(servers), len(ALGOS), a.reps
    fleet, algo, rep = (g.ravel() for g in np.meshgrid(np.arange(1, F + 1), np.arange(A), np.arange(R), indexing="ij"))
    cols = {("lb_algorithm",): [ALGOS[x] for x in algo]}
    cols.update({("lb_covered", s): (fleet > j).astype(float) for j, s in enumerate(servers)})
    one = SweepRunner(flat, len(rep), cols, seed=3, streams=rep)
    spec = SweepSpec(flat, len(rep), cols)
    cells = [(f, x) for f in range(1, F + 1) for x in range(A)]
    apart = []
    for f, x in cells:                      # the reduced scenario of the cell, R rows on streams 0..R-1
        row = int(np.flatnonzero((fleet == f) & (algo == x))[0])
        apart.append(SweepRunner(spec.payload_for(payload, row), R, None, seed=3, streams=np.arange(R)))

    def run_one():
        t = time.perf_counter()
        res = one.run()
        return res, time.perf_counter() - t, one.last_ms[0] / 1e3

    def run_apart():
        t, dev, out = time.perf_counter(), 0.0, []
        for r in apart:
            out.append(r.run())
            dev += r.last_ms[0] / 1e3
        return out, time.perf_counter() - t, dev

    run_one()
    run_apart()                             # warm-up: engines, allocations
    wall = {"one": [], "apart": []}
    dev = {"one": [], "apart": []}
    for k in range(a.rounds):               # alternate, direction flipped every round
        for key in (("one", "apart") if k % 2 == 0 else ("apart", "one")):
            res, w, d = run_one() if key == "one" else run_apart()
            wall[key].append(w)
            dev[key].append(d)
            if key == "one":
                res_one = res
            else:
                res_apart = res
    same = True
    for (f, x), r in zip(cells, res_apart):
        rows = np.flatnonzero((fleet == f) & (algo == x))
        keep = [flat.edge_ids.index(e) for e in r.flat.edge_ids]
        for fld in ("generated", "completed", "n_events", "lat_sum", "lat_max"):
            same = same and np.array_equal(res_one.stats[fld][rows], r.stats[fld])
        same = same and np.array_equal(res_one.edge_sent[rows][:, keep], r.edge_sent)
    done = float(res_one.stats["completed"].sum())
    info = gpu_info()
    out = {"replicas": int(len(rep)), "cells": len(cells), "horizon": a.horizon, "users": a.users,
           "one_launch_device": done / float(np.median(dev["one"])), "one_launch_end_to_end": done / float(np.median(wall["one"])),
           "fxa_launches_device": done / float(np.median(dev["apart"])),
           "fxa_launches_end_to_end": done / float(np.median(wall["apart"])), "identical": bool(same), **info}
    print(f"{len(rep)} replicas ({F} fleets x {A} algorithms x {R}), horizon {a.horizon} s, users {a.users:g}; "
          f"{info['gpu']}, power limit {info['power_limit']}")
    for key, name in (("one_launch", "one launch"), ("fxa_launches", f"{len(cells)} launches")):
        print(f"  {name:<12s} {out[key + '_device']:.4g} completions/s device, {out[key + '_end_to_end']:.4g} end to end")
    print(f"  speed-up of one launch: {out['one_launch_device'] / out['fxa_launches_device']:.2f}x device, "
          f"{out['one_launch_end_to_end'] / out['fxa_launches_end_to_end']:.2f}x end to end; outputs identical: {same}")
    print(json.dumps(out))
    one.close()
    for r in apart:
        r.close()


if __name__ == "__main__":
    main()
