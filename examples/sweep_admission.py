"""What admission limit per server keeps the p99 of admitted requests under the SLO, and how much traffic does it shed?
C3 (two servers behind a load balancer) under a load ramp, every limit of a small set on both servers, many repetitions
each, all in one launch.

``("server_max_in_service", server)`` gives a row's server an admission limit: a request that arrives while the limit
is in service there is shed at the door (DESIGN.md §3.12).  With ``streams = repetition index`` repetition k of every
limit sees the same users and arrivals, so the limits are compared on the same traffic.  Prints, per load and limit,
the shed fraction, the goodput (completions per second) and the p99 of the admitted requests, and per load the limit
that sheds least while meeting the SLO.

    python examples/sweep_admission.py [--reps N] [--horizon S] [--slo-ms MS] [--dry-run]
"""
import argparse
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, SweepSpec, flatten  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=200, help="repetitions per (load, limit)")
ap.add_argument("--horizon", type=int, default=60, help="simulated seconds")
ap.add_argument("--slo-ms", type=float, default=60.0, help="p99 objective for admitted requests, ms")
ap.add_argument("--dry-run", action="store_true", help="build the grid and check its rows; run nothing")
args = ap.parse_args()
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = args.horizon
flat = flatten(payload)
base = float(flat.pod.users_mean)
users = base * np.array([2.0, 4.0, 6.0, 8.0])
limits = np.array([0, 2, 4, 8, 16])                   # 0: no limit
R, L, C = args.reps, len(users), len(limits)
load, lim, rep = (g.ravel() for g in np.meshgrid(np.arange(L), np.arange(C), np.arange(R), indexing="ij"))
cols = {("users_mean",): users[load]}
cols.update({("server_max_in_service", s): limits[lim].astype(float) for s in flat.server_ids})
if args.dry_run:
    spec = SweepSpec(flat, len(rep), cols)
    print(f"{len(rep)} rows: {L} loads x {C} limits x {R} repetitions, {spec.n_columns} columns; one launch")
    sys.exit(0)
sweep = SweepRunner(flat, len(rep), cols, seed=5, streams=rep)
res = sweep.run()
into = flat.edge_ids.index(next(e["id"] for e in payload["topology_graph"]["edges"] if e["target"] == flat.lb_id))
print(f"{len(rep)} replicas in one launch, {args.horizon} s each: {L} loads x limits {limits.tolist()} x {R} repetitions, "
      f"repetition k on stream k; SLO p99 of admitted requests < {args.slo_ms:g} ms")
for k, u in enumerate(users):
    best = None
    for c, m in enumerate(limits):
        rows = np.flatnonzero((load == k) & (lim == c))
        arrived = res.edge_sent[rows, into].astype(float) - res.edge_dropped[rows, into]
        shed = res.server_rejected[rows].sum(axis=1) / np.maximum(arrived, 1.0)
        good = res.stats["completed"][rows] / float(args.horizon)
        p99 = float(np.nanmean(res.stats["p99"][rows]))
        meets = p99 < args.slo_ms / 1e3
        print(f"users {u:6.0f}  limit {('none' if m == 0 else str(m)):>4s}: shed {100 * shed.mean():6.2f} %, goodput "
              f"{good.mean():8.1f} req/s, p99 admitted {1e3 * p99:8.2f} ms{'  meets the SLO' if meets else ''}")
        if meets and (best is None or shed.mean() < best[1]):
            best = (m, shed.mean())
    print(f"users {u:6.0f}: " + ("no limit meets the SLO" if best is None else
                                  f"the least-shedding limit meeting the SLO is {'none' if best[0] == 0 else best[0]} "
                                  f"({100 * best[1]:.2f} % shed)"))
sweep.close()
