"""How much goodput do server deadlines recover past saturation, and which deadline gives the most?
C3 (two servers behind a load balancer) at two loads past its CPU capacity, clients that give up after T seconds, and
server deadlines of none, T/2 and T on both servers, many repetitions each, all in one launch.

``("server_deadline", server)`` makes a row's server drop a request older than the deadline when it next gets a core,
instead of serving work whose client has given up; ``("client_timeout",)`` counts a completion later than T as late
(DESIGN.md §3.13).  Goodput = completions - late ones.  With ``streams = repetition index`` repetition k of every
deadline sees the same users and arrivals, so ``paired()`` compares each deadline with none on the same traffic.
Prints, per load and deadline, the goodput, the share of requests the servers dropped and the p99, and the paired
difference in goodput against no deadline with its 95 % interval.

    python examples/sweep_deadline.py [--reps N] [--horizon S] [--timeout-s T] [--dry-run]
"""
import argparse
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, SweepSpec, flatten  # noqa: E402
from asyncflow_b200 import _capi as K  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=200, help="repetitions per (load, deadline)")
ap.add_argument("--horizon", type=int, default=60, help="simulated seconds")
ap.add_argument("--timeout-s", type=float, default=0.0, help="client timeout T (default: 20 x a request's CPU time)")
ap.add_argument("--dry-run", action="store_true", help="build the grid and check its rows; run nothing")
args = ap.parse_args()
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = args.horizon
flat = flatten(payload)
# the fleet's CPU capacity in requests per second (every endpoint of a server taken as its first)
pod = flat.pod
cpu = [sum(pod.steps[pod.endpoints[s.endpoint_begin].step_begin + k].duration
           for k in range(pod.endpoints[s.endpoint_begin].n_steps)
           if pod.steps[pod.endpoints[s.endpoint_begin].step_begin + k].kind == K.STEP_CPU)
       for s in (pod.servers[i] for i in range(flat.n_servers))]
capacity = sum(pod.servers[i].cpu_cores / max(cpu[i], 1e-9) for i in range(flat.n_servers))
T = args.timeout_s or 20.0 * max(cpu)
offered = np.array([1.1, 1.3])                         # load / capacity: past saturation
users = offered * capacity / float(pod.rate_per_user)
deadlines = np.array([0.0, T / 2, T])                  # 0: none
R, L, D = args.reps, len(users), len(deadlines)
load, dl, rep = (g.ravel() for g in np.meshgrid(np.arange(L), np.arange(D), np.arange(R), indexing="ij"))
cols = {("users_mean",): users[load], ("client_timeout",): np.full(len(rep), T)}
cols.update({("server_deadline", s): deadlines[dl] for s in flat.server_ids})
if args.dry_run:
    spec = SweepSpec(flat, len(rep), cols)
    print(f"{len(rep)} rows: {L} loads x {D} deadlines x {R} repetitions, {spec.n_columns} columns, T = {T:g} s; "
          "one launch")
    sys.exit(0)
sweep = SweepRunner(flat, len(rep), cols, seed=5, streams=rep)
res = sweep.run()
good = res.stats["completed"].astype(np.float64) - res.late
expired = res.server_expired.sum(axis=1) / np.maximum(res.stats["generated"].astype(np.float64), 1.0)
print(f"{len(rep)} replicas in one launch, {args.horizon} s each: loads {offered.tolist()} x capacity "
      f"({capacity:.0f} req/s), deadlines none / T/2 / T with client timeout T = {1e3 * T:.1f} ms, {R} repetitions, "
      "repetition k on stream k")
for k, u in enumerate(users):
    none = np.flatnonzero((load == k) & (dl == 0))
    for c, d in enumerate(deadlines):
        rows = np.flatnonzero((load == k) & (dl == c))
        p99 = float(np.nanmean(res.stats["p99"][rows]))
        line = (f"load {offered[k]:.1f}x  deadline {('none' if d == 0 else f'{1e3 * d:.1f} ms'):>9s}: goodput "
                f"{good[rows].mean() / args.horizon:8.1f} req/s, expired {100 * expired[rows].mean():6.2f} %, "
                f"p99 {1e3 * p99:9.2f} ms")
        if c:
            pr = res.paired(good / args.horizon, rows, none)
            line += (f", goodput vs none {pr['estimate']:+8.1f} req/s [{pr['lo']:+.1f}, {pr['hi']:+.1f}] "
                     f"(unpaired +/- {pr['unpaired_half_width']:.1f})")
        print(line)
sweep.close()
