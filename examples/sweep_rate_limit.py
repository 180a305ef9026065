"""A gateway rate limit, per-instance rate limits or per-instance concurrency caps: which keeps the p99 of admitted
requests down through overload and an outage, and how much does each shed?  C3 (two servers behind a load balancer) at
several loads around its CPU capacity, with one server down for the middle third of the run or the outage moved to the
horizon's last millisecond, under four policies, many repetitions each, all in one launch:

  none      no limit;
  gateway   the load balancer limited to the fleet's capacity (``("lb_rate",)``, ``("lb_burst",)``);
  instance  each server limited to its own capacity (``("server_rate"|"server_burst", server)``);
  cap       each server capped at a number of requests in service (``("server_max_in_service", server)``, §3.12).

A rate limit sheds on arrival rate and ignores how busy a server is; a cap sheds on work in service (DESIGN.md §3.14).
The outage is an event-time row (``("event_start"|"event_end", event)``, §3.9).  With ``streams = repetition index``
repetition k of every policy sees the same users and arrivals, so ``paired()`` compares each policy with none on the same
traffic.  Prints, per load, outage and policy, the share of requests throttled and shed, the p99 of completions and the
goodput against a client timeout, and the paired difference in goodput against no limit with its 95 % interval.

    python examples/sweep_rate_limit.py [--reps N] [--horizon S] [--burst B] [--cap C] [--timeout-s T] [--dry-run]
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
ap.add_argument("--reps", type=int, default=100, help="repetitions per (load, outage, policy)")
ap.add_argument("--horizon", type=int, default=60, help="simulated seconds")
ap.add_argument("--burst", type=int, default=50, help="the gateway's burst (each instance gets half)")
ap.add_argument("--cap", type=int, default=20, help="requests in service per server under the cap policy")
ap.add_argument("--timeout-s", type=float, default=0.0, help="client timeout T (default: 20 x a request's CPU time)")
ap.add_argument("--dry-run", action="store_true", help="build the grid and check its rows; run nothing")
args = ap.parse_args()
H = args.horizon
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = H
down = payload["topology_graph"]["nodes"]["servers"][1]["id"]
payload["events"] = [{"event_id": "down", "target_id": down, "start": {"kind": "server_down", "t_start": H / 3},
                      "end": {"kind": "server_up", "t_end": 2 * H / 3}}]
flat = flatten(payload)
# the fleet's CPU capacity in requests per second (every endpoint of a server taken as its first)
pod = flat.pod
cpu = [sum(pod.steps[pod.endpoints[s.endpoint_begin].step_begin + k].duration
           for k in range(pod.endpoints[s.endpoint_begin].n_steps)
           if pod.steps[pod.endpoints[s.endpoint_begin].step_begin + k].kind == K.STEP_CPU)
       for s in (pod.servers[i] for i in range(flat.n_servers))]
per_server = [pod.servers[i].cpu_cores / max(cpu[i], 1e-9) for i in range(flat.n_servers)]
capacity = sum(per_server)
T = args.timeout_s or 20.0 * max(cpu)
offered = np.array([0.8, 1.0, 1.2])                    # load / capacity
users = offered * capacity / float(pod.rate_per_user)
POLICIES = ("none", "gateway", "instance", "cap")
OUTAGES = ((H / 3, 2 * H / 3), (H - 1e-3, float(H)))   # the middle third, or the last millisecond
R, L, O, P = args.reps, len(users), len(OUTAGES), len(POLICIES)
load, out, pol, rep = (g.ravel() for g in np.meshgrid(np.arange(L), np.arange(O), np.arange(P), np.arange(R),
                                                       indexing="ij"))
n = len(rep)
half = max(1, args.burst // flat.n_servers)
cols = {("users_mean",): users[load], ("client_timeout",): np.full(n, T),
        ("event_start", "down"): np.array([OUTAGES[o][0] for o in out]),
        ("event_end", "down"): np.array([OUTAGES[o][1] for o in out]),
        ("lb_rate",): np.where(pol == 1, capacity, 0.0), ("lb_burst",): np.full(n, args.burst)}
for i, s in enumerate(flat.server_ids):
    cols[("server_rate", s)] = np.where(pol == 2, per_server[i], 0.0)
    cols[("server_burst", s)] = np.full(n, half)
    cols[("server_max_in_service", s)] = np.where(pol == 3, args.cap, 0)
if args.dry_run:
    spec = SweepSpec(flat, n, cols)
    print(f"{n} rows: {L} loads x {O} outages x {P} policies x {R} repetitions, {spec.n_columns} columns, "
          f"capacity {capacity:.0f} req/s, T = {T:g} s; one launch")
    sys.exit(0)
sweep = SweepRunner(flat, n, cols, seed=5, streams=rep)
res = sweep.run()
gen = np.maximum(res.stats["generated"].astype(np.float64), 1.0)
throttled = (res.server_throttled.sum(axis=1) + res.lb_throttled) / gen
shed = res.server_rejected.sum(axis=1) / gen
good = (res.stats["completed"].astype(np.float64) - res.late) / H
print(f"{n} replicas in one launch, {H} s each: loads {offered.tolist()} x capacity ({capacity:.0f} req/s), "
      f"server {down} down for the middle third or the last millisecond, client timeout T = {1e3 * T:.1f} ms, "
      f"{R} repetitions, repetition k on stream k")
for k in range(L):
    for o in range(O):
        none = np.flatnonzero((load == k) & (out == o) & (pol == 0))
        for c, name in enumerate(POLICIES):
            rows = np.flatnonzero((load == k) & (out == o) & (pol == c))
            p99 = float(np.nanmean(res.stats["p99"][rows]))
            line = (f"load {offered[k]:.1f}x  {'outage' if o == 0 else 'no outage':>9s}  {name:>8s}: throttled "
                    f"{100 * throttled[rows].mean():6.2f} %, shed {100 * shed[rows].mean():6.2f} %, p99 "
                    f"{1e3 * p99:9.2f} ms, goodput {good[rows].mean():8.1f} req/s")
            if c:
                pr = res.paired(good, rows, none)
                line += (f", vs none {pr['estimate']:+8.1f} req/s [{pr['lo']:+.1f}, {pr['hi']:+.1f}] "
                         f"(unpaired +/- {pr['unpaired_half_width']:.1f})")
            print(line)
sweep.close()
