"""Where the time goes as load grows: C3 (two single-core servers behind a load balancer, 20 requests per minute per
user) over a sweep of users_mean up to near saturation, a few hundred Monte-Carlo repetitions per point.

``SweepRunner(occupancy=True)`` integrates on the device, per replica, the requests in each state over the whole run:
blocked on a server's RAM, queued for its core, on the core, in I/O, and on each edge.  Prints, per load point, the p95
latency and each state's share of the request-seconds and seconds per generated request (``results.breakdown``): the
CPU-wait share grows as the single core of each server saturates, while the time on the core and in I/O per request
stays put.

    python examples/sweep_time_breakdown.py [--replicas N] [--horizon S]
"""
import argparse
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, flatten  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--replicas", type=int, default=500, help="repetitions per load point")
ap.add_argument("--horizon", type=int, default=60, help="simulated seconds")
args = ap.parse_args()
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = args.horizon
flat = flatten(payload)
users = np.array([400.0, 1200.0, 2000.0, 2600.0, 2900.0])        # the two single-core servers saturate near 3 000
point = np.repeat(np.arange(len(users)), args.replicas)
sweep = SweepRunner(flat, len(point), {("users_mean",): users[point]}, seed=7, occupancy=True)
res = sweep.run()
states = ("ram_wait", "cpu_wait", "cpu", "io", "transit")
print(f"{len(point)} replicas, {args.horizon} s each; time per request split by state (both servers, every edge)")
print(f"{'users_mean':>10} {'p95 [ms]':>9} " + " ".join(f"{s:>17}" for s in states))
for k, u in enumerate(users):
    sel = np.flatnonzero(point == k)
    b = res.breakdown(sel)
    share = {s: np.nansum([x for x, st in zip(b["share"], b["state"]) if st == s]) for s in states}
    per_rq = {s: np.nansum([x for x, st in zip(b["per_request"], b["state"]) if st == s]) for s in states}
    p95 = 1e3 * float(np.nanmean(res.stats["p95"][sel]))
    print(f"{u:10.0f} {p95:9.2f} " + " ".join(f"{100 * share[s]:6.1f} % {1e3 * per_rq[s]:6.2f} ms" for s in states))
