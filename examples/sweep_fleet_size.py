"""How many servers does the service need, and does least-connections beat round-robin there?  C4 (eight single-core
servers behind a load balancer; its injected spike and outage left out) at a few loads, every fleet of 1 to 8 servers
(the first k of the load balancer's) under both algorithms, many repetitions each, all in one launch.

``("lb_covered", server)`` takes a server out of the load balancer's pool row by row, ``("lb_algorithm",)`` picks the
row's algorithm.  With ``streams = repetition index`` repetition k of every fleet and algorithm sees the same users,
arrivals and network delays, so ``results.paired()`` compares round-robin and least-connections on the same traffic.
Prints, per load, the smallest fleet whose p95 latency interval lies below the SLO under round-robin, and the paired
p95 difference round-robin - least-connections at that fleet.

    python examples/sweep_fleet_size.py [--reps N] [--horizon S] [--slo-ms MS]
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
ap.add_argument("--reps", type=int, default=200, help="repetitions per (load, fleet, algorithm)")
ap.add_argument("--horizon", type=int, default=30, help="simulated seconds")
ap.add_argument("--slo-ms", type=float, default=40.0, help="p95 latency objective, ms")
args = ap.parse_args()
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c4_lb8_events.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = args.horizon
payload.pop("events", None)
flat = flatten(payload)
servers = payload["topology_graph"]["nodes"]["load_balancer"]["server_covered"]
users = np.array([800.0, 1600.0, 3200.0])
algos = ["round_robin", "least_connection"]
R, F, A, L = args.reps, len(servers), len(algos), len(users)
# row = (load, fleet, algorithm, repetition)
load, fleet, algo, rep = (g.ravel() for g in np.meshgrid(np.arange(L), np.arange(1, F + 1), np.arange(A), np.arange(R),
                                                         indexing="ij"))
cols = {("users_mean",): users[load], ("lb_algorithm",): [algos[a] for a in algo]}
cols.update({("lb_covered", s): (fleet > j).astype(float) for j, s in enumerate(servers)})
sweep = SweepRunner(flat, len(rep), cols, seed=11, streams=rep)
res = sweep.run()
print(f"{len(rep)} replicas in one launch, {args.horizon} s each: {L} loads x fleets 1..{F} x {A} algorithms x {R} "
      f"repetitions, repetition k on stream k; SLO p95 < {args.slo_ms:g} ms")
for k, u in enumerate(users):
    best = None
    for f in range(1, F + 1):
        rr = np.flatnonzero((load == k) & (fleet == f) & (algo == 0))      # ordered by repetition: pairs (rr[j], lc[j])
        _, _, hi = res.confidence_interval("p95", rr)
        if hi < args.slo_ms / 1e3:
            best = f
            break
    if best is None:
        print(f"users {u:6.0f}: no fleet of up to {F} servers meets the SLO")
        continue
    rr = np.flatnonzero((load == k) & (fleet == best) & (algo == 0))
    lc = np.flatnonzero((load == k) & (fleet == best) & (algo == 1))
    p = res.paired("p95", rr, lc)
    print(f"users {u:6.0f}: smallest fleet {best} (p95 {1e3 * res.confidence_interval('p95', rr)[0]:.3f} ms); "
          f"round_robin - least_connection p95 {1e3 * p['estimate']:+.4f} ± {1e3 * p['half_width']:.4f} ms paired "
          f"(± {1e3 * p['unpaired_half_width']:.4f} ms unpaired)")
