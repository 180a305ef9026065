"""Common random numbers: is a 1.5 ms parsing step faster than a 2 ms one, and by how much?  C3 (two single-core
servers behind a load balancer) at a few loads, both servers' parsing step at 2 ms (variant A) and at 1.5 ms
(variant B), many repetitions per (load, variant), all in one launch.

``SweepRunner(streams=...)`` gives each row the random stream it draws from.  With ``streams = repetition index``,
repetition k of A and of B see the same users, arrivals, network delays and endpoint choices, so most of the noise
cancels in their difference.  ``results.paired()`` gives the mean difference with its interval and, for comparison,
the interval the same rows would give as independent samples.  Prints, per load, each variant's mean latency and p95,
the paired difference with its interval, and the unpaired interval.

    python examples/sweep_paired_steps.py [--replicas N] [--horizon S]
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
ap.add_argument("--replicas", type=int, default=1000, help="repetitions per (load, variant)")
ap.add_argument("--horizon", type=int, default=10, help="simulated seconds")
args = ap.parse_args()
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c3_lb_two_servers.yml").read_text())
payload["sim_settings"]["total_simulation_time"] = args.horizon
flat = flatten(payload)
users = np.array([600.0, 1500.0, 2400.0])
parse = np.array([0.002, 0.0015])                                   # variant A, variant B
R, V, L = args.replicas, len(parse), len(users)
rep = np.tile(np.arange(R), L * V)                                  # row = (load, variant, repetition)
variant = np.tile(np.repeat(np.arange(V), R), L)
load = np.repeat(np.arange(L), V * R)
cols = {("users_mean",): users[load], ("step_duration", "srv-1", 0, 0): parse[variant],
        ("step_duration", "srv-2", 0, 0): parse[variant]}
sweep = SweepRunner(flat, len(rep), cols, seed=7, streams=rep)
res = sweep.run()
print(f"{len(rep)} replicas in one launch, {args.horizon} s each; parsing step A = 2 ms, B = 1.5 ms; "
      f"{R} repetitions per point, repetition k of A and B on stream k")
for k, u in enumerate(users):
    a = np.flatnonzero((load == k) & (variant == 0))                # ordered by repetition: pairs (a[j], b[j])
    b = np.flatnonzero((load == k) & (variant == 1))
    for what in ("mean", "p95"):
        p = res.paired(what, a, b)
        ma, mb = (res.confidence_interval(what, s)[0] for s in (a, b))
        gain = p["unpaired_half_width"] / p["half_width"] if p["half_width"] > 0 else float("nan")
        print(f"users {u:6.0f} {what:>4}: A {1e3 * ma:8.4f} ms  B {1e3 * mb:8.4f} ms  A - B {1e3 * p['estimate']:8.4f} "
              f"± {1e3 * p['half_width']:.4f} ms paired (corr {p['corr']:.2f}), ± {1e3 * p['unpaired_half_width']:.4f} "
              f"ms unpaired ({gain:.1f}x narrower)")
