"""Per-tick distribution bands around an injected outage: C4 (eight servers behind a load balancer, a network spike on
the client->LB edge at 100-160 s, srv-3 down at 180-240 s) over a few spike sizes x ~1 000 Monte-Carlo repetitions each.

Each spike size is one group of rows, and the device counts per tick how many of the group's replicas hold each value
of srv-1's and srv-2's ready queues (``SweepRunner(dist_series=...)``): one bin per value below 64, 16 log-linear bins
per octave above.  No replica is traced.  Prints, second by second around the outage window, the p5 / p50 / p95 fan
of srv-1's ready queue and the probability that it holds at least K requests, per spike size (tick k is taken at
(k + 1) x sample_period; `group_dist()["t"]` follows get_series' axis, k x sample_period).

    python examples/sweep_outage_dist.py [repetitions_per_size] [K]
"""
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, flatten  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
K = int(sys.argv[2]) if len(sys.argv) > 2 else 4        # below 64 every value is a bin edge
spikes = np.array([0.010, 0.030, 0.060])                # spike_s of ev-spike, seconds
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c4_lb8_events.yml").read_text())
flat = flatten(payload)
n = reps * len(spikes)
size = np.repeat(np.arange(len(spikes)), reps)         # row -> its spike size = its group
sweep = SweepRunner(flat, n, {("spike_delta", "ev-spike"): spikes[size]}, seed=11, bands=size,
                    dist_series=[("ready_queue_len", "srv-1"), ("ready_queue_len", "srv-2")])
res = sweep.run()
d = res.group_dist("ready_queue_len", "srv-1", q=(0.05, 0.5, 0.95), at_least=K)
per_s = int(round(1.0 / flat.sample_period))
print(f"{n} replicas ({reps} per spike size), {int(res.completed.sum()):,} completions, "
      f"{int(res.overflowed.sum())} overflowed; srv-3 is down at 180-240 s")
print("  t[s]" + "".join(f" | spike {1e3 * s:4.0f} ms: srv-1 queue p5/p50/p95  P(queue >= {K})" for s in spikes))
for sec in range(175, 251):
    k = sec * per_s - 1                                   # the tick taken at simulated time t = sec
    if k >= d["n"].shape[1]:
        break
    row = f"{sec:6d}"
    for g in range(len(spikes)):
        p5, p50, p95 = d["q"][g, :, k]
        row += f" | {p5:9.0f} {p50:5.0f} {p95:5.0f}            {d['p_at_least'][g, k]:6.3f}"
    print(row)
