"""Per-window latency bands around an injected spike and outage: C4 (eight servers behind a load balancer, a network
spike on the client->LB edge at 100-160 s, srv-3 down at 180-240 s) over a few spike sizes x ~1 000 Monte-Carlo
repetitions each.

Each spike size is one group of rows, and the device sums, per group and one-second window of finish time, the
completions per latency bin and their exact fixed-point latency sum (``SweepRunner(latency_window_s=1)``): no replica
is traced.  Prints, second by second around the spike and the outage, the mean and p95 latency clients saw and the
throughput per replica, per spike size, then the same over the whole run.

    python examples/sweep_outage_latency.py [repetitions_per_size]
"""
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, flatten  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
spikes = np.array([0.010, 0.030, 0.060])                # spike_s of ev-spike, seconds
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c4_lb8_events.yml").read_text())
flat = flatten(payload)
n = reps * len(spikes)
size = np.repeat(np.arange(len(spikes)), reps)         # row -> its spike size = its group
sweep = SweepRunner(flat, n, {("spike_delta", "ev-spike"): spikes[size]}, seed=11, bands=size, latency_window_s=1,
                    sampled_bands=False)
res = sweep.run()
sweep.close()
lat = res.group_latency()
print(f"{n} replicas ({reps} per spike size), {int(res.completed.sum()):,} completions, "
      f"{int(res.overflowed.sum())} overflowed; the spike is on at 100-160 s, srv-3 is down at 180-240 s")
print("  t[s]" + "".join(f" | spike {1e3 * s:3.0f} ms: mean   p95 [ms]   rps" for s in spikes))
for sec in list(range(95, 166)) + list(range(175, 246)):
    k = sec - 1                                          # window k holds the finishes in (k, k + 1]
    if k >= lat["t"].size:
        break
    row = f"{int(lat['t'][k]):6d}"
    for g in range(len(spikes)):
        row += f" | {1e3 * lat['mean'][g, k]:17.2f} {1e3 * lat['p95'][g, k]:7.2f} {lat['rps'][g, k]:6.1f}"
    print(row)
tot = lat["total"]
print(" total" + "".join(f" | {1e3 * tot['mean'][g]:17.2f} {1e3 * tot['p95'][g]:7.2f} {tot['rps'][g]:6.1f}"
                         for g in range(len(spikes))))
