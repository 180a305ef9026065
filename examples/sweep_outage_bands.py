"""Per-tick bands around an injected outage: C4 (eight servers behind a load balancer, a network spike on the
client->LB edge at 100-160 s, srv-3 down at 180-240 s) over a few spike sizes x ~1 000 Monte-Carlo repetitions each.

Each spike size is one group of rows, and the device sums every sampled series per tick over the group's replicas
(``SweepRunner(bands=...)``): no replica is traced, so the cost is a few MB per group, not n_series x n_ticks x 4 B
per replica.  Prints, second by second around the outage window, the mean and 95 % interval of srv-1's ready queue
and of the client->LB connections, per spike size, as the collector read them at that simulated second (tick k is
taken at (k + 1) x sample_period; `group_bands()["t"]` follows get_series' axis, k x sample_period).

    python examples/sweep_outage_bands.py [repetitions_per_size]
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
sweep = SweepRunner(flat, n, {("spike_delta", "ev-spike"): spikes[size]}, seed=11, bands=size)
res = sweep.run()
q = res.group_bands("ready_queue_len", "srv-1")
c = res.group_bands("edge_concurrent_connection", "client-lb")
per_s = int(round(1.0 / flat.sample_period))
print(f"{n} replicas ({reps} per spike size), {int(res.completed.sum()):,} completions, "
      f"{int(res.overflowed.sum())} overflowed; srv-3 is down at 180-240 s")
head = "  t[s]" + "".join(f" | spike {1e3 * s:4.0f} ms: srv-1 ready queue   client->LB conns " for s in spikes)
print(head)
for sec in range(175, 251):
    k = sec * per_s - 1                                   # the tick taken at simulated time t = sec
    if k >= q["mean"].shape[1]:
        break
    row = f"{sec:6d}"
    for g in range(len(spikes)):
        row += (f" | {q['mean'][g, k]:7.3f} [{q['lo'][g, k]:7.3f},{q['hi'][g, k]:7.3f}]"
                f" {c['mean'][g, k]:7.2f} [{c['lo'][g, k]:6.2f},{c['hi'][g, k]:6.2f}]")
    print(row)
