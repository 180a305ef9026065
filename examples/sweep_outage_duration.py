"""How long can a server be down?  C4 (eight servers behind a load balancer, a network spike on the client->LB edge at
100-160 s) with srv-3 down for one of several durations, ~1 000 Monte-Carlo repetitions each, the outage starting at a
random time per replica in [120, 200) s -- sometimes inside the spike, sometimes after it.

Every replica gets its own event timeline (``("event_start", ...)`` / ``("event_end", ...)`` sweep columns), so the
whole study is ONE launch.  The device sums, per group of rows and one-second window of finish time, the completions
per latency bin (``latency_window_s=1``).  Windows are in simulation time, so a second-by-second table only lines up
across replicas whose outage starts together: each duration has two groups, ``reps`` rows with the outage at 180 s
(printed second by second around it) and ``reps`` rows with a random start (their whole-run p95 next to the fixed
start's).

    python examples/sweep_outage_duration.py [repetitions_per_duration]
"""
import sys
from pathlib import Path

import numpy as np
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from asyncflow_b200 import SweepRunner, flatten  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
durations = np.array([5.0, 15.0, 30.0, 60.0])          # seconds srv-3 stays down
payload = yaml.safe_load((ROOT / "tests" / "scenarios" / "c4_lb8_events.yml").read_text())
flat = flatten(payload)
rng = np.random.default_rng(7)
G = len(durations)
n = 2 * reps * G                                       # per duration: reps rows starting at 180 s, reps at random times
dur = np.repeat(durations, 2 * reps)
random_start = np.tile(np.repeat([False, True], reps), G)
start = np.where(random_start, rng.uniform(120.0, 200.0, n), 180.0)
group = np.repeat(np.arange(G), 2 * reps) * 2 + random_start   # 2 g: fixed start, 2 g + 1: random start
sweep = SweepRunner(flat, n, {("event_start", "ev-srv3-down"): start, ("event_end", "ev-srv3-down"): start + dur},
                    seed=11, bands=group, latency_window_s=1, sampled_bands=False)
res = sweep.run()
sweep.close()
lat = res.group_latency()
print(f"{n} replicas in one launch ({reps} per duration and start kind), {int(res.completed.sum()):,} completions, "
      f"{int(res.overflowed.sum())} overflowed; the spike is on at 100-160 s")
print("srv-3 down from t = 180 s:")
print("  t[s]" + "".join(f" | down {d:3.0f} s: p95 [ms]   rps" for d in durations))
for sec in range(175, 246):
    k = sec - 1                                          # window k holds the finishes in (k, k + 1]
    if k >= lat["t"].size:
        break
    row = f"{int(lat['t'][k]):6d}"
    for g in range(G):
        row += f" | {1e3 * lat['p95'][2 * g, k]:18.2f} {lat['rps'][2 * g, k]:6.1f}"
    print(row)
tot = lat["total"]
print(" whole run, p95 [ms] (fixed start | random start in [120, 200) s):")
for g, d in enumerate(durations):
    print(f"  down {d:3.0f} s: {1e3 * tot['p95'][2 * g]:7.2f} | {1e3 * tot['p95'][2 * g + 1]:7.2f}")
