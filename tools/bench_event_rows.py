"""What per-replica event timelines cost on the c4 workload (``bench.make_workload("c4")``: a network spike and an
outage of srv-3, swept spike amplitude x client-LB RTT), on one GPU, alternating settings:

* ``scenario``  the bench's sweep as it is: every replica reads the scenario's one timeline (``spike_delta`` column);
* ``rows``      the same sweep with ``("event_start", ...)`` / ``("event_end", ...)`` columns equal to the scenario's
                times: every replica reads its own timeline row, with the same marks (the amplitude folded in);
* ``random``    every event drawn per replica (the spike starting in [60, 200) s for 10-90 s, the outage in
                [120, 240) s for 5-60 s): every replica reads its own, different timeline row.

A ``--horizon`` other than the scenario's 300 s scales every event time by horizon / 300.

Each launch is timed with the engine's CUDA events (rows resident on the device, as bench.py's ``value`` steps).
Prints the median completions/s per setting, the rate difference of ``rows`` and ``random`` against ``scenario``,
whether every output of ``rows`` (stats, edge counts, sampled sums and maxima, the reduced latency histogram) was
bit-identical to ``scenario``'s, and the GPU's name and power limit.

    python tools/bench_event_rows.py [--replicas N] [--horizon H] [--reps 3]
"""

from __future__ import annotations

import argparse
import hashlib
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402

from asyncflow_b200 import SweepRunner, flatten  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (x.strip() for x in out.split(",", 1))
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": f"unknown ({e})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=None)
    ap.add_argument("--horizon", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    w = bench.make_workload("c4", a.horizon, a.replicas)
    n = w.replicas
    s = w.horizon / 300.0                                      # the scenario's times are for its 300 s: scale them
    for e in w.payload["events"]:
        e["start"]["t_start"], e["end"]["t_end"] = e["start"]["t_start"] * s, e["end"]["t_end"] * s
    flat = flatten(w.payload)
    base = w.columns(flat, np.arange(n, dtype=np.int64), n)
    same = dict(base)
    for e in flat.events:
        same[("event_start", e.event_id)] = np.full(n, e.t_start)
        same[("event_end", e.event_id)] = np.full(n, e.t_end)
    rng = np.random.default_rng(5)
    rand = dict(base)
    for eid, lo, hi, dlo, dhi in (("ev-spike", 60.0, 200.0, 10.0, 90.0), ("ev-srv3-down", 120.0, 240.0, 5.0, 60.0)):
        start = rng.uniform(lo * s, hi * s, n)
        rand[("event_start", eid)] = start
        rand[("event_end", eid)] = start + rng.uniform(dlo * s, dhi * s, n)
    runners = {k: SweepRunner(flat, n, cols, seed=bench.SEED, histogram=True, throughput=False)
               for k, cols in (("scenario", base), ("rows", same), ("random", rand))}
    eng = runners["scenario"].engine()

    def launch(key: str):
        sw = runners[key]
        eng.upload_sweep(sw.spec, 0, row_first=0, row_count=n)
        eng.configure(request_capacity=sw.request_capacity, event_capacity=sw.event_capacity, histogram=True,
                      throughput=False)
        eng.run(bench.SEED, 0, n)
        eng.sync()
        ms = eng.last_run_ms()[0]
        st = eng.stats()
        sent, dropped = eng.edge_counts()
        ssum, smax = eng.sampled()
        h = hashlib.sha256()
        for x in (st, sent, dropped, ssum, smax, eng.reduced_histogram()):
            h.update(np.ascontiguousarray(x).tobytes())
        return float(st["completed"].sum()) / (ms / 1e3), h.hexdigest()

    keys = list(runners)
    for k in keys:                                              # warm-up (allocations)
        launch(k)
    rate = {k: [] for k in keys}
    digest: dict[str, set] = {k: set() for k in keys}
    for rep in range(a.reps):                                   # alternate, direction flipped every rep
        for k in (keys if rep % 2 == 0 else keys[::-1]):
            r, d = launch(k)
            rate[k].append(r)
            digest[k].add(d)
    med = {k: float(np.median(rate[k])) for k in keys}
    identical = digest["rows"] == digest["scenario"] and len(digest["scenario"]) == 1
    info = gpu_info()
    print(f"{w.key}: {n} replicas, horizon {w.horizon} s; {info['gpu']}, power limit {info['power_limit']}")
    for k in keys:
        diff = "" if k == "scenario" else f"  rate {100.0 * (med[k] / med['scenario'] - 1.0):+.1f} % vs scenario"
        print(f"  {k:<9s} {med[k]:.4g} completions/s  (median of {len(rate[k])}){diff}")
    print(f"  rows equal to the scenario's timeline: every output identical: {identical}")
    print(json.dumps({"config": w.key, "replicas": n, **info, **med, "rows_identical": identical}))
    runners["scenario"].close()


if __name__ == "__main__":
    main()
