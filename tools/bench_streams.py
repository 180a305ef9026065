"""What a random-stream table costs on the bench workload (``bench.make_workload("c3")``, the sweep ``bench.py`` runs),
on one GPU, alternating settings:

* ``none``      no table: every replica draws as its own id;
* ``identity``  a table with stream i for replica i: the same draws, read from the table;
* ``shared``    streams ``arange(n) % 1000``: a thousand streams, each shared by every thousandth replica (common
                random numbers across the sweep's points).

Each launch is timed with the engine's CUDA events (table and rows resident on the device, as bench.py's ``value``
steps).  Prints the median completions/s per setting, the rate difference of ``identity`` and ``shared`` against
``none``, whether every output of ``identity`` (stats, edge counts, sampled sums and maxima, the reduced latency
histogram) was bit-identical to ``none``'s, and the GPU's name and power limit.

    python tools/bench_streams.py [--replicas N] [--horizon H] [--reps 3]
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
    w = bench.make_workload("c3", a.horizon, a.replicas)
    n = w.replicas
    flat = flatten(w.payload)
    sw = SweepRunner(flat, n, w.columns(flat, np.arange(n, dtype=np.int64), n), seed=bench.SEED, histogram=True,
                     throughput=False)
    eng = sw.engine()
    eng.upload_sweep(sw.spec, 0, row_first=0, row_count=n)
    eng.configure(request_capacity=sw.request_capacity, event_capacity=sw.event_capacity, histogram=True,
                  throughput=False)
    tables = {"none": None, "identity": np.arange(n, dtype=np.uint64), "shared": np.arange(n, dtype=np.uint64) % 1000}

    def launch(key: str):
        eng.upload_streams(tables[key], 0)
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

    keys = list(tables)
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
    identical = digest["identity"] == digest["none"] and len(digest["none"]) == 1
    info = gpu_info()
    print(f"{w.key}: {n} replicas, horizon {w.horizon} s; {info['gpu']}, power limit {info['power_limit']}")
    for k in keys:
        diff = "" if k == "none" else f"  rate {100.0 * (med[k] / med['none'] - 1.0):+.1f} % vs none"
        print(f"  {k:<9s} {med[k]:.4g} completions/s  (median of {len(rate[k])}){diff}")
    print(f"  identity table: every output identical to no table: {identical}")
    print(json.dumps({"config": w.key, "replicas": n, **info, **med, "identity_identical": identical}))
    sw.close()


if __name__ == "__main__":
    main()
