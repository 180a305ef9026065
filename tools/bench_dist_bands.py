"""What per-tick distribution bands cost on the bench workload: the same launch with them off and on, over two series
(both servers' ready queues) or every sampled series, with G groups (G = 1, 100 by default), alternating, on one GPU.

Every launch runs the bench's sweep (``bench.make_workload``; rows resident on the device, as bench.py's ``value``
steps) and is timed with the engine's CUDA events, which include the zeroing of the rows and the scan.  Group g holds
the rows whose index is g modulo G.  The per-tick sampled bands stay off, so "on" adds the distribution bands alone.
Prints, per setting, the median completions/s, its change against off (rate) and the extra device time per launch
(time = off / on - 1), then whether every other output (stats, edge counts, sampled sums and maxima, the reduced
latency histogram) was bit-identical to the off launch, and the GPU's name and power limit.

    python tools/bench_dist_bands.py [--config c3] [--replicas N] [--horizon H] [--groups 1,100] [--reps 3]
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
    ap.add_argument("--config", default="c3", choices=["c2", "c3", "c4", "c5"])
    ap.add_argument("--replicas", type=int, default=None)
    ap.add_argument("--horizon", type=int, default=None)
    ap.add_argument("--groups", default="1,100")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    w = bench.make_workload(a.config, a.horizon, a.replicas)
    n = w.replicas
    flat = flatten(w.payload)
    sw = SweepRunner(flat, n, w.columns(flat, np.arange(n, dtype=np.int64), n), seed=bench.SEED, histogram=True,
                     throughput=False)
    eng = sw.engine()
    eng.upload_sweep(sw.spec, 0, row_first=0, row_count=n)
    both = [3 * i for i in range(min(flat.n_servers, 2))]      # the servers' ready queues
    every = list(range(flat.n_series))
    off_key = ("off", 0)
    settings = [off_key] + [(name, int(g)) for name in ("2", "all") for g in a.groups.split(",")]
    eng.configure_bands(sampled=False)

    def launch(key):
        name, G = key
        eng.configure_dist_bands(None if name == "off" else (both if name == "2" else every))
        eng.upload_bands(None if G == 0 else (np.arange(n) % G).astype(np.uint32), 0, G or None)
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
        return float(st["completed"].sum()) / (ms / 1e3), ms, h.hexdigest()

    for key in settings:                                        # warm-up (allocations)
        launch(key)
    rate = {key: [] for key in settings}
    digest: dict[tuple, set] = {key: set() for key in settings}
    for rep in range(a.reps):                                   # alternate off / on, direction flipped every rep
        order = settings[1:] if rep % 2 == 0 else settings[1:][::-1]
        for key in order:
            for k in (off_key, key):
                r, _, d = launch(k)
                rate[k].append(r)
                digest[k].add(d)
    off = float(np.median(rate[off_key]))
    same = all(digest[k] == digest[off_key] for k in settings) and len(digest[off_key]) == 1
    T = int(flat.horizon_s / flat.sample_period)
    info = gpu_info()
    print(f"{w.key}: {n} replicas, horizon {w.horizon} s, {flat.n_series} series, ~{T} ticks; {info['gpu']}, power limit "
          f"{info['power_limit']}")
    print(f"  dist bands off            {off:.6g} completions/s  (medians of {len(rate[off_key])} launches off, {a.reps} on)")
    for key in settings[1:]:
        on = float(np.median(rate[key]))
        print(f"  dist {key[0]:>3s} series G={key[1]:<5d} {on:.6g} completions/s  rate {100.0 * (on / off - 1.0):+.2f} %  "
              f"time {100.0 * (off / on - 1.0):+.2f} %  (launches {', '.join(f'{r:.4g}' for r in rate[key])})")
    print(f"  every other output identical with distribution bands on and off: {same}")
    print(json.dumps({"config": w.key, "replicas": n, **info, "off": off,
                      **{f"{k[0]}_G{k[1]}": float(np.median(rate[k])) for k in settings[1:]}, "outputs_identical": same}))
    sw.close()


if __name__ == "__main__":
    main()
