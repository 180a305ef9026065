"""What per-tick bands cost on the bench workload: the same launch with bands off and with G groups (G = 1, 100, 1000
by default), alternating, on one GPU.

Every launch runs the bench's sweep (``bench.make_workload``; rows resident on the device, as bench.py's ``value``
steps) and is timed with the engine's CUDA events.  Group g holds the rows whose index is g modulo G, so every group
is spread over the whole sweep.  Prints, per setting, the median completions/s, its change against bands off (rate)
and the extra device time per launch (time = off / on - 1), then whether every other output (stats, edge counts,
sampled sums and maxima, the reduced latency histogram) was bit-identical to the bands-off launch, and the GPU's name
and power limit.

    python tools/bench_bands.py [--config c3] [--replicas N] [--horizon H] [--groups 1,100,1000] [--reps 3]
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
    ap.add_argument("--groups", default="1,100,1000")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    w = bench.make_workload(a.config, a.horizon, a.replicas)
    n = w.replicas
    flat = flatten(w.payload)
    sw = SweepRunner(flat, n, w.columns(flat, np.arange(n, dtype=np.int64), n), seed=bench.SEED, histogram=True,
                     throughput=False)
    eng = sw.engine()
    eng.upload_sweep(sw.spec, 0, row_first=0, row_count=n)
    settings = [0] + [int(g) for g in a.groups.split(",")]

    def launch(G: int):
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

    launch(0)                                                   # warm-up (allocations)
    for G in settings[1:]:
        launch(G)
    rate = {G: [] for G in settings}
    digest: dict[int, set] = {G: set() for G in settings}
    for rep in range(a.reps):                                   # alternate off / on, direction flipped every rep
        order = settings[1:] if rep % 2 == 0 else settings[1:][::-1]
        for G in order:
            for g in (0, G):
                r, _, d = launch(g)
                rate[g].append(r)
                digest[g].add(d)
    off = float(np.median(rate[0]))
    same = all(digest[G] == digest[0] for G in settings) and len(digest[0]) == 1
    T = int(flat.horizon_s / flat.sample_period)
    info = gpu_info()
    print(f"{w.key}: {n} replicas, horizon {w.horizon} s, {flat.n_series} series, ~{T} ticks; {info['gpu']}, power limit "
          f"{info['power_limit']}")
    print(f"  bands off        {off:.4g} completions/s  (medians of {len(rate[0])} launches off, {a.reps} on)")
    for G in settings[1:]:
        on = float(np.median(rate[G]))
        mb = (G + 1) * (1 + 2 * flat.n_series) * (T + 2) * 8 / 1e6
        print(f"  bands G={G:<6d}  {on:.4g} completions/s  rate {100.0 * (on / off - 1.0):+.1f} %  "
              f"time {100.0 * (off / on - 1.0):+.1f} %  (band rows {mb:.1f} MB)")
    print(f"  every non-band output identical with bands on and off: {same}")
    print(json.dumps({"config": w.key, "replicas": n, **info, "off": off,
                      **{f"G{G}": float(np.median(rate[G])) for G in settings[1:]}, "outputs_identical": same}))
    sw.close()


if __name__ == "__main__":
    main()
