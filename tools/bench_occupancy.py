"""What occupancy integrals cost on the bench workload: the same launch with them off and on, alternating, on one GPU.

Every launch runs the bench's sweep (``bench.make_workload``; rows resident on the device, as bench.py's ``value``
steps) and is timed with the engine's CUDA events.  "On" uses the fraction bits ``SweepRunner(occupancy=True)`` picks
for the sweep.  Prints the median completions/s off and on, the change (rate) and the extra device time per launch
(time = off / on - 1), whether every other output (stats, edge counts, sampled sums and maxima, the reduced latency
histogram) was bit-identical to the off launch, and the GPU's name and power limit, read in the same run.

    python tools/bench_occupancy.py [--config c3] [--replicas N] [--horizon H] [--reps 5]
"""

from __future__ import annotations

import argparse
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import bench  # noqa: E402
from bench_dist_bands import gpu_info  # noqa: E402

from asyncflow_b200 import SweepRunner, flatten  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=["c2", "c3", "c4", "c5"])
    ap.add_argument("--replicas", type=int, default=None)
    ap.add_argument("--horizon", type=int, default=None)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    w = bench.make_workload(a.config, a.horizon, a.replicas)
    n = w.replicas
    flat = flatten(w.payload)
    sw = SweepRunner(flat, n, w.columns(flat, np.arange(n, dtype=np.int64), n), seed=bench.SEED, histogram=True,
                     throughput=False, occupancy=True)
    eng = sw.engine()
    eng.upload_sweep(sw.spec, 0, row_first=0, row_count=n)

    def launch(on: bool):
        eng.configure_occupancy(on, sw.occ_frac_bits)
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

    launch(False)                                               # warm-up (allocations)
    launch(True)
    rate: dict[bool, list] = {False: [], True: []}
    digest: dict[bool, set] = {False: set(), True: set()}
    for rep in range(a.reps):                                   # alternate off / on, direction flipped every rep
        for on in ((False, True) if rep % 2 == 0 else (True, False)):
            r, d = launch(on)
            rate[on].append(r)
            digest[on].add(d)
    off, on = float(np.median(rate[False])), float(np.median(rate[True]))
    same = digest[False] == digest[True] and len(digest[False]) == 1
    occ, f = eng.occupancy()
    info = gpu_info()
    print(f"{w.key}: {n} replicas, horizon {w.horizon} s, {occ.shape[1]} occupancy columns, f = {f}; {info['gpu']}, "
          f"power limit {info['power_limit']}")
    print(f"  occupancy off  {off:.6g} completions/s  (launches {', '.join(f'{r:.4g}' for r in rate[False])})")
    print(f"  occupancy on   {on:.6g} completions/s  rate {100.0 * (on / off - 1.0):+.2f} %  time "
          f"{100.0 * (off / on - 1.0):+.2f} %  (launches {', '.join(f'{r:.4g}' for r in rate[True])})")
    print(f"  every other output identical with occupancy on and off: {same}")
    print(json.dumps({"config": w.key, "replicas": n, **info, "frac_bits": f, "off": off, "on": on,
                      "rate_change": on / off - 1.0, "outputs_identical": same}))
    sw.close()


if __name__ == "__main__":
    main()
