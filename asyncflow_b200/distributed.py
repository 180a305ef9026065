"""Multi-GPU: replicas shard by range, one collective at the end.

Replicas are independent and AF-RNG is keyed by the GLOBAL replica id, so a sweep
over G GPUs is G disjoint replica ranges with zero traffic during simulation and
results that do not depend on G.  The only exchange is one all-gather of each
rank's *summary block* (the device-reduced latency histogram plus totals; a few
KB) over NCCL/NVLink -- BASELINE.json north_star, SURVEY.md 8e.  The reference
has nothing to mirror here (single process, single thread).

One process per GPU (``torchrun``); ``torch.distributed`` is plumbing only.  The
same code runs on the ``gloo`` backend for the CPU-tier tests.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import _capi as K
from .results import SweepResults, hist_percentiles, pad_dist_bins

N_TOTALS = 8     # completed, generated, events, replicas, overflowed, ticks, reserved x2


def shard_bounds(n_replicas: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous replica range of ``rank``: sizes differ by at most one."""
    base, extra = divmod(int(n_replicas), int(world))
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


def summary_block(stats: np.ndarray, reduced_hist: np.ndarray | None) -> tuple[np.ndarray, np.ndarray]:
    """(int64 block, float64 block) a rank contributes to the final all-gather."""
    ints = np.zeros(K.AF_HIST_BINS + N_TOTALS, dtype=np.int64)
    if reduced_hist is not None:
        ints[: K.AF_HIST_BINS] = reduced_hist.astype(np.int64)
    t = ints[K.AF_HIST_BINS:]
    t[0] = int(stats["completed"].sum())
    t[1] = int(stats["generated"].sum())
    t[2] = int(stats["n_events"].sum())
    t[3] = int(stats.shape[0])
    t[4] = int(((stats["flags"] & (K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW)) != 0).sum())
    t[5] = int(stats["n_ticks"].sum())
    flts = np.array([float(stats["lat_sum"].sum()), float(stats["lat_sumsq"].sum()),
                     float(stats["lat_min"][stats["completed"] > 0].min()) if (stats["completed"] > 0).any() else np.inf,
                     float(stats["lat_max"].max()) if stats.shape[0] else 0.0], dtype=np.float64)
    return ints, flts


@dataclass
class GlobalSummary:
    histogram: np.ndarray      # [AF_HIST_BINS] summed over every rank
    completed: int
    generated: int
    events: int
    replicas: int
    overflowed: int
    lat_sum: float
    lat_min: float
    lat_max: float
    per_rank_completed: list[int]

    @property
    def mean_latency(self) -> float:
        return self.lat_sum / max(self.completed, 1)

    def percentile(self, q: float) -> float:
        """numpy-'linear' percentile of ALL completions, read off the merged histogram."""
        return float(hist_percentiles(self.histogram, q))


def all_gather_summary(ints: np.ndarray, flts: np.ndarray, device: str | None = None) -> GlobalSummary:
    """One all-gather of the summary blocks (NCCL on GPUs, gloo on CPU); works without
    an initialised process group (world = 1)."""
    import torch  # noqa: PLC0415
    import torch.distributed as dist  # noqa: PLC0415

    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        all_i, all_f = ints[None, :], flts[None, :]
    else:
        dev = device or ("cuda" if dist.get_backend() == "nccl" else "cpu")
        ti = torch.from_numpy(ints).to(dev)
        tf = torch.from_numpy(flts).to(dev)
        gi = [torch.empty_like(ti) for _ in range(world)]
        gf = [torch.empty_like(tf) for _ in range(world)]
        dist.all_gather(gi, ti)
        dist.all_gather(gf, tf)
        all_i = torch.stack(gi).cpu().numpy()
        all_f = torch.stack(gf).cpu().numpy()
    tot = all_i[:, K.AF_HIST_BINS:]
    return GlobalSummary(
        histogram=all_i[:, : K.AF_HIST_BINS].sum(axis=0).astype(np.int64),
        completed=int(tot[:, 0].sum()), generated=int(tot[:, 1].sum()), events=int(tot[:, 2].sum()),
        replicas=int(tot[:, 3].sum()), overflowed=int(tot[:, 4].sum()),
        lat_sum=float(all_f[:, 0].sum()), lat_min=float(all_f[:, 2].min()), lat_max=float(all_f[:, 3].max()),
        per_rank_completed=[int(x) for x in tot[:, 0]])


BAND_FIELDS = ("band_count", "band_sum", "band_sumsq", "lat_hist", "lat_sum_hi", "lat_sum_lo", "group_size", "dist_hist")


def all_reduce_bands(res: SweepResults, device: str | None = None) -> SweepResults:
    """Sum the band rows of ``res`` -- the per-tick sampled-metric bands, the per-window latency bands, the per-tick
    distribution bands and the group sizes a rank's shard holds -- over every rank, in place, with one all-reduce:
    afterwards each rank holds the bands of the whole sweep, as :meth:`SweepResults.concatenate` of every rank's
    results would.  The unsigned sums travel as int64; their modular addition gives the same bits.  Ranks may size
    their distribution bins differently (each launch by its own rows): one all-reduce of the largest bin count comes
    first, and every rank pads to it.  Works without an initialised process group."""
    import torch  # noqa: PLC0415
    import torch.distributed as dist  # noqa: PLC0415

    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    if world == 1 or not any(getattr(res, k) is not None for k in BAND_FIELDS):
        return res
    dev = device or ("cuda" if dist.get_backend() == "nccl" else "cpu")
    if res.dist_hist is not None:
        b = torch.tensor([res.dist_hist.shape[-1]], dtype=torch.int64, device=dev)
        dist.all_reduce(b, op=dist.ReduceOp.MAX)
        res.dist_hist = pad_dist_bins(res.dist_hist, int(b.item()))
    present = [(k, getattr(res, k)) for k in BAND_FIELDS if getattr(res, k) is not None]
    flat = np.concatenate([a.astype(np.uint64).view(np.int64).ravel() if a.dtype != np.int64 else a.ravel()
                           for _, a in present])
    t = torch.from_numpy(flat).to(dev)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    out = t.cpu().numpy()
    at = 0
    for k, a in present:
        v = out[at:at + a.size].reshape(a.shape)
        at += a.size
        setattr(res, k, v.view(np.uint64).astype(a.dtype) if a.dtype != np.int64 else v.copy())
    return res


def run_sharded(runner, *, with_histogram: bool = True):
    """Run ``runner`` (a :class:`~asyncflow_b200.runner.SweepRunner` built for the WHOLE sweep)
    on this rank's replica range and all-gather the summaries.

    One process per GPU (``torchrun``); call ``torch.distributed.init_process_group("nccl")``
    first.  Returns ``(local SweepResults, GlobalSummary)``; the per-replica rows of other
    ranks stay on those ranks -- only the summary block crosses NVLink.
    """
    import torch.distributed as dist  # noqa: PLC0415

    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    begin, end = shard_bounds(runner.n_replicas, rank, world)
    if end <= begin:
        # more ranks than replicas: nothing to launch here, but the collective must still complete
        from . import _capi as K  # noqa: PLC0415
        res = None
        ints, flts = summary_block(np.zeros(0, dtype=K.STATS_DTYPE), None)
        return res, all_gather_summary(ints, flts)
    res = runner.run(begin, end)
    hist = runner.engine().reduced_histogram() if (with_histogram and runner.histogram) else None
    ints, flts = summary_block(res.stats, hist)
    return res, all_gather_summary(ints, flts)
