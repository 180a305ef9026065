"""Results: the OUT side of the drop-in boundary.

The reference hands its run to ``ResultsAnalyzer(client=, servers=, edges=,
settings=)`` (reference ``metrics/analyzer.py:51-58``), which reads only
duck-typed attributes: ``client.rqs_clock`` (objects with ``.start`` /
``.finish``), ``server.server_config.id`` + ``server.enabled_metrics``,
``edge.edge_config.id`` + ``edge.enabled_metrics`` and
``settings.total_simulation_time`` / ``sample_period_s`` (``analyzer.py:77-140``;
proved by ``tests/unit/metrics/test_analyzer.py:34-126``).

* :class:`ReplicaResults` carries the full trace of ONE materialised replica and
  answers the analyzer's getters itself (same keys, same arithmetic), and
  :meth:`ReplicaResults.to_reference_analyzer` builds the reference's *real*
  ``ResultsAnalyzer`` from holders when the ``asyncflow`` package is importable,
  so its matplotlib plots work unchanged.
* :class:`SweepResults` is the Monte-Carlo summary over many replicas
  (per-replica counters, exact mean/std/min/max, histogram percentiles).
"""

from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import Any

import numpy as np

from . import _capi as K
from .flatten import FlatScenario

SERVER_SERIES = ("ready_queue_len", "event_loop_io_sleep", "ram_in_use")
EDGE_SERIES = "edge_concurrent_connection"
LATENCY_ORDER = ("total_requests", "mean", "median", "std_dev", "p95", "p99", "min", "max")
#: the occupancy integrals' states of a server, in column order (``af_fetch_occupancy``); an edge's one state
OCC_SERVER_STATES = ("ram_wait", "cpu_wait", "cpu", "io", "ram_mb")
OCC_EDGE_STATE = "transit"
#: the occupancy state whose count a sampled gauge reads
GAUGE_STATE = {"ready_queue_len": "cpu_wait", "event_loop_io_sleep": "io", "ram_in_use": "ram_mb",
               "edge_concurrent_connection": "transit"}


def hist_percentiles(hist: np.ndarray, q: float, *, lo: np.ndarray | None = None,
                     hi: np.ndarray | None = None) -> np.ndarray:
    """numpy-'linear' percentile ``q`` of the completions each latency histogram counts (``hist[..., AF_HIST_BINS]``,
    the log-linear bins of the engine): the two order statistics around ``q / 100 * (n - 1)``, each placed inside its
    bin by its rank among the bin's counts, interpolated linearly.  NaN where a histogram is empty.  Returns
    ``hist.shape[:-1]``.

    ``lo`` / ``hi`` (``hist.shape[:-1]``): each histogram's exact smallest and largest latency (a replica's ``lat_min``
    / ``lat_max``).  The end bins also count the latencies clamped into them, so with these given bin 0 spans
    ``[min(edge(0), lo), edge(1))`` and the last bin ``[edge(B - 1), max(edge(B), hi)]`` -- the engine's per-replica
    ``p50`` / ``p95`` / ``p99``.  Without them every bin keeps its own edges (histograms summed over replicas)."""
    h = np.asarray(hist)
    flat = h.reshape(-1, h.shape[-1])
    out = np.full(flat.shape[0], np.nan)
    lat_lo = np.full(flat.shape[0], np.inf) if lo is None else np.asarray(lo, dtype=np.float64).reshape(-1)
    lat_hi = np.zeros(flat.shape[0]) if hi is None else np.asarray(hi, dtype=np.float64).reshape(-1)
    base = (1023 + K.AF_HIST_MIN_EXP) << K.AF_HIST_SUB_BITS
    for c in range(0, flat.shape[0], 1024):                   # bounded temporaries: [rows, bins] at a time
        cum = np.cumsum(flat[c:c + 1024], axis=1, dtype=np.int64)
        n = cum[:, -1]
        ok = n > 0
        if not ok.any():
            continue
        cum, n = cum[ok], n[ok]
        rows = flat[c:c + 1024][ok]
        r_lo, r_hi = lat_lo[c:c + 1024][ok], lat_hi[c:c + 1024][ok]

        def order_stat(rank: np.ndarray, cum=cum, rows=rows, r_lo=r_lo, r_hi=r_hi) -> np.ndarray:
            b = (cum <= rank[:, None]).sum(axis=1)          # searchsorted(cum, rank, side="right") per row
            b = np.minimum(b, cum.shape[1] - 1)
            before = np.where(b > 0, cum[np.arange(b.size), np.maximum(b - 1, 0)], 0)
            lo = ((b + base).astype(np.uint64) << np.uint64(52 - K.AF_HIST_SUB_BITS)).view(np.float64)
            hi = ((b + 1 + base).astype(np.uint64) << np.uint64(52 - K.AF_HIST_SUB_BITS)).view(np.float64)
            lo = np.where((b == 0) & (r_lo < lo), r_lo, lo)
            hi = np.where((b == cum.shape[1] - 1) & (r_hi > hi), r_hi, hi)
            frac = ((rank - before).astype(np.float64) + 0.5) / rows[np.arange(b.size), b].astype(np.float64)
            return lo + frac * (hi - lo)

        pos = q / 100.0 * (n - 1).astype(np.float64)
        lo = np.floor(pos)
        frac = pos - lo
        lo = lo.astype(np.int64)
        a = order_stat(lo)
        nxt = np.minimum(lo + 1, n - 1)
        b = order_stat(nxt)
        out[c + np.flatnonzero(ok)] = np.where((frac == 0.0) | (lo + 1 >= n), a, a + frac * (b - a))
    return out.reshape(h.shape[:-1])


def gauge_bin_edges(n_bins: int) -> np.ndarray:
    """Lower edges of the first ``n_bins`` value bins of the distribution bands (``af_dist_bands_configure``), ``[n_bins]``
    int64: one bin per value below 64, then 16 log-linear bins per octave (the engine's ``afr::gauge_bin``).  Bin ``b``
    holds the values in ``[edges[b], edges[b + 1])``."""
    b = np.arange(int(n_bins), dtype=np.int64)
    hi = np.maximum(b - 64, 0)
    m = hi // 16 + 6                                          # the octave: index of the highest set bit
    return np.where(b < 64, b, (16 + hi % 16) << np.maximum(m - 4, 0))


def pad_dist_bins(hist: np.ndarray, n_bins: int) -> np.ndarray:
    """Distribution-band counts ``[..., b]`` widened to ``n_bins`` bins with zeros.  A launch sizes its bins by the largest
    value it can see (the request capacity or the largest ``ram_mb`` of its own sweep rows), so shards of one sweep may
    differ in their bin count; the edges (:func:`gauge_bin_edges`) are the same for all, so the extra bins are empty."""
    b = hist.shape[-1]
    if b == n_bins:
        return hist
    if b > n_bins:
        msg = f"cannot narrow {b} distribution bins to {n_bins}"
        raise ValueError(msg)
    out = np.zeros(hist.shape[:-1] + (int(n_bins),), dtype=hist.dtype)
    out[..., :b] = hist
    return out


def occupancy_columns(flat: FlatScenario) -> list[tuple[str, str]]:
    """``(entity_id, state)`` of each occupancy column: five per server (:data:`OCC_SERVER_STATES`), then one per edge."""
    return ([(sid, st) for sid in flat.server_ids for st in OCC_SERVER_STATES]
            + [(eid, OCC_EDGE_STATE) for eid in flat.edge_ids])


def occ_frac_bits(bound: int, horizon_s: int) -> int:
    """The most fraction bits f <= 32 with ``bound * horizon_s * 2**f <= 2**64 - 1`` (the engine's ``afh::occ_frac_bits``):
    ``bound`` is the largest count a column can hold -- the request capacity or the largest ``ram_mb``."""
    bh = max(int(bound), 1) * max(int(horizon_s), 1)
    if bh > (1 << 64) - 1:
        return -1
    return min(32, (((1 << 64) - 1) // bh).bit_length() - 1)


def series_index(flat: FlatScenario, key: Any, entity_id: str) -> int | None:
    """Row of ``(key, entity_id)`` -- as ``ResultsAnalyzer.get_series`` takes them -- in the sampled series, or ``None``
    when the scenario does not sample that metric."""
    name = str(getattr(key, "value", key))
    en = set(flat.enabled_metrics)
    if name in SERVER_SERIES:
        i = list(flat.server_ids).index(entity_id)
        return 3 * i + SERVER_SERIES.index(name) if all(m in en for m in SERVER_SERIES) else None
    if name == EDGE_SERIES:
        e = list(flat.edge_ids).index(entity_id)
        return 3 * flat.n_servers + e if EDGE_SERIES in en else None
    msg = f"unknown sampled metric {name!r}"
    raise KeyError(msg)


def fixed32_mean(sum_hi: np.ndarray, sum_lo: np.ndarray, n: np.ndarray) -> np.ndarray:
    """Mean latency from the two words of a 32.32 fixed-point latency sum (``sum_hi * 2**32 + sum_lo``) over ``n``
    completions; NaN where ``n == 0``."""
    s = np.asarray(sum_hi).astype(np.float64) + np.asarray(sum_lo).astype(np.float64) * 2.0 ** -32
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(n > 0, s / np.maximum(n, 1), np.nan)


class _Name(str):
    """A metric name that also answers ``.value`` like the reference's StrEnum."""

    @property
    def value(self) -> str:
        return str(self)


@dataclass
class ReplicaResults:
    flat: FlatScenario
    clocks: np.ndarray                 # [n, 2] (start, finish), completion order
    series: np.ndarray                 # [n_series, n_ticks]
    generated: int
    edge_sent: dict[str, int]
    edge_dropped: dict[str, int]
    n_events: int
    flags: int
    server_rejected: dict[str, int] = field(default_factory=dict)   # requests each server shed at its admission limit
    server_expired: dict[str, int] = field(default_factory=dict)    # requests each server dropped past its deadline
    late: int = 0                                                    # completions later than the client timeout
    server_throttled: dict[str, int] = field(default_factory=dict)  # requests each server throttled at its rate limit
    lb_throttled: int = 0                                            # requests the load balancer throttled

    # -- analyzer-compatible getters (metrics/analyzer.py:147-262) -------------
    def list_server_ids(self) -> list[str]:
        return list(self.flat.server_ids)

    @property
    def latencies(self) -> np.ndarray:
        return self.clocks[:, 1] - self.clocks[:, 0]

    def get_latency_stats(self) -> dict[str, float]:
        arr = self.latencies
        if arr.size == 0:
            return {}
        return {
            "total_requests": float(arr.size), "mean": float(np.mean(arr)),
            "median": float(np.median(arr)), "std_dev": float(np.std(arr)),
            "p95": float(np.percentile(arr, 95)), "p99": float(np.percentile(arr, 99)),
            "min": float(np.min(arr)), "max": float(np.max(arr)),
        }

    def format_latency_stats(self) -> str:
        st = self.get_latency_stats()
        if not st:
            return "Latency stats: (empty)"
        lines = ["════════ LATENCY STATS ════════"]
        lines += [f"{k.upper():<20} = {st[k]:.6f}" for k in LATENCY_ORDER]
        return "\n".join(lines)

    def get_throughput_series(self, window_s: float | None = None) -> tuple[list[float], list[float]]:
        w = 1.0 if window_s is None else float(window_s)
        finish = np.sort(self.clocks[:, 1])
        end_time = self.flat.horizon_s
        ts: list[float] = []
        rps: list[float] = []
        idx = 0
        cur = w
        while cur <= end_time:                     # analyzer.py:108-125
            j = int(np.searchsorted(finish, cur, side="right"))
            ts.append(cur)
            rps.append((j - idx) / w)
            idx = j
            cur += w
        return ts, rps

    def get_sampled_metrics(self) -> dict[str, dict[str, list[float]]]:
        out: dict[str, dict[str, list[float]]] = defaultdict(dict)
        en = set(self.flat.enabled_metrics)
        if all(m in en for m in SERVER_SERIES):
            for i, sid in enumerate(self.flat.server_ids):
                for m, name in enumerate(SERVER_SERIES):
                    out[name][sid] = self.series[3 * i + m].tolist()
        else:
            for name in SERVER_SERIES:
                if name in en:
                    for sid in self.flat.server_ids:
                        out[name][sid] = []
        if EDGE_SERIES in en:
            base = 3 * self.flat.n_servers
            for j, eid in enumerate(self.flat.edge_ids):
                out[EDGE_SERIES][eid] = self.series[base + j].tolist()
        return out

    def get_metric_map(self, key: Any) -> dict[str, list[float]]:
        return self.get_sampled_metrics().get(str(getattr(key, "value", key)), {})

    def get_series(self, key: Any, entity_id: str) -> tuple[list[float], list[float]]:
        vals = self.get_metric_map(key).get(entity_id, [])
        times = (np.arange(len(vals)) * self.flat.sample_period).tolist()
        return times, vals

    # -- the reference's own analyzer, fed through its duck-typed seam ---------
    def holders(self) -> dict[str, Any]:
        sampled = self.get_sampled_metrics()
        clock = [SimpleNamespace(start=float(a), finish=float(b)) for a, b in self.clocks]
        servers = [
            SimpleNamespace(server_config=SimpleNamespace(id=sid),
                            enabled_metrics={_Name(n): sampled[n][sid] for n in SERVER_SERIES if sid in sampled.get(n, {})})
            for sid in self.flat.server_ids]
        edges = [
            SimpleNamespace(edge_config=SimpleNamespace(id=eid),
                            enabled_metrics=({_Name(EDGE_SERIES): sampled[EDGE_SERIES][eid]}
                                             if eid in sampled.get(EDGE_SERIES, {}) else {}))
            for eid in self.flat.edge_ids]
        settings = SimpleNamespace(total_simulation_time=self.flat.horizon_s,
                                   sample_period_s=self.flat.sample_period)
        return {"client": SimpleNamespace(rqs_clock=clock), "servers": servers, "edges": edges,
                "settings": settings}

    def to_reference_analyzer(self):
        """``asyncflow.metrics.analyzer.ResultsAnalyzer`` over these results (needs the reference package)."""
        from asyncflow.metrics.analyzer import ResultsAnalyzer  # noqa: PLC0415
        return ResultsAnalyzer(**self.holders())


def series_bands(replicas: list[ReplicaResults], key: Any, entity_id: str) -> dict[str, np.ndarray]:
    """Per-tick mean / min / max of one sampled series across fully traced replicas (SURVEY.md 8f-1).

    ``key`` / ``entity_id`` are what ``ResultsAnalyzer.get_series`` takes (``metrics/analyzer.py:239-262``);
    returns ``{"t", "mean", "min", "max", "n"}`` -- the band a dashboard draws around one replica's curve.
    """
    cols = [np.asarray(r.get_series(key, entity_id)[1], dtype=np.float64) for r in replicas]
    cols = [c for c in cols if c.size]
    if not cols:
        z = np.zeros(0)
        return {"t": z, "mean": z, "min": z, "max": z, "n": 0}
    m = min(c.size for c in cols)
    a = np.stack([c[:m] for c in cols])
    return {"t": np.arange(m) * replicas[0].flat.sample_period, "mean": a.mean(axis=0), "min": a.min(axis=0),
            "max": a.max(axis=0), "n": len(cols)}


class SweepResults:
    """Per-replica summaries of a sweep (all arrays have one row per replica)."""

    def __init__(self, flat: FlatScenario, stats: np.ndarray, edge_sent: np.ndarray,
                 edge_dropped: np.ndarray, samp_sum: np.ndarray, samp_max: np.ndarray,
                 throughput: np.ndarray | None = None, histograms: np.ndarray | None = None,
                 replica_begin: int = 0) -> None:
        self.flat = flat
        self.stats = stats
        self.edge_sent = edge_sent
        self.edge_dropped = edge_dropped
        self.samp_sum = samp_sum
        self.samp_max = samp_max
        self.throughput = throughput
        self.histograms = histograms
        self.replica_begin = replica_begin
        # requests each server shed at its admission limit, [n, n_servers] u32 (zeros without limits; DESIGN.md §3.12)
        self.server_rejected = np.zeros((len(stats), flat.n_servers if flat is not None else 0), dtype=np.uint32)
        # requests each server dropped past its deadline, [n, n_servers] u32, and completions later than the client
        # timeout, [n] u32 (zeros without deadlines / a timeout; DESIGN.md §3.13).  Goodput: completed - late
        self.server_expired = np.zeros_like(self.server_rejected)
        self.late = np.zeros(len(stats), dtype=np.uint32)
        # requests each server throttled at its rate limit, [n, n_servers] u32, and the load balancer throttled, [n] u32
        # (zeros without rate limits; DESIGN.md §3.14)
        self.server_throttled = np.zeros_like(self.server_rejected)
        self.lb_throttled = np.zeros(len(stats), dtype=np.uint32)
        self.rows: np.ndarray | None = None      # sweep row of each result row (set by SweepRunner)
        self.streams: np.ndarray | None = None   # random stream of each result row (SweepRunner.stream_ids; set by collect)
        self.traced: list[ReplicaResults] = []    # full clocks + sampled series of the first `trace_replicas` replica ids
        self.exact: np.ndarray | None = None      # rows whose p50/p95/p99 are exact (SweepRunner.exact_percentiles)
        # per-tick bands (SweepRunner(bands=...)): per group g, series j, tick k: replicas that contribute the tick,
        # sum of their values, sum of the squares -- [G, T] u32, [G, n_series, T] u64, [G, n_series, T] u64
        self.band_count: np.ndarray | None = None
        self.band_sum: np.ndarray | None = None
        self.band_sumsq: np.ndarray | None = None
        # per-window latency bands (SweepRunner(latency_window_s=w)): per group g and window k of w seconds, the
        # completions per latency bin [G, W, AF_HIST_BINS] u64 and the two words of their latencies' 32.32 fixed-point
        # sum [G, W] u64; the replicas of each group [G]
        self.lat_window_s: int = 0
        self.lat_hist: np.ndarray | None = None
        self.lat_sum_hi: np.ndarray | None = None
        self.lat_sum_lo: np.ndarray | None = None
        self.group_size: np.ndarray | None = None
        # per-tick distribution bands (SweepRunner(dist_series=[...])): per group g, selected series s (dist_series[s],
        # a (metric, entity_id) key), tick k and value bin b (gauge_bin_edges), the replicas that contribute the tick
        # with a value in the bin -- [G, n_dist, T, n_bins] u32
        self.dist_series: list[tuple[str, str]] = []
        self.dist_hist: np.ndarray | None = None
        # occupancy integrals (SweepRunner(occupancy=True)): per replica and column (occ_columns), the request-seconds
        # in that state over [0, horizon) in fixed point with occ_frac_bits fraction bits -- [n, 5 n_servers + n_edges] u64
        self.occupancy: np.ndarray | None = None
        self.occ_frac_bits: int = 0

    def __len__(self) -> int:
        return int(self.stats.shape[0])

    @property
    def completed(self) -> np.ndarray:
        return self.stats["completed"]

    @property
    def generated(self) -> np.ndarray:
        return self.stats["generated"]

    @property
    def overflowed(self) -> np.ndarray:
        return (self.stats["flags"] & (K.FLAG_EVENT_OVERFLOW | K.FLAG_REQUEST_OVERFLOW | K.FLAG_NOWQ_OVERFLOW)) != 0

    @property
    def mean_latency(self) -> np.ndarray:
        c = np.maximum(self.completed, 1)
        return np.where(self.completed > 0, self.stats["lat_sum"] / c, np.nan)

    @property
    def std_latency(self) -> np.ndarray:
        c = np.maximum(self.completed, 1).astype(np.float64)
        m = self.stats["lat_sum"] / c
        v = np.maximum(self.stats["lat_sumsq"] / c - m * m, 0.0)
        return np.where(self.completed > 0, np.sqrt(v), np.nan)

    def latency_stats(self, i: int) -> dict[str, float]:
        """Same keys as ``ResultsAnalyzer.get_latency_stats`` for replica ``i``;
        median/p95/p99 come from the log-linear histogram (bins <= 1.6 % wide)."""
        s = self.stats[i]
        if s["completed"] == 0:
            return {}
        return {
            "total_requests": float(s["completed"]), "mean": float(self.mean_latency[i]),
            "median": float(s["p50"]), "std_dev": float(self.std_latency[i]),
            "p95": float(s["p95"]), "p99": float(s["p99"]),
            "min": float(s["lat_min"]), "max": float(s["lat_max"]),
        }

    def sampled_mean(self) -> np.ndarray:
        """Mean over ticks of every sampled series, ``[n, n_series]``."""
        t = np.maximum(self.stats["n_ticks"], 1).astype(np.float64)[:, None]
        return self.samp_sum.astype(np.float64) / t

    def _statistic(self, what: Any) -> np.ndarray:
        """A per-replica statistic as f64: ``"mean"`` (latency), ``"p50"``, ``"p95"``, ``"p99"``, ``"completed"``,
        ``"generated"``, ``"lat_min"``, ``"lat_max"``, or any array of one float per result row (e.g. ``time_in(...)``)."""
        if isinstance(what, str):
            if what == "mean":
                return self.mean_latency
            if what in ("p50", "p95", "p99", "completed", "generated", "lat_min", "lat_max"):
                return self.stats[what].astype(np.float64)
            msg = f"unknown statistic {what!r}"
            raise KeyError(msg)
        x = np.asarray(what, dtype=np.float64)
        if x.shape != (len(self),):
            msg = f"a statistic has one value per result row ({len(self)}), got shape {x.shape}"
            raise ValueError(msg)
        return x

    def confidence_interval(self, what: Any = "mean", select: np.ndarray | None = None,
                            level: float = 0.95) -> tuple[float, float, float]:
        """Monte-Carlo estimate over replicas of a per-replica statistic (a name or an array, see :meth:`_statistic`):
        ``(estimate, lo, hi)`` with a normal ``level`` interval on the mean across the selected replicas (reference
        ROADMAP.md:23-27)."""
        x = self._statistic(what)
        if select is not None:
            x = x[select]
        x = x[np.isfinite(x)]
        if x.size == 0:
            return float("nan"), float("nan"), float("nan")
        m = float(x.mean())
        if x.size == 1:
            return m, m, m
        from statistics import NormalDist  # noqa: PLC0415
        z = NormalDist().inv_cdf(0.5 + level / 2.0)
        half = z * float(x.std(ddof=1)) / float(np.sqrt(x.size))
        return m, m - half, m + half

    def paired(self, what: Any, a, b, level: float = 0.95) -> dict[str, Any]:
        """Paired comparison of two alternatives: the mean of ``x[a] - x[b]`` over the pairs ``(a[k], b[k])`` of result
        rows, ``x`` a statistic as :meth:`confidence_interval` takes it.  Rows that share a random stream
        (``SweepRunner(streams=)``) see the same traffic, so their difference cancels most of the noise both share
        (common random numbers).  Pairs
        with a non-finite side are dropped.  Returns ``estimate``, ``lo``, ``hi`` (the normal ``level`` interval of the
        mean difference), ``half_width``, ``n`` (pairs kept), ``corr`` (correlation of the two sides), and
        ``unpaired`` = ``(estimate, lo, hi)`` with ``unpaired_half_width``: the interval of the same difference had the
        two sides been independent (``sqrt(var_a / n + var_b / n)``), so the gain of the pairing is visible."""
        x = self._statistic(what)
        a = np.atleast_1d(np.asarray(a, dtype=np.int64))
        b = np.atleast_1d(np.asarray(b, dtype=np.int64))
        if a.shape != b.shape or a.ndim != 1:
            msg = f"paired: a and b are row-index arrays of one length, got shapes {a.shape} and {b.shape}"
            raise ValueError(msg)
        xa, xb = x[a], x[b]
        keep = np.isfinite(xa) & np.isfinite(xb)
        xa, xb = xa[keep], xb[keep]
        n = int(xa.size)
        nan = float("nan")
        out: dict[str, Any] = {"estimate": nan, "lo": nan, "hi": nan, "half_width": nan, "n": n, "corr": nan,
                               "unpaired": (nan, nan, nan), "unpaired_half_width": nan}
        if n == 0:
            return out
        d = xa - xb
        m = float(d.mean())
        half = half_u = 0.0
        if n > 1:
            from statistics import NormalDist  # noqa: PLC0415
            z = NormalDist().inv_cdf(0.5 + level / 2.0)
            half = z * float(d.std(ddof=1)) / float(np.sqrt(n))
            sa, sb = float(xa.std(ddof=1)), float(xb.std(ddof=1))
            half_u = z * float(np.sqrt((sa * sa + sb * sb) / n))
            if sa > 0.0 and sb > 0.0:
                out["corr"] = float(((xa - xa.mean()) * (xb - xb.mean())).sum() / (n - 1) / (sa * sb))
        mu = float(xa.mean()) - float(xb.mean())
        out.update(estimate=m, lo=m - half, hi=m + half, half_width=half, unpaired=(mu, mu - half_u, mu + half_u),
                   unpaired_half_width=half_u)
        return out

    def summary(self) -> dict[str, float]:
        ok = self.completed > 0
        tot_c = int(self.completed.sum())
        return {
            "replicas": float(len(self)), "completed": float(tot_c),
            "generated": float(self.generated.sum()),
            "events": float(self.stats["n_events"].sum()),
            "mean_latency": float(self.stats["lat_sum"].sum() / max(tot_c, 1)),
            "p50_mean": float(np.nanmean(self.stats["p50"][ok])) if ok.any() else float("nan"),
            "p95_mean": float(np.nanmean(self.stats["p95"][ok])) if ok.any() else float("nan"),
            "p99_mean": float(np.nanmean(self.stats["p99"][ok])) if ok.any() else float("nan"),
            "overflowed": float(self.overflowed.sum()),
        }

    def take(self, index: Any) -> "SweepResults":
        """Rows ``index`` (any numpy index) as a new SweepResults -- e.g. the inverse of a launch order."""
        g = lambda a: None if a is None else a[index]  # noqa: E731
        out = SweepResults(self.flat, self.stats[index], self.edge_sent[index], self.edge_dropped[index],
                           self.samp_sum[index], self.samp_max[index], g(self.throughput), g(self.histograms),
                           self.replica_begin)
        out.traced = self.traced
        out.server_rejected = self.server_rejected[index]
        out.server_expired = self.server_expired[index]
        out.late = self.late[index]
        out.server_throttled = self.server_throttled[index]
        out.lb_throttled = self.lb_throttled[index]
        out.streams = g(self.streams)
        out.band_count, out.band_sum, out.band_sumsq = self.band_count, self.band_sum, self.band_sumsq
        out.lat_window_s, out.lat_hist, out.lat_sum_hi, out.lat_sum_lo = (self.lat_window_s, self.lat_hist,
                                                                          self.lat_sum_hi, self.lat_sum_lo)
        out.group_size = self.group_size
        out.dist_series, out.dist_hist = self.dist_series, self.dist_hist
        out.occupancy, out.occ_frac_bits = g(self.occupancy), self.occ_frac_bits
        return out

    def bands(self, key: Any, entity_id: str) -> dict[str, np.ndarray]:
        """``series_bands`` over this sweep's traced replicas (``SweepRunner(trace_replicas=k)``)."""
        return series_bands(self.traced, key, entity_id)

    def series_index(self, key: Any, entity_id: str) -> int | None:
        """Row of ``(key, entity_id)`` -- as ``ResultsAnalyzer.get_series`` takes them -- in the sampled series, or
        ``None`` when the scenario does not sample that metric."""
        return series_index(self.flat, key, entity_id)

    def group_bands(self, key: Any, entity_id: str, level: float = 0.95) -> dict[str, np.ndarray]:
        """Per group and tick, over the group's replicas, of one sampled series (``SweepRunner(bands=...)``):
        ``{"t", "n", "mean", "std", "lo", "hi"}``, each ``[G, T]`` but ``t`` (``[T]``, seconds).  ``t[k] = k *
        sample_period``, the time axis ``get_series`` gives the same samples (so a band overlays a traced replica's
        curve); the collector takes tick ``k`` at simulated time ``(k + 1) * sample_period``.  ``std`` has
        ddof = 1 and ``lo`` / ``hi`` are a normal ``level`` interval on the mean, as in :meth:`confidence_interval`;
        NaN where fewer than two replicas contribute the tick.  ``key`` / ``entity_id`` as in
        ``ResultsAnalyzer.get_series`` (``metrics/analyzer.py:239-262``), lifted from one replica to a sweep."""
        if self.band_count is None:
            msg = "no bands: run the sweep with SweepRunner(bands=...)"
            raise ValueError(msg)
        j = self.series_index(key, entity_id)
        G, T = self.band_count.shape
        if j is None:
            z = np.zeros((G, 0))
            return {"t": np.zeros(0), "n": self.band_count[:, :0], "mean": z, "std": z, "lo": z, "hi": z}
        n = self.band_count.astype(np.float64)
        s = self.band_sum[:, j, :].astype(np.float64)
        sq = self.band_sumsq[:, j, :].astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = np.where(n > 0, s / n, np.nan)
            var = np.where(n > 1, np.maximum(sq - s * mean, 0.0) / (n - 1.0), np.nan)
            std = np.sqrt(var)
            from statistics import NormalDist  # noqa: PLC0415
            half = NormalDist().inv_cdf(0.5 + level / 2.0) * std / np.sqrt(n)
        return {"t": np.arange(T) * self.flat.sample_period, "n": self.band_count, "mean": mean, "std": std,
                "lo": mean - half, "hi": mean + half}

    def group_dist(self, key: Any, entity_id: str, q=(0.05, 0.25, 0.5, 0.75, 0.95),
                   at_least: int | None = None) -> dict[str, Any]:
        """Per group and tick, the distribution over the group's replicas of one sampled series the sweep selected
        (``SweepRunner(dist_series=[...])``): ``{"t", "n", "min", "max", "q", "p_at_least"}``.  ``t`` (``[T]``,
        seconds) is the axis of :meth:`group_bands`; ``n`` (``[G, T]``) the replicas that contribute the tick; ``q``
        (``[G, len(q), T]``) each quantile as ``numpy.quantile(..., method="inverted_cdf")`` gives it -- the smallest value
        whose cumulative count reaches ``q * n`` -- reported, like ``min`` and ``max`` (``[G, T]``), as the lower edge of
        its bin (:func:`gauge_bin_edges`): the value itself below 64, within 1/16 above.  ``p_at_least`` (``[G, T]``,
        ``None`` without ``at_least``) is the fraction of the contributing replicas whose value is ``>= at_least``;
        exact, as ``at_least`` must be a bin edge.  NaN where no replica contributes the tick."""
        if self.dist_hist is None:
            msg = "no distribution bands: run the sweep with SweepRunner(bands=..., dist_series=[...])"
            raise ValueError(msg)
        want = (str(getattr(key, "value", key)), entity_id)
        if want not in self.dist_series:
            msg = f"{want} is not among the sweep's distribution series {self.dist_series}"
            raise KeyError(msg)
        h = self.dist_hist[:, self.dist_series.index(want)]            # [G, T, n_bins]
        G, T, B = h.shape
        edges = gauge_bin_edges(B + 1)
        p_idx = None
        if at_least is not None:
            p_idx = int(np.searchsorted(edges, at_least))
            if p_idx > B or edges[min(p_idx, B)] != at_least:
                lo, hi = int(edges[max(p_idx - 1, 0)]), (int(edges[p_idx]) if p_idx <= B else None)
                msg = (f"at_least={at_least!r} is not a bin edge: p_at_least is exact at edges only; the neighbouring "
                       f"edges are {lo} and {hi}" if hi is not None else
                       f"at_least={at_least!r} is above the last bin edge {int(edges[B])}")
                raise ValueError(msg)
        cum = np.cumsum(h, axis=-1, dtype=np.int64)
        n = cum[..., -1] if B else np.zeros((G, T), dtype=np.int64)
        ok = n > 0
        val = edges[:B].astype(np.float64)

        def at_rank(r: np.ndarray) -> np.ndarray:     # the value of 0-based order statistic r: the first bin with cum > r
            b = np.minimum((cum <= r[..., None]).sum(axis=-1), max(B - 1, 0))
            return np.where(ok, val[b], np.nan)

        nf = n.astype(np.float64)
        qs = []
        for qq in np.atleast_1d(np.asarray(q, dtype=np.float64)):
            idx = nf * qq - 1.0                          # numpy's inverted_cdf: virtual index n q - 1, up to the next
            prev = np.floor(idx)                         # order statistic unless it is whole
            r = np.where(idx - prev == 0, prev, prev + 1)
            qs.append(at_rank(np.clip(r, 0, np.maximum(nf - 1, 0)).astype(np.int64)))
        first = np.where(ok, val[np.minimum((cum == 0).sum(axis=-1), max(B - 1, 0))], np.nan)
        last = at_rank(np.maximum(n - 1, 0))
        with np.errstate(invalid="ignore", divide="ignore"):
            p = None if p_idx is None else np.where(ok, (n - (cum[..., p_idx - 1] if p_idx else 0)) / nf, np.nan)
        return {"t": np.arange(T) * self.flat.sample_period, "n": n, "min": first, "max": last,
                "q": np.stack(qs, axis=1) if qs else np.zeros((G, 0, T)), "p_at_least": p}

    @property
    def occ_columns(self) -> list[tuple[str, str]]:
        """``(entity_id, state)`` of each column of :attr:`occupancy`."""
        return occupancy_columns(self.flat)

    def _occ_column(self, state: str, entity_id: str) -> int:
        if self.occupancy is None:
            msg = "no occupancy: run the sweep with SweepRunner(occupancy=True)"
            raise ValueError(msg)
        try:
            return self.occ_columns.index((entity_id, state))
        except ValueError:
            msg = f"no occupancy column ({entity_id!r}, {state!r}): states {OCC_SERVER_STATES} of a server, {OCC_EDGE_STATE!r} of an edge"
            raise KeyError(msg) from None

    def time_in(self, state: str, entity_id: str) -> np.ndarray:
        """Per replica, the request-seconds spent in ``state`` at ``entity_id`` over the run, ``[n]`` float64: the
        integral over [0, horizon) of the number of requests in that state (MB-seconds for ``"ram_mb"``).  A server's
        states are ``ram_wait`` (blocked on RAM), ``cpu_wait`` (queued for a core), ``cpu`` (holding a core), ``io`` and
        ``ram_mb``; an edge's is ``transit``."""
        j = self._occ_column(state, entity_id)
        return self.occupancy[:, j].astype(np.float64) * 2.0 ** -self.occ_frac_bits

    def time_average(self, key: Any, entity_id: str) -> np.ndarray:
        """Per replica, the exact time-weighted mean over [0, horizon) of a sampled gauge (``key`` / ``entity_id`` as
        ``ResultsAnalyzer.get_series`` takes them), ``[n]`` float64.  :meth:`sampled_mean` reads the same gauge at the
        collector's ticks only; this counts every change, however short, whether the scenario samples the gauge or not."""
        name = str(getattr(key, "value", key))
        if name not in GAUGE_STATE:
            msg = f"unknown sampled metric {name!r}"
            raise KeyError(msg)
        return self.time_in(GAUGE_STATE[name], entity_id) / float(self.flat.horizon_s)

    def breakdown(self, select: Any = None) -> dict[str, Any]:
        """Where the selected replicas' requests spent their time (``select``: any numpy index of the rows, default all):
        per occupancy column, ``{"entity", "state"}`` (lists), ``"raw"`` (the column summed exactly over the replicas,
        Python ints in units of 2**-f s), ``"seconds"`` (float64), ``"share"`` (of the request-seconds of every column but
        ``ram_mb``; NaN for ``ram_mb``, which counts MB-seconds) and ``"per_request"`` (seconds per generated request).
        ``per_request`` is a finite-horizon Little's-law ratio: the time requests spend in a state over [0, horizon)
        divided by the requests generated, so it includes the time of requests still in flight at the horizon."""
        if self.occupancy is None:
            msg = "no occupancy: run the sweep with SweepRunner(occupancy=True)"
            raise ValueError(msg)
        occ = self.occupancy if select is None else self.occupancy[select]
        occ = occ.reshape(-1, occ.shape[-1])
        hi = (occ >> np.uint64(32)).sum(axis=0, dtype=np.uint64)           # exact while fewer than 2^32 replicas
        lo = (occ & np.uint64(0xFFFFFFFF)).sum(axis=0, dtype=np.uint64)
        raw = [(int(h) << 32) + int(w) for h, w in zip(hi, lo)]
        f = self.occ_frac_bits
        seconds = np.array([r / (1 << f) for r in raw], dtype=np.float64)
        cols = self.occ_columns
        req = np.array([st != "ram_mb" for _, st in cols])
        total = sum(r for r, q in zip(raw, req) if q) / (1 << f)
        gen = self.stats["generated"] if select is None else self.stats["generated"][select]
        n_gen = float(np.asarray(gen, dtype=np.float64).sum())
        with np.errstate(invalid="ignore", divide="ignore"):
            share = np.where(req, seconds / total if total > 0 else np.nan, np.nan)
            per_request = seconds / n_gen if n_gen > 0 else np.full(len(cols), np.nan)
        return {"entity": [e for e, _ in cols], "state": [st for _, st in cols], "raw": raw, "seconds": seconds,
                "share": share, "per_request": per_request}

    def group_latency(self) -> dict[str, Any]:
        """Per group and window, over the group's replicas, the latency and throughput of the completions that
        finish in the window (``SweepRunner(latency_window_s=w)``): ``{"t", "n", "rps", "mean", "p50", "p95",
        "p99", "total"}``.  ``t`` (``[W]``, seconds) are the window ends, the ``ts`` of ``get_throughput_series(w)``
        (``metrics/analyzer.py:187-216``; a last window cut at the horizon ends there); the rest are ``[G, W]``:
        ``n`` completions, ``rps`` = n / (window width x replicas in the group), comparable with one replica's
        throughput series, the mean from the exact fixed-point sums, and histogram percentiles as in
        :attr:`stats`.  ``total`` holds the same statistics (``[G]``) over the whole run, as
        ``get_latency_stats`` (``analyzer.py:83-105``) lifted to a group.  NaN where a window has no completion."""
        if self.lat_hist is None:
            msg = "no latency bands: run the sweep with SweepRunner(bands=..., latency_window_s=w)"
            raise ValueError(msg)
        w, H = int(self.lat_window_s), int(self.flat.horizon_s)
        G, W = self.lat_sum_hi.shape
        start = np.arange(W, dtype=np.float64) * w
        end = np.minimum(start + w, float(H))
        size = np.asarray(self.group_size, dtype=np.float64)

        def stats(hist, hi, lo, width):
            n = hist.sum(axis=-1, dtype=np.uint64)
            with np.errstate(invalid="ignore", divide="ignore"):
                rps = n.astype(np.float64) / (width * size.reshape(size.shape + (1,) * (n.ndim - 1)))
            return {"n": n, "rps": rps, "mean": fixed32_mean(hi, lo, n), "p50": hist_percentiles(hist, 50.0),
                    "p95": hist_percentiles(hist, 95.0), "p99": hist_percentiles(hist, 99.0)}

        out: dict[str, Any] = {"t": end}
        out.update(stats(self.lat_hist, self.lat_sum_hi, self.lat_sum_lo, (end - start)[None, :]))
        out["total"] = stats(self.lat_hist.sum(axis=1, dtype=np.uint64), self.lat_sum_hi.sum(axis=1, dtype=np.uint64),
                             self.lat_sum_lo.sum(axis=1, dtype=np.uint64), float(H))
        return out

    @staticmethod
    def concatenate(parts: list["SweepResults"]) -> "SweepResults":
        f = parts[0]
        cat = lambda xs: None if xs[0] is None else np.concatenate(xs)  # noqa: E731
        out = SweepResults(
            f.flat, np.concatenate([p.stats for p in parts]), np.concatenate([p.edge_sent for p in parts]),
            np.concatenate([p.edge_dropped for p in parts]), np.concatenate([p.samp_sum for p in parts]),
            np.concatenate([p.samp_max for p in parts]), cat([p.throughput for p in parts]),
            cat([p.histograms for p in parts]), f.replica_begin)
        out.server_rejected = np.concatenate([p.server_rejected for p in parts])
        out.server_expired = np.concatenate([p.server_expired for p in parts])
        out.late = np.concatenate([p.late for p in parts])
        out.server_throttled = np.concatenate([p.server_throttled for p in parts])
        out.lb_throttled = np.concatenate([p.lb_throttled for p in parts])
        if all(p.streams is not None for p in parts):
            out.streams = np.concatenate([p.streams for p in parts])
        if all(p.band_count is not None for p in parts):      # integer sums over disjoint replicas: they add exactly
            out.band_count = np.sum([p.band_count for p in parts], axis=0, dtype=np.uint32)
            out.band_sum = np.sum([p.band_sum for p in parts], axis=0, dtype=np.uint64)
            out.band_sumsq = np.sum([p.band_sumsq for p in parts], axis=0, dtype=np.uint64)
        if all(p.lat_hist is not None for p in parts):
            out.lat_window_s = f.lat_window_s
            out.lat_hist = np.sum([p.lat_hist for p in parts], axis=0, dtype=np.uint64)
            out.lat_sum_hi = np.sum([p.lat_sum_hi for p in parts], axis=0, dtype=np.uint64)
            out.lat_sum_lo = np.sum([p.lat_sum_lo for p in parts], axis=0, dtype=np.uint64)
        if all(p.group_size is not None for p in parts):
            out.group_size = np.sum([p.group_size for p in parts], axis=0, dtype=np.int64)
        if all(p.dist_hist is not None for p in parts):       # counts over disjoint replicas: u32 sums, exact below 2^32
            for p in parts:
                if list(p.dist_series) != list(f.dist_series):
                    msg = f"concatenate: distribution bands of different series ({f.dist_series} and {p.dist_series})"
                    raise ValueError(msg)
            out.dist_series = list(f.dist_series)
            B = max(p.dist_hist.shape[-1] for p in parts)        # shards may size their bins differently: pad
            out.dist_hist = np.sum([pad_dist_bins(p.dist_hist, B) for p in parts], axis=0, dtype=np.uint32)
        if all(p.occupancy is not None for p in parts):       # per-replica rows: one scale for all of them
            bits = sorted({p.occ_frac_bits for p in parts})
            if len(bits) > 1:
                msg = f"concatenate: occupancy rows in different fixed-point scales (fraction bits {bits})"
                raise ValueError(msg)
            out.occupancy, out.occ_frac_bits = np.concatenate([p.occupancy for p in parts]), bits[0]
        return out
