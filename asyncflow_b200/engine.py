"""Thin object wrapper over the C ABI (``include/asyncflow_b200.h``).

Owns one ``af_engine`` (one CUDA device).  All arrays that cross the boundary
are caller-visible numpy arrays; device memory belongs to the C side.
"""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as K
from .flatten import FlatScenario, SweepSpec


class EngineError(RuntimeError):
    pass


class Engine:
    def __init__(self, device: int = 0) -> None:
        self._lib = K.load()
        h = C.c_void_p()
        rc = self._lib.af_engine_create(int(device), C.byref(h))
        if rc != 0:
            msg = self._lib.af_last_error(None).decode()
            raise K.EngineUnavailable(f"af_engine_create({device}) failed ({rc}): {msg}")
        self._h = h
        self.device = int(device)
        self.flat: FlatScenario | None = None
        self._n = 0
        self._opt = K.AfOptions(0, 0, 0, 0, 1, 1, 0, 0)
        self._keep: list = []
        self._band_groups = self._run_band_groups = 0
        self._band_opt = K.AfBandOptions(1, 0)
        self._run_band_opt = (1, 0)
        self._dist_n = self._run_dist_n = 0

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc: int, what: str) -> None:
        if rc != 0:
            raise EngineError(f"{what} failed ({rc}): {self._lib.af_last_error(self._h).decode()}")

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.af_engine_destroy(self._h)
            self._h = None

    def __del__(self) -> None:  # pragma: no cover - best effort
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    def __enter__(self) -> "Engine":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    # ------------------------------------------------------------------ inputs
    def configure(self, *, event_capacity: int = 0, request_capacity: int = 0,
                  warps_per_block: int = 0, blocks_per_sm: int = 0, histogram: bool = True,
                  throughput: bool = True, trace_replicas: int = 0,
                  trace_clock_capacity: int = 0) -> None:
        self._opt = K.AfOptions(event_capacity, request_capacity, warps_per_block, blocks_per_sm,
                                int(histogram), int(throughput), trace_replicas, trace_clock_capacity)
        self._check(self._lib.af_engine_configure(self._h, C.byref(self._opt)), "af_engine_configure")

    def set_mode(self, mode: str | int) -> None:
        """Pass structure of :meth:`run`: ``"two_pass"`` (thread-per-replica kernel, flagged replicas re-run one per
        warp), ``"auto"`` (two_pass when the launch is large enough for it to pay off, else one replica per warp),
        ``"warp"`` or ``"lane"`` (one kernel only) -- ``af_engine_set_mode``."""
        m = K.MODES[mode] if isinstance(mode, str) else int(mode)
        self._check(self._lib.af_engine_set_mode(self._h, m), "af_engine_set_mode")

    def upload(self, flat: FlatScenario) -> None:
        self._check(self._lib.af_scenario_upload(self._h, C.byref(flat.pod)), "af_scenario_upload")
        self.flat = flat

    def upload_sweep(self, spec: SweepSpec | None, first_replica: int = 0, *, row_first: int = 0,
                     row_count: int | None = None) -> None:
        """Rows ``[row_first, row_first+row_count)`` of ``spec`` describe replicas starting at ``first_replica``: its
        columns (``af_sweep_upload``) and, when it sweeps event times, the same rows' timelines (``af_timeline_upload``;
        otherwise the timeline rows are cleared).  ``None`` clears both."""
        if spec is None:
            self._check(self._lib.af_sweep_upload(self._h, None, 0), "af_sweep_upload")
            self._check(self._lib.af_timeline_upload(self._h, None, 0), "af_timeline_upload")
            return
        sw, keep = spec.pod(row_first, row_count)
        self._check(self._lib.af_sweep_upload(self._h, C.byref(sw), int(first_replica)), "af_sweep_upload")
        tl, keep_tl = spec.timeline_pod(row_first, row_count)
        self._check(self._lib.af_timeline_upload(self._h, None if tl is None else C.byref(tl), int(first_replica)),
                    "af_timeline_upload")
        del keep, keep_tl

    def upload_streams(self, streams, first_replica: int = 0) -> None:
        """Replica ``first_replica + i`` draws its random numbers as stream ``streams[i]`` (u64) from the next run on;
        every other replica as its own id.  ``None`` clears the table (``af_streams_upload``)."""
        if streams is None:
            self._check(self._lib.af_streams_upload(self._h, None, 0, 0), "af_streams_upload")
            return
        s = np.ascontiguousarray(streams, dtype=np.uint64)
        self._check(self._lib.af_streams_upload(self._h, s.ctypes.data if s.size else None, s.size, int(first_replica)),
                    "af_streams_upload")

    # ------------------------------------------------------------------ run
    def run(self, seed: int, replica_begin: int, replica_end: int) -> None:
        self._check(self._lib.af_run(self._h, int(seed), int(replica_begin), int(replica_end)), "af_run")
        self._n = int(replica_end) - int(replica_begin)
        self._run_band_groups = self._band_groups
        self._run_band_opt = (self._band_opt.sampled, self._band_opt.latency_window_s)
        self._run_dist_n = self._dist_n

    def sync(self) -> None:
        self._check(self._lib.af_sync(self._h), "af_sync")

    def last_run_ms(self) -> tuple[float, float]:
        a, b = C.c_float(), C.c_float()
        self._check(self._lib.af_last_run_ms(self._h, C.byref(a), C.byref(b)), "af_last_run_ms")
        return a.value, b.value

    def selftest_rng(self, kind: int, n: int, *, seed: int, replica: int, dist: int = 0, mean: float = 0.0,
                     sigma: float = 0.0, hop: int = 1) -> tuple[np.ndarray, np.ndarray]:
        """AF-RNG known-answer hook (``af_selftest_rng``): ``n`` device draws of ``kind`` as two f64 arrays."""
        a, b = np.empty(n, dtype=np.float64), np.empty(n, dtype=np.float64)
        self._check(self._lib.af_selftest_rng(self._h, int(seed), int(replica), int(kind), int(dist), float(mean),
                                              float(sigma), int(hop), int(n), a.ctypes.data, b.ctypes.data), "af_selftest_rng")
        return a, b

    def last_run_passes(self) -> dict:
        """What the last run did: which kernels, the lane pass's occupancy and pool sizes, replicas per pass."""
        p = K.AfRunPasses()
        self._check(self._lib.af_last_run_passes(self._h, C.byref(p)), "af_last_run_passes")
        return {k: int(getattr(p, k)) for k, _ in K.AfRunPasses._fields_}

    @property
    def launch_count(self) -> int:
        return int(self._lib.af_launch_count(self._h))

    # ------------------------------------------------------------------ outputs
    def stats(self, out: np.ndarray | None = None) -> np.ndarray:
        out = np.empty(self._n, dtype=K.STATS_DTYPE) if out is None else out
        self._check(self._lib.af_fetch_stats(self._h, out.ctypes.data, self._n), "af_fetch_stats")
        return out

    def edge_counts(self, sent: np.ndarray | None = None,
                    dropped: np.ndarray | None = None) -> tuple[np.ndarray, np.ndarray]:
        ne = self.flat.n_edges
        sent = np.empty((self._n, ne), dtype=np.uint32) if sent is None else sent
        dropped = np.empty((self._n, ne), dtype=np.uint32) if dropped is None else dropped
        self._check(self._lib.af_fetch_edge_counts(self._h, sent.ctypes.data, dropped.ctypes.data, self._n),
                    "af_fetch_edge_counts")
        return sent, dropped

    def server_rejected(self, out: np.ndarray | None = None) -> np.ndarray:
        """Requests each server shed at its admission limit, ``[n, n_servers]`` -- ``af_fetch_server_rejected``."""
        out = np.empty((self._n, self.flat.n_servers), dtype=np.uint32) if out is None else out
        self._check(self._lib.af_fetch_server_rejected(self._h, out.ctypes.data, self._n), "af_fetch_server_rejected")
        return out

    def server_expired(self, out: np.ndarray | None = None) -> np.ndarray:
        """Requests each server dropped past its deadline, ``[n, n_servers]`` -- ``af_fetch_server_expired``."""
        out = np.empty((self._n, self.flat.n_servers), dtype=np.uint32) if out is None else out
        self._check(self._lib.af_fetch_server_expired(self._h, out.ctypes.data, self._n), "af_fetch_server_expired")
        return out

    def late(self, out: np.ndarray | None = None) -> np.ndarray:
        """Completions later than the client timeout, ``[n]`` -- ``af_fetch_late``."""
        out = np.empty(self._n, dtype=np.uint32) if out is None else out
        self._check(self._lib.af_fetch_late(self._h, out.ctypes.data, self._n), "af_fetch_late")
        return out

    def throttled(self, out: np.ndarray | None = None) -> np.ndarray:
        """Requests each site throttled at its rate limit, ``[n, n_servers + 1]`` (column ``n_servers``: the load
        balancer) -- ``af_fetch_throttled``."""
        out = np.empty((self._n, self.flat.n_servers + 1), dtype=np.uint32) if out is None else out
        self._check(self._lib.af_fetch_throttled(self._h, out.ctypes.data, self._n), "af_fetch_throttled")
        return out

    def histograms(self) -> np.ndarray:
        out = np.empty((self._n, K.AF_HIST_BINS), dtype=np.uint32)
        self._check(self._lib.af_fetch_histograms(self._h, out.ctypes.data, self._n), "af_fetch_histograms")
        return out

    def throughput(self, out: np.ndarray | None = None) -> np.ndarray:
        out = np.empty((self._n, self.flat.horizon_s), dtype=np.uint32) if out is None else out
        self._check(self._lib.af_fetch_throughput(self._h, out.ctypes.data, self._n), "af_fetch_throughput")
        return out

    def sampled(self, sums: np.ndarray | None = None,
                maxima: np.ndarray | None = None) -> tuple[np.ndarray, np.ndarray]:
        ns = self.flat.n_series
        sums = np.empty((self._n, ns), dtype=np.uint64) if sums is None else sums
        maxima = np.empty((self._n, ns), dtype=np.uint32) if maxima is None else maxima
        self._check(self._lib.af_fetch_sampled(self._h, sums.ctypes.data, maxima.ctypes.data, self._n),
                    "af_fetch_sampled")
        return sums, maxima

    def reduced_histogram(self) -> np.ndarray:
        """Sum of all replicas' latency histograms, reduced on the device (``[AF_HIST_BINS]`` u64)."""
        out = np.empty(K.AF_HIST_BINS, dtype=np.uint64)
        self._check(self._lib.af_reduce_histograms(self._h, out.ctypes.data), "af_reduce_histograms")
        return out

    def upload_bands(self, groups: np.ndarray | None, first_replica: int = 0, n_groups: int | None = None) -> None:
        """Per-tick bands from the next run on: ``groups[i]`` = group of replica ``first_replica + i`` (``None``: bands
        off), ``n_groups`` groups (default: the largest group + 1) -- ``af_bands_upload``.  Replicas without an entry
        contribute nothing."""
        if groups is None:
            self._check(self._lib.af_bands_upload(self._h, None, 0, 0, 0), "af_bands_upload")
            self._band_groups = 0
            return
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        if n_groups is None:
            n_groups = int(g.max()) + 1 if g.size else 0
        self._check(self._lib.af_bands_upload(self._h, g.ctypes.data, g.size, int(first_replica), n_groups),
                    "af_bands_upload")
        self._band_groups = n_groups

    def configure_bands(self, *, sampled: bool = True, latency_window_s: int = 0) -> None:
        """Which bands the uploaded groups accumulate from the next run on: the per-tick sampled-metric bands
        (:meth:`bands`) and / or per-window latency bands of ``latency_window_s`` whole seconds (0: off;
        :meth:`latency_bands`) -- ``af_bands_configure``."""
        opt = K.AfBandOptions(int(bool(sampled)), int(latency_window_s))
        self._check(self._lib.af_bands_configure(self._h, C.byref(opt)), "af_bands_configure")
        self._band_opt = opt

    def configure_dist_bands(self, series) -> None:
        """Per-tick distribution bands of the sampled series ``series`` (indices in the order of :meth:`sampled`; empty
        or ``None``: off) over the uploaded groups from the next run on (:meth:`dist_bands`) --
        ``af_dist_bands_configure``."""
        s = np.ascontiguousarray([] if series is None else series, dtype=np.int32)
        self._check(self._lib.af_dist_bands_configure(self._h, s.ctypes.data if s.size else None, int(s.size)),
                    "af_dist_bands_configure")
        self._dist_n = int(s.size)

    def configure_occupancy(self, on: bool = True, frac_bits: int = 32) -> None:
        """Occupancy integrals from the next run on (:meth:`occupancy`): per replica, the request-seconds spent in each
        state in fixed point with ``frac_bits`` fraction bits -- ``af_occupancy_configure``."""
        opt = K.AfOccupancyOptions(int(bool(on)), int(frac_bits))
        self._check(self._lib.af_occupancy_configure(self._h, C.byref(opt)), "af_occupancy_configure")

    def occupancy(self, out: np.ndarray | None = None) -> tuple[np.ndarray, int]:
        """Occupancy integrals of the last run: ``([n, 5 n_servers + n_edges] u64, f)`` -- the column layout of
        ``af_fetch_occupancy``, ``value / 2**f`` request-seconds (MB-seconds for ``ram_mb``)."""
        flat = self.flat
        out = np.empty((self._n, 5 * flat.n_servers + flat.n_edges), dtype=np.uint64) if out is None else out
        f = C.c_int32()
        self._check(self._lib.af_fetch_occupancy(self._h, out.ctypes.data, self._n, C.byref(f)), "af_fetch_occupancy")
        return out, int(f.value)

    def dist_bands(self) -> np.ndarray:
        """Distribution bands of the last run: ``[G, n_dist, T, n_bins]`` u32 -- per group, selected series, tick and
        value bin (``results.gauge_bin_edges``), the replicas that contribute the tick with a value in the bin
        (``af_fetch_dist_bands``)."""
        T, B = C.c_uint64(), C.c_uint32()
        self._check(self._lib.af_fetch_dist_bands(self._h, None, 0, C.byref(T), C.byref(B)), "af_fetch_dist_bands")
        rows = self._run_band_groups * self._run_dist_n
        out = np.empty((self._run_band_groups, self._run_dist_n, T.value, B.value), dtype=np.uint32)
        if rows and T.value:
            self._check(self._lib.af_fetch_dist_bands(self._h, out.ctypes.data, T.value, C.byref(T), C.byref(B)),
                        "af_fetch_dist_bands")
        return out

    def latency_bands(self) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Latency bands of the last run: ``(hist [G, W, AF_HIST_BINS] u64, sum_hi [G, W] u64, sum_lo [G, W] u64)`` --
        per group and window, the completions per latency bin and the two words of their latencies' 32.32 fixed-point
        sum, ``sum_hi * 2**32 + sum_lo`` (``af_fetch_latency_bands``)."""
        G, w = self._run_band_groups, self._run_band_opt[1]
        cap = -(-int(self.flat.horizon_s) // max(int(w), 1))
        hist = np.empty((G, cap, K.AF_HIST_BINS), dtype=np.uint64)
        hi = np.empty((G, cap), dtype=np.uint64)
        lo = np.empty((G, cap), dtype=np.uint64)
        n = C.c_uint64()
        self._check(self._lib.af_fetch_latency_bands(self._h, hist.ctypes.data, hi.ctypes.data, lo.ctypes.data, cap,
                                                     C.byref(n)), "af_fetch_latency_bands")
        W = n.value
        return hist[:, :W], hi[:, :W], lo[:, :W]

    def bands(self) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Bands of the last run: ``(count [G, T] u32, sum [G, S, T] u64, sumsq [G, S, T] u64)`` -- per group, series
        (the order of :meth:`sampled`) and tick, the replicas that contribute the tick, the sum of their values and
        of their squares (``af_fetch_bands``)."""
        flat = self.flat
        cap = int(flat.horizon_s / flat.sample_period) + 2
        G, S = self._run_band_groups, flat.n_series
        count = np.empty((G, cap), dtype=np.uint32)
        s = np.empty((G, S, cap), dtype=np.uint64)
        sq = np.empty((G, S, cap), dtype=np.uint64)
        n = C.c_uint64()
        self._check(self._lib.af_fetch_bands(self._h, count.ctypes.data, s.ctypes.data, sq.ctypes.data, cap, C.byref(n)),
                    "af_fetch_bands")
        T = n.value
        return count[:, :T].copy(), s[:, :, :T].copy(), sq[:, :, :T].copy()

    def trace_clocks(self, local_replica: int) -> np.ndarray:
        cap = max(1, self._opt.trace_clock_capacity)
        out = np.empty((cap, 2), dtype=np.float64)
        n = C.c_uint64()
        self._check(self._lib.af_fetch_trace_clocks(self._h, int(local_replica), out.ctypes.data, cap, C.byref(n)),
                    "af_fetch_trace_clocks")
        return out[: n.value].copy()

    def trace_series(self, local_replica: int) -> np.ndarray:
        """``[n_series, n_ticks]`` sampled values (see ``af_fetch_sampled`` for the series order)."""
        flat = self.flat
        cap = int(flat.horizon_s / flat.sample_period) + 2
        out = np.empty((flat.n_series, cap), dtype=np.uint32)
        n = C.c_uint64()
        self._check(self._lib.af_fetch_trace_series(self._h, int(local_replica), out.ctypes.data, cap, C.byref(n)),
                    "af_fetch_trace_series")
        return out[:, : n.value].copy()
