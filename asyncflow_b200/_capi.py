"""ctypes mirror of ``include/asyncflow_b200.h`` and loader of the CUDA library.

The product path is the sm_90a shared library ``asyncflow_b200/_lib/libasyncflow_b200.so``
built by ``__graft_entry__.build()``.  There is NO CPU fallback: if the library
is missing or no CUDA device is usable, :func:`load` / ``af_engine_create``
raise :class:`EngineUnavailable`.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path

AF_ABI_VERSION = 7
AF_HIST_BINS = 4096
AF_HIST_SUB_BITS = 7
AF_HIST_MIN_EXP = -20

DIST = {"poisson": 0, "normal": 1, "log_normal": 2, "exponential": 3, "uniform": 4}
TARGET_CLIENT, TARGET_LB, TARGET_SERVER = 0, 1, 2
STEP_CPU, STEP_IO = 0, 1
LB_NONE, LB_ROUND_ROBIN, LB_LEAST_CONNECTIONS = -1, 0, 1
METRIC_BITS = {"ready_queue_len": 1, "event_loop_io_sleep": 2, "ram_in_use": 4,
               "edge_concurrent_connection": 8}
FIELDS = {
    "users_mean": 0, "users_sigma": 1, "rate_per_user": 2, "edge_mean": 3, "edge_sigma": 4,
    "edge_dropout": 5, "server_cpu_cores": 6, "server_ram_mb": 7, "step_duration": 8,
    "endpoint_ram": 9, "spike_delta": 10,
}
FLAG_EVENT_OVERFLOW, FLAG_REQUEST_OVERFLOW, FLAG_TRACE_TRUNCATED, FLAG_NOWQ_OVERFLOW, FLAG_LB_EMPTY = 1, 2, 4, 8, 16
MODE_AUTO, MODE_WARP, MODE_LANE, MODE_TWO_PASS = 0, 1, 2, 3
SELFTEST_EDGE, SELFTEST_GEN_UNIFORM, SELFTEST_GEN_USERS, SELFTEST_ENDPOINT = 0, 1, 2, 3
SELFTEST_LOG, SELFTEST_EXP = 4, 5
MODES = {"auto": MODE_AUTO, "warp": MODE_WARP, "lane": MODE_LANE, "two_pass": MODE_TWO_PASS}


class AfEdge(C.Structure):
    _fields_ = [("mean", C.c_double), ("sigma", C.c_double), ("dropout", C.c_double),
                ("dist", C.c_int32), ("target_kind", C.c_int32), ("target_index", C.c_int32),
                ("reserved", C.c_int32)]


class AfServer(C.Structure):
    _fields_ = [("cpu_cores", C.c_int32), ("ram_mb", C.c_int32), ("out_edge", C.c_int32),
                ("endpoint_begin", C.c_int32), ("n_endpoints", C.c_int32), ("reserved", C.c_int32)]


class AfEndpoint(C.Structure):
    _fields_ = [("step_begin", C.c_int32), ("n_steps", C.c_int32), ("total_ram", C.c_int32),
                ("reserved", C.c_int32)]


class AfStep(C.Structure):
    _fields_ = [("duration", C.c_double), ("kind", C.c_int32), ("reserved", C.c_int32)]


class AfSpikeMark(C.Structure):
    _fields_ = [("fire_time", C.c_double), ("delta", C.c_double), ("edge", C.c_int32),
                ("reserved", C.c_int32)]


class AfOutageMark(C.Structure):
    _fields_ = [("fire_time", C.c_double), ("lb_edge", C.c_int32), ("down", C.c_int32)]


class AfScenario(C.Structure):
    _fields_ = [
        ("users_dist", C.c_int32), ("window_s", C.c_int32),
        ("users_mean", C.c_double), ("users_sigma", C.c_double), ("rate_per_user", C.c_double),
        ("horizon_s", C.c_int32), ("metrics_mask", C.c_uint32), ("sample_period", C.c_double),
        ("n_edges", C.c_int32), ("n_servers", C.c_int32), ("n_endpoints", C.c_int32),
        ("n_steps", C.c_int32), ("n_lb_edges", C.c_int32), ("lb_algo", C.c_int32),
        ("gen_edge", C.c_int32), ("client_edge", C.c_int32),
        ("n_spike_marks", C.c_int32), ("n_outage_marks", C.c_int32),
        ("edges", C.POINTER(AfEdge)), ("servers", C.POINTER(AfServer)),
        ("endpoints", C.POINTER(AfEndpoint)), ("steps", C.POINTER(AfStep)),
        ("lb_edges", C.POINTER(C.c_int32)), ("spike_marks", C.POINTER(AfSpikeMark)),
        ("outage_marks", C.POINTER(AfOutageMark)),
    ]


class AfSweepColumn(C.Structure):
    _fields_ = [("field", C.c_int32), ("index", C.c_int32)]


class AfSweep(C.Structure):
    _fields_ = [("n_columns", C.c_int32), ("reserved", C.c_int32), ("n_rows", C.c_uint64),
                ("columns", C.POINTER(AfSweepColumn)), ("values", C.POINTER(C.c_double))]


class AfOptions(C.Structure):
    _fields_ = [("event_capacity", C.c_int32), ("request_capacity", C.c_int32),
                ("warps_per_block", C.c_int32), ("blocks_per_sm", C.c_int32),
                ("collect_histogram", C.c_int32), ("collect_throughput", C.c_int32),
                ("trace_replicas", C.c_int32), ("trace_clock_capacity", C.c_int32)]


class AfReplicaStats(C.Structure):
    _fields_ = [("n_events", C.c_uint64), ("generated", C.c_uint32), ("completed", C.c_uint32),
                ("flags", C.c_uint32), ("n_ticks", C.c_uint32), ("peak_events", C.c_uint32),
                ("peak_requests", C.c_uint32), ("lat_sum", C.c_double), ("lat_sumsq", C.c_double),
                ("lat_min", C.c_double), ("lat_max", C.c_double), ("p50", C.c_double),
                ("p95", C.c_double), ("p99", C.c_double)]


import numpy as np  # noqa: E402

STATS_DTYPE = np.dtype([
    ("n_events", "<u8"), ("generated", "<u4"), ("completed", "<u4"), ("flags", "<u4"),
    ("n_ticks", "<u4"), ("peak_events", "<u4"), ("peak_requests", "<u4"),
    ("lat_sum", "<f8"), ("lat_sumsq", "<f8"), ("lat_min", "<f8"), ("lat_max", "<f8"),
    ("p50", "<f8"), ("p95", "<f8"), ("p99", "<f8"),
], align=True)
assert STATS_DTYPE.itemsize == C.sizeof(AfReplicaStats)


class AfRunPasses(C.Structure):
    _fields_ = [("lane_pass", C.c_int32), ("warp_pass", C.c_int32), ("lane_warps_per_sm", C.c_int32),
                ("lane_bytes", C.c_int32), ("lane_events_smem", C.c_int32), ("lane_requests_smem", C.c_int32),
                ("lane_replicas", C.c_uint64), ("warp_replicas", C.c_uint64), ("lane_pool_elems", C.c_int32),
                ("lane_lean", C.c_int32)]


class AfBandOptions(C.Structure):
    _fields_ = [("sampled", C.c_int32), ("latency_window_s", C.c_int32)]


class AfOccupancyOptions(C.Structure):
    _fields_ = [("on", C.c_int32), ("frac_bits", C.c_int32)]


class EngineUnavailable(RuntimeError):
    """The CUDA engine cannot run here (library not built or no usable GPU)."""


LIB_PATH = Path(__file__).resolve().parent / "_lib" / "libasyncflow_b200.so"

EXPORTS = [
    "af_abi_version", "af_engine_create", "af_engine_destroy", "af_last_error",
    "af_engine_configure", "af_scenario_upload", "af_sweep_upload", "af_run", "af_sync",
    "af_last_run_ms", "af_launch_count", "af_fetch_stats", "af_fetch_edge_counts",
    "af_fetch_histograms", "af_fetch_throughput", "af_fetch_sampled", "af_fetch_trace_clocks",
    "af_fetch_trace_series", "af_reduce_histograms", "af_engine_set_mode", "af_last_run_passes",
    "af_selftest_rng", "af_bands_upload", "af_fetch_bands", "af_bands_configure", "af_fetch_latency_bands",
    "af_dist_bands_configure", "af_fetch_dist_bands", "af_occupancy_configure", "af_fetch_occupancy",
]

_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree CUDA library and declare every export of the header."""
    global _lib
    if _lib is not None:
        return _lib
    import os  # noqa: PLC0415
    path = Path(os.environ.get("ASYNCFLOW_B200_LIB", LIB_PATH))   # override: kernel experiments only
    if not path.exists():
        msg = (f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; "
               "g.build()'` (nvcc, sm_90a).  asyncflow_b200 has no CPU fallback.")
        raise EngineUnavailable(msg)
    lib = C.CDLL(str(path))
    vp, u64, i32 = C.c_void_p, C.c_uint64, C.c_int
    lib.af_abi_version.restype = i32
    lib.af_engine_create.argtypes = [i32, C.POINTER(vp)]
    lib.af_engine_destroy.argtypes = [vp]
    lib.af_engine_destroy.restype = None
    lib.af_last_error.argtypes = [vp]
    lib.af_last_error.restype = C.c_char_p
    lib.af_engine_configure.argtypes = [vp, C.POINTER(AfOptions)]
    lib.af_scenario_upload.argtypes = [vp, C.POINTER(AfScenario)]
    lib.af_sweep_upload.argtypes = [vp, C.POINTER(AfSweep), u64]
    lib.af_run.argtypes = [vp, u64, u64, u64]
    lib.af_sync.argtypes = [vp]
    lib.af_last_run_ms.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lib.af_launch_count.argtypes = [vp]
    lib.af_launch_count.restype = u64
    lib.af_fetch_stats.argtypes = [vp, vp, u64]
    lib.af_fetch_edge_counts.argtypes = [vp, vp, vp, u64]
    lib.af_fetch_histograms.argtypes = [vp, vp, u64]
    lib.af_fetch_throughput.argtypes = [vp, vp, u64]
    lib.af_fetch_sampled.argtypes = [vp, vp, vp, u64]
    lib.af_fetch_trace_clocks.argtypes = [vp, u64, vp, u64, C.POINTER(u64)]
    lib.af_fetch_trace_series.argtypes = [vp, u64, vp, u64, C.POINTER(u64)]
    lib.af_reduce_histograms.argtypes = [vp, vp]
    lib.af_engine_set_mode.argtypes = [vp, i32]
    lib.af_last_run_passes.argtypes = [vp, C.POINTER(AfRunPasses)]
    lib.af_selftest_rng.argtypes = [vp, u64, u64, i32, i32, C.c_double, C.c_double, C.c_uint32, u64, vp, vp]
    lib.af_bands_upload.argtypes = [vp, vp, u64, u64, C.c_uint32]
    lib.af_fetch_bands.argtypes = [vp, vp, vp, vp, u64, C.POINTER(u64)]
    lib.af_bands_configure.argtypes = [vp, C.POINTER(AfBandOptions)]
    lib.af_fetch_latency_bands.argtypes = [vp, vp, vp, vp, u64, C.POINTER(u64)]
    lib.af_dist_bands_configure.argtypes = [vp, vp, C.c_int32]
    lib.af_fetch_dist_bands.argtypes = [vp, vp, u64, C.POINTER(u64), C.POINTER(C.c_uint32)]
    lib.af_occupancy_configure.argtypes = [vp, C.POINTER(AfOccupancyOptions)]
    lib.af_fetch_occupancy.argtypes = [vp, vp, u64, C.POINTER(C.c_int32)]
    for name in EXPORTS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("af_abi_version",):
            fn.restype = i32
    if lib.af_abi_version() != AF_ABI_VERSION:
        msg = f"ABI mismatch: library {lib.af_abi_version()} != python {AF_ABI_VERSION}"
        raise EngineUnavailable(msg)
    _lib = lib
    return lib
