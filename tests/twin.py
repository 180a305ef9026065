"""Python face of the CPU twin of both engines (tests/host_twin/af_twin.cpp) -- TEST INFRASTRUCTURE ONLY.

Runs the engines' state machines (asyncflow_b200/csrc/af_lane.cuh and af_core.cuh compiled for the host, one-lane
warp) so CPU-only tests can check event semantics, bands and occupancy against the oracle, and GPU tests the device
against the twin.  Never imported by the product package."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from asyncflow_b200 import _capi as K

_DIR = Path(__file__).resolve().parent / "host_twin"
_SO = _DIR / "_build" / "libaf_twin.so"
_SRC = [_DIR / "af_twin.cpp"] + sorted((_DIR.parent.parent / "asyncflow_b200" / "csrc").glob("*.*h")) \
    + [_DIR.parent.parent / "include" / "asyncflow_b200.h"]
OUTPUTS = ("stats", "sent", "dropped", "hist", "thr", "samp_sum", "samp_max", "trace_clocks", "trace_series",
           "trace_counts")
#: pool splits of the lane engine: every replica by one estimate, each sweep row by its own (as af_run), at random
SPLITS = {"scenario": 0, "rows": 1, "random": 2}
#: words of one latency-band window: AF_HIST_BINS counts, then the latency sum's high and low 32 bits
LAT_ROW = K.AF_HIST_BINS + 2


class TwinLaunch(C.Structure):
    _fields_ = [("sweep_first", C.c_uint64), ("lane_bytes", C.c_int32), ("ev_need", C.c_int32),
                ("split", C.c_int32), ("lean", C.c_int32), ("split_seed", C.c_uint64), ("order", C.c_void_p),
                ("sampled", C.c_int32), ("lat_window", C.c_int32), ("group_of", C.c_void_p),
                ("band_first", C.c_uint64), ("band_n", C.c_uint64), ("n_groups", C.c_uint32), ("n_dist", C.c_int32),
                ("band_rows", C.c_void_p), ("band_from", C.c_void_p), ("lat_rows", C.c_void_p),
                ("lat_from", C.c_void_p), ("dist_series", C.c_void_p), ("dist_capacity", C.c_int32),
                ("occ_bits", C.c_int32), ("dist_rows", C.c_void_p), ("occ", C.c_void_p), ("redo", C.c_void_p),
                ("n_redo", C.c_uint64)]


class TwinOutputs(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in OUTPUTS]


def build() -> Path:
    if os.environ.get("AF_TWIN_SO"):          # experiments: a twin built by hand (e.g. under a sanitizer)
        return Path(os.environ["AF_TWIN_SO"])
    so = _SO
    newest = max(p.stat().st_mtime for p in _SRC)
    if not so.exists() or so.stat().st_mtime < newest:
        so.parent.mkdir(exist_ok=True)
        tmp = so.with_name(f"{so.name}.{os.getpid()}")
        subprocess.run(
            ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-x", "c++",
             "-o", str(tmp), str(_DIR / "af_twin.cpp")], check=True)
        tmp.replace(so)
    return so


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        vp, u64, i32, u32, dbl, s = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32, C.c_double, C.c_char_p
        sc, sw, opt = C.POINTER(K.AfScenario), C.POINTER(K.AfSweep), C.POINTER(K.AfOptions)
        for name, res, args in (
                ("error", s, []),
                ("trace_tick_capacity", i32, [sc]),
                ("ticks", u32, [sc]),
                ("ticks_fit", i32, [sc, s, C.c_int]),
                ("sumsq_fits", i32, [sc, sw, opt, u64, C.POINTER(u64), s, C.c_int]),
                ("lat_fits", i32, [i32, i32, u64, u64, s, C.c_int]),
                ("dist_fits", i32, [sc, sw, opt, vp, i32, u64, u64, C.POINTER(u32), C.POINTER(u32), s, C.c_int]),
                ("occ_fits", i32, [sc, sw, opt, i32, s, C.c_int]),
                ("gauge_bin", u32, [u32]),
                ("fixed32", u64, [dbl]),
                ("hist_bin", i32, [dbl]),
                ("frac_bits", i32, [u64, i32]),
                ("occ_fixed", u64, [dbl, i32]),
                ("hist_percentile", dbl, [vp, u64, dbl, dbl, dbl]),
                ("lean_qualifies", i32, [sc, i32]),
                ("pending_events_estimate", i32, [sc, sw]),
                ("lane_split", i32, [sc, sw, i32, i32, vp]),
                ("row_splits", i32, [sc, sw, i32, vp]),
                ("sizeof", i32, [C.c_int]),
                ("run_lane", i32, [sc, sw, opt, u64, u64, u64, C.POINTER(TwinLaunch), C.POINTER(TwinOutputs)]),
                ("run_warp", i32, [sc, sw, opt, u64, u64, u64, C.POINTER(TwinLaunch), C.POINTER(TwinOutputs)])):
            f = getattr(L, "af_twin_" + name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _sweep(sweep, sweep_first: int = 0):
    """(pointer, what keeps it alive): rows [sweep_first, end) of the table describe replicas sweep_first, ..."""
    if sweep is None:
        return None, None
    sw, keep = sweep.pod(sweep_first, None)
    return C.byref(sw), (sw, keep)


def _why(f, *args, cap: int = 400) -> tuple[bool, str]:
    why = C.create_string_buffer(cap)
    return bool(f(*args, why, cap)), why.value.decode()


# ---- the launch checks and sizes ------------------------------------------------------------------------------------
def ticks(flat) -> int:
    """The ticks a replica that reaches the horizon takes (what ``af_fetch_bands`` reports as ``n_ticks``)."""
    return int(lib().af_twin_ticks(C.byref(flat.pod)))


def ticks_fit(flat) -> tuple[bool, str]:
    """The tick-count check ``af_bands_upload`` / ``af_run`` apply: (fits, why not)."""
    return _why(lib().af_twin_ticks_fit, C.byref(flat.pod), cap=256)


def sumsq_fits(flat, group: int, *, request_capacity: int = 0, sweep=None) -> tuple[bool, int, str]:
    """The check ``af_bands_upload`` applies: (fits, bound on a gauge, what sets the bound)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    sw_p, keep = _sweep(sweep)
    bound = C.c_uint64()
    ok, what = _why(lib().af_twin_sumsq_fits, C.byref(flat.pod), sw_p, C.byref(opt), int(group), C.byref(bound), cap=256)
    del keep
    return ok, int(bound.value), what


def lat_fits(window_s: int, horizon_s: int, n_groups: int, mem_total: int) -> tuple[bool, str]:
    return _why(lib().af_twin_lat_fits, int(window_s), int(horizon_s), int(n_groups), int(mem_total), cap=256)


def dist_fits(flat, series, n_groups: int, mem_total: int = 1 << 62, *, request_capacity: int = 0, sweep=None):
    """The checks ``af_dist_bands_configure`` / ``af_bands_upload`` / ``af_run`` apply: (fits, ticks, bins, why)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    s = np.ascontiguousarray(series, dtype=np.int32)
    sw_p, keep = _sweep(sweep)
    t, b = C.c_uint32(), C.c_uint32()
    ok, why = _why(lib().af_twin_dist_fits, C.byref(flat.pod), sw_p, C.byref(opt), s.ctypes.data, s.size,
                   int(n_groups), int(mem_total), C.byref(t), C.byref(b))
    del keep
    return ok, int(t.value), int(b.value), why


def occ_fits(flat, f: int, *, request_capacity: int = 0, sweep=None) -> tuple[bool, str]:
    """The check ``af_run`` applies to a launch with f fraction bits: (fits, why not)."""
    opt = K.AfOptions(0, request_capacity, 0, 0, 1, 1, 0, 0)
    sw_p, keep = _sweep(sweep)
    out = _why(lib().af_twin_occ_fits, C.byref(flat.pod), sw_p, C.byref(opt), int(f))
    del keep
    return out


def gauge_bin(v: int) -> int:
    return int(lib().af_twin_gauge_bin(int(v)))


def frac_bits(bound: int, horizon_s: int) -> int:
    """``afh::occ_frac_bits``: the f af_run's users pick for a bound and a horizon."""
    return int(lib().af_twin_frac_bits(int(bound), int(horizon_s)))


def occ_fixed(rest: float, f: int) -> int:
    """``afr::occ_fixed`` on the host."""
    return int(lib().af_twin_occ_fixed(float(rest), int(f)))


def occ_cols(flat) -> int:
    return 5 * flat.n_servers + flat.n_edges


def lean_qualifies(flat, trace_replicas: int = 0) -> bool:
    """``aflh::lean_launch``: whether af_run runs the launch on the lean build of the lane loop."""
    return bool(lib().af_twin_lean_qualifies(C.byref(flat.pod), trace_replicas))


def row_splits(flat, spec, lane_bytes: int):
    """(pool, reported (ev_s, rq_s), [(estimate, ev_s, rq_s) per row]) as af_run splits lanes of `lane_bytes`."""
    sw, keep = spec.pod(0, None)
    out = (C.c_int32 * (3 + 3 * sw.n_rows))()
    assert lib().af_twin_row_splits(C.byref(flat.pod), C.byref(sw), lane_bytes, out) == 0
    rows = [tuple(out[3 + 3 * r: 6 + 3 * r]) for r in range(sw.n_rows)]
    del keep
    return out[0], (out[1], out[2]), rows


def band_rows(flat, n_groups: int) -> np.ndarray:
    """Zeroed difference rows of ``n_groups`` groups plus the one of replicas without a group."""
    return np.zeros(((n_groups + 1), 1 + 2 * flat.n_series, ticks(flat) + 1), dtype=np.uint64)


def lat_windows(flat, w: int) -> int:
    return -(-int(flat.horizon_s) // int(w))


def lat_rows(flat, n_groups: int, w: int) -> np.ndarray:
    return np.zeros((n_groups + 1, max(lat_windows(flat, w), 1), LAT_ROW), dtype=np.uint64)


def lat_split(rows: np.ndarray, n_groups: int):
    """Rows -> (hist [G, W, AF_HIST_BINS], sum_hi [G, W], sum_lo [G, W]) of the fetched groups."""
    r = rows[:n_groups]
    return r[:, :, :K.AF_HIST_BINS], r[:, :, K.AF_HIST_BINS], r[:, :, K.AF_HIST_BINS + 1]


def dist_rows(flat, series, n_groups: int, request_capacity: int, sweep=None) -> np.ndarray:
    ok, T, B, why = dist_fits(flat, series, n_groups, request_capacity=request_capacity, sweep=sweep)
    assert ok, why
    return np.zeros((n_groups + 1, max(len(series), 1), T + 1, B), dtype=np.uint32)


# ---- the engines --------------------------------------------------------------------------------------------------
def _outputs(flat, n: int, trace: int, clock_cap: int) -> dict:
    nser = flat.n_series
    tick_cap = lib().af_twin_trace_tick_capacity(C.byref(flat.pod))
    return {
        "stats": np.zeros(n, dtype=K.STATS_DTYPE),
        "sent": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "dropped": np.zeros((n, flat.n_edges), dtype=np.uint32),
        "hist": np.zeros((n, K.AF_HIST_BINS), dtype=np.uint32),
        "thr": np.zeros((n, flat.horizon_s), dtype=np.uint32),
        "samp_sum": np.zeros((n, nser), dtype=np.uint64),
        "samp_max": np.zeros((n, nser), dtype=np.uint32),
        "trace_clocks": np.zeros((max(trace, 1), max(clock_cap, 1), 2), dtype=np.float64),
        "trace_series": np.zeros((max(trace, 1), nser, tick_cap), dtype=np.uint32),
        "trace_counts": np.zeros((max(n, 1), 2), dtype=np.uint32),
    }


def _ptr(a) -> int | None:
    return None if a is None else a.ctypes.data


def _launch(fn, flat, out: dict, *, seed, n, replica_begin, sweep, sweep_first, groups, n_groups, band_first, sampled,
            window, series, f, bin_capacity, opt, **knobs) -> dict:
    """Adds the rows ``out`` lacks (a zero word for a kind that is off), runs ``fn`` (af_twin_run_lane / _warp) over
    them and returns ``out``."""
    s = np.ascontiguousarray(series, dtype=np.int32)
    g = np.ascontiguousarray(groups if groups is not None else np.zeros(0), dtype=np.uint32)
    assert g.size == 0 or int(g.max()) < n_groups
    out.setdefault("band_rows", band_rows(flat, n_groups) if sampled else np.zeros(1, dtype=np.uint64))
    out.setdefault("band_from", np.full(n, 0xFFFFFFFF, dtype=np.uint32))
    out.setdefault("lat_rows", lat_rows(flat, n_groups, window) if window else np.zeros(1, dtype=np.uint64))
    out.setdefault("lat_from", np.full(n, 0xFFFFFFFF, dtype=np.uint32))
    out.setdefault("dist_rows", dist_rows(flat, s, n_groups, bin_capacity, sweep) if s.size
                   else np.zeros(1, dtype=np.uint32))
    out.setdefault("occ", np.zeros((n, occ_cols(flat)), dtype=np.uint64))
    k = TwinLaunch(sweep_first=sweep_first, sampled=int(sampled), lat_window=int(window), group_of=g.ctypes.data,
                   band_first=band_first, band_n=g.size, n_groups=n_groups, n_dist=s.size,
                   band_rows=_ptr(out["band_rows"]), band_from=_ptr(out["band_from"]), lat_rows=_ptr(out["lat_rows"]),
                   lat_from=_ptr(out["lat_from"]), dist_series=s.ctypes.data, dist_capacity=bin_capacity,
                   occ_bits=int(f), dist_rows=_ptr(out["dist_rows"]), occ=_ptr(out["occ"]), **knobs)
    o = TwinOutputs(*[_ptr(out[key]) for key in OUTPUTS])
    sw_p, keep = _sweep(sweep, sweep_first)
    rc = fn(C.byref(flat.pod), sw_p, C.byref(opt), seed, replica_begin, n, C.byref(k), C.byref(o))
    if rc != 0:
        raise RuntimeError(lib().af_twin_error().decode())
    del keep
    return out


def run_lane(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, sweep_first: int = 0, groups=None,
             n_groups: int = 1, band_first: int = 0, sampled: bool = False, window: int = 0, series=(),
             lean: bool = False, f: int = 0, split: str = "rows", split_seed: int = 0, ev_need: int | None = None,
             order=None, trace: int = 0, clock_cap: int = 0, event_capacity: int = 2048, request_capacity: int = 16384,
             lane_bytes: int = 1816, bin_capacity: int = 0) -> dict:
    """The thread-per-replica engine over replicas ``[replica_begin, replica_begin + n)`` (sweep rows from replica
    ``sweep_first``), pulled in id order or ``order`` (a permutation of local indices), in the lean or the full build
    of its loop.  ``split``: the pool split of each replica (``SPLITS``; ``"scenario"`` splits by ``ev_need``, default
    the scenario's estimate, 0 = even; ``"random"`` draws from ``split_seed`` and the replica).  Optionally the
    per-tick (``sampled``), latency (``window`` s) and distribution (``series``; bins sized by ``bin_capacity``,
    default the request capacity) bands over ``groups[i]`` = group of replica ``band_first + i``, and occupancy
    integrals of ``f`` fraction bits.  Returns the outputs plus ``band_rows`` / ``band_from``, ``lat_rows`` /
    ``lat_from`` (per local replica: where a stopped one stopped), ``dist_rows`` and ``occ``."""
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    if order is not None:
        order = np.ascontiguousarray(order, dtype=np.uint32)
        assert order.shape == (n,) and np.array_equal(np.sort(order), np.arange(n))
    return _launch(lib().af_twin_run_lane, flat, _outputs(flat, n, trace, clock_cap), seed=seed, n=n,
                   replica_begin=replica_begin, sweep=sweep, sweep_first=sweep_first, groups=groups, n_groups=n_groups,
                   band_first=band_first, sampled=sampled, window=window, series=series, f=f,
                   bin_capacity=bin_capacity or request_capacity, opt=opt, lane_bytes=lane_bytes,
                   ev_need=-1 if ev_need is None else ev_need, split=SPLITS[split], lean=int(lean),
                   split_seed=split_seed, order=_ptr(order))


def run_warp(flat, *, seed: int, n: int, replica_begin: int = 0, sweep=None, sweep_first: int = 0, groups=None,
             n_groups: int = 1, band_first: int = 0, sampled: bool = False, window: int = 0, series=(), f: int = 0,
             trace: int = 0, clock_cap: int = 0, event_capacity: int = 0, request_capacity: int = 0, redo=None,
             band_from=None, into: dict | None = None, bin_capacity: int = 0) -> dict:
    """The warp-per-replica engine, with the bands and occupancy of :func:`run_lane`.  First-hand (``redo=None``):
    every replica of the launch.  A re-run (``redo`` = local indices, ``into`` = the lane pass's outputs): those
    replicas again, as af_run's second pass, their bands continuing from ``into``'s ``band_from`` (or ``band_from``)
    and ``lat_from`` and adding to its rows, their other outputs and occupancy rows overwritten there."""
    opt = K.AfOptions(event_capacity, request_capacity, 0, 0, 1, 1, trace, clock_cap)
    out = into if into is not None else _outputs(flat, n, trace, clock_cap)
    lst = None if redo is None else np.ascontiguousarray(redo, dtype=np.uint32)
    if lst is not None and band_from is not None:
        out["band_from"] = np.ascontiguousarray(band_from, dtype=np.uint32)
    return _launch(lib().af_twin_run_warp, flat, out, seed=seed, n=n, replica_begin=replica_begin, sweep=sweep,
                   sweep_first=sweep_first, groups=groups, n_groups=n_groups, band_first=band_first, sampled=sampled,
                   window=window, series=series, f=f, bin_capacity=bin_capacity or request_capacity or 16384, opt=opt,
                   redo=_ptr(lst), n_redo=0 if lst is None else lst.size)


#: which state machine run() drives when the caller does not say: "lane" = af_lane.cuh (thread per replica, the
#: product's first pass), "warp" = af_core.cuh (warp per replica, the product's pass for flagged replicas)
DEFAULT_ENGINE = os.environ.get("AF_TWIN_ENGINE", "lane")
#: the lane's share of shared memory in the twin (the CUDA engine derives it from the occupancy it picks)
DEFAULT_LANE_BYTES = int(os.environ.get("AF_TWIN_LANE_BYTES", "1816"))


def run(flat, *, seed: int, replica_begin: int = 0, n: int = 1, sweep=None, sweep_first: int = 0, trace: int = 0,
        clock_cap: int = 0, event_capacity: int = 0, request_capacity: int = 0,
        engine: str | None = None, lane_bytes: int | None = None, ev_need: int = 0) -> dict:
    """One launch on either state machine, no bands.  ``ev_need``: the pending-events estimate the lane engine splits
    its shared memory by (af_run computes it from the scenario and the sweep; 0 = the even split)."""
    kw = dict(seed=seed, n=n, replica_begin=replica_begin, sweep=sweep, sweep_first=sweep_first, trace=trace,
              clock_cap=clock_cap)
    if (engine or DEFAULT_ENGINE) == "lane":  # same default capacities as the warp engine (the CUDA lane pass has smaller ones and escalates)
        out = run_lane(flat, event_capacity=event_capacity or 2048, request_capacity=request_capacity or 16384,
                       lane_bytes=lane_bytes or DEFAULT_LANE_BYTES, split="scenario", ev_need=max(int(ev_need), 0), **kw)
    else:
        out = run_warp(flat, event_capacity=event_capacity, request_capacity=request_capacity, **kw)
    return {k: out[k] for k in OUTPUTS}
