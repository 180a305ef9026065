"""Random per-row event times for the event-timeline tests (``("event_start"|"event_end", event_id)`` sweep columns):
rows that pass the payload rules, half of their times on a coarse grid so that ends and starts tie."""

from __future__ import annotations

import numpy as np


def event_time_columns(flat, n: int, rng: np.random.Generator, *, grid: float = 0.5, spike_delta: bool = False,
                       lo: float = 0.0, hi: float | None = None) -> dict:
    """Every event of ``flat`` gets a random ``[t_start, t_end)`` inside ``[lo, hi]`` (default the horizon) per row.  A
    server's outages get disjoint slots of that span, so they never overlap (they may touch); a scenario that covers
    every server with outages is not supported.  ``spike_delta``: a random amplitude per spike event too."""
    hi = float(flat.horizon_s) if hi is None else hi
    by_server: dict[int, list] = {}
    for e in flat.events:
        if not e.spike:
            by_server.setdefault(e.server, []).append(e)
    assert len(by_server) < flat.n_servers, "every server has an outage: rows could take them all down"

    def draw(a: float, b: float) -> tuple[np.ndarray, np.ndarray]:
        x, y = rng.uniform(a, b, n), rng.uniform(a, b, n)
        s, t = np.minimum(x, y), np.maximum(x, y)
        snap = rng.random(n) < 0.5
        s = np.where(snap, np.floor(s / grid) * grid, s)
        t = np.where(snap, np.ceil(t / grid) * grid, t)
        return s, np.where(t > s, t, s + grid)

    cols: dict = {}
    for e in flat.events:
        if e.spike:
            s, t = draw(lo, hi)
            if spike_delta:
                # dyadic amplitudes: overlapping spikes add and remove exactly, so an edge's spike never ends a hair
                # below zero (the reference refuses the negative delay that would give)
                cols[("spike_delta", e.event_id)] = rng.choice([2.0**-10, 2.0**-7, 2.0**-5], n)
        else:
            evs = by_server[e.server]
            k = evs.index(e)
            edges = np.round(np.linspace(lo, hi, len(evs) + 1) / grid) * grid
            s, t = draw(float(edges[k]), float(edges[k + 1]))
        cols[("event_start", e.event_id)] = s
        cols[("event_end", e.event_id)] = t
    return cols
