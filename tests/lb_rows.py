"""Load-balancer sweep rows for the tests (``("lb_covered", server)`` / ``("lb_algorithm",)`` columns) and the comparison
of one engine replica, laid out over the scenario's edges, with the oracle run on its reduced payload."""

from __future__ import annotations

import numpy as np
from helpers import assert_matches_oracle

from asyncflow_b200.flatten import flatten


def lb_servers(payload: dict) -> list[str]:
    return list(payload["topology_graph"]["nodes"]["load_balancer"]["server_covered"])


def uncoverable(payload: dict) -> tuple[list[str], str]:
    """(servers a row may uncover, the server every row keeps): no spike on the server's LB edge, and the kept one
    never goes down."""
    lb = payload["topology_graph"]["nodes"]["load_balancer"]["id"]
    events = payload.get("events") or []
    down = {e["target_id"] for e in events if "spike_s" not in e["start"]}
    spiked = {e["target_id"] for e in events if "spike_s" in e["start"]}
    edge = {e["target"]: e["id"] for e in payload["topology_graph"]["edges"] if e["source"] == lb}
    ok = [s for s in lb_servers(payload) if edge[s] not in spiked]
    keep = next(s for s in ok if s not in down)
    return [s for s in ok if s != keep], keep


def lb_columns(payload: dict, n: int, rng: np.random.Generator, *, p_off: float = 0.4) -> dict:
    """Random fleets (each uncoverable server off with probability ``p_off``) and algorithms for ``n`` rows."""
    free, _ = uncoverable(payload)
    cols: dict = {("lb_covered", s): (rng.random(n) >= p_off).astype(np.float64) for s in free}
    cols[("lb_algorithm",)] = rng.choice(["round_robin", "least_connection"], n).tolist()
    return cols


def edge_view(flat, reduced) -> list[int]:
    """Index, in ``flat``'s edges, of each edge of the reduced scenario."""
    return [flat.edge_ids.index(e) for e in reduced.edge_ids]


def series_view(flat, reduced) -> list[int]:
    ns = 3 * flat.n_servers
    return list(range(ns)) + [ns + i for i in edge_view(flat, reduced)]


def check_replica(o: dict, flat, p: dict, *, stats, sent, dropped, thr, clocks=None, series=None) -> None:
    """One replica of a launch over ``flat`` (its outputs over ``flat``'s edges) equals oracle run ``o`` of its reduced
    payload ``p``, and every edge the reduced payload lacks carried nothing."""
    red = flatten(p)
    keep = edge_view(flat, red)
    gone = [j for j in range(flat.n_edges) if j not in keep]
    assert stats["flags"] == 0
    assert_matches_oracle(o, red, stats=stats, clocks=clocks, sent=np.asarray(sent)[keep], dropped=np.asarray(dropped)[keep],
                          series=None if series is None else np.asarray(series)[series_view(flat, red)], throughput=thr)
    assert not np.asarray(sent)[gone].any() and not np.asarray(dropped)[gone].any()
    if series is not None:
        assert not np.asarray(series)[[3 * flat.n_servers + j for j in gone]].any()
