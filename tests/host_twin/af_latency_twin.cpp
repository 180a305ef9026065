// CPU twin of both engines with PER-WINDOW LATENCY BANDS -- TEST INFRASTRUCTURE ONLY.
//
// af_run accumulates per-window latency bands (af_bands_configure) in complete() of both engines: the thread-per-replica
// engine while no stop flag is set, recording for a stopped replica how many completions it added (lat_from), and the
// warp-per-replica engine from completion lat_from on when it re-runs a flagged replica.  This file drives both state
// machines that way, with the caller's capacities (small ones force stops), so tests can pin the rows to the oracle's
// clocks and check the stitching of the two passes.  The per-tick sampled bands ride along when asked for, so tests can
// also check that the two kinds of bands leave each other alone.  Loaded by tests/latency_twin.py only.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_lat_twin_error() { return g_err.c_str(); }
extern "C" int af_lat_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" uint32_t af_lat_twin_ticks(const AfScenario* sc) { return afh::band_ticks(*sc); }
extern "C" uint64_t af_lat_twin_fixed32(double lat) { return afr::lat_fixed32(lat); }
extern "C" int32_t af_lat_twin_hist_bin(double lat) { return afr::hist_bin(lat); }
// the check af_bands_configure / af_bands_upload / af_run apply: 1 when latency bands of `window_s` seconds over
// n_groups groups fit a device of mem_total bytes, else 0 and why
extern "C" int af_lat_twin_fits(int32_t window_s, int32_t horizon_s, uint64_t n_groups, uint64_t mem_total, char* why, int why_cap) {
    std::string w;
    const bool ok = afh::lat_bands_fit(window_s, horizon_s, n_groups, mem_total, w);
    snprintf(why, (size_t)why_cap, "%s", w.c_str());
    return ok ? 1 : 0;
}

// The thread-per-replica engine, replicas [replica_begin, replica_begin + n).  sampled / lat_window != 0 select
// run_lane's bands; the groups are group_of[i] for replica band_first + i.  lat_rows: (n_groups + 1) x n_windows x
// afr::LAT_ROW u64, zeroed by the caller; lat_from[local] = the completions a stopped replica added.
extern "C" int af_lat_twin_run_lane(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t lane_bytes,
                                    uint64_t seed, uint64_t replica_begin, uint64_t n, int32_t sampled, int32_t lat_window,
                                    const uint32_t* group_of, uint64_t band_first, uint64_t band_n, uint32_t n_groups,
                                    uint64_t* band_rows, uint32_t* band_from, uint64_t* lat_rows, uint32_t* lat_from,
                                    AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                    uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                    uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
    uint32_t ticks = 0;
    if (sampled && !afh::band_ticks_fit(*sc, ticks, g_err)) return AF_ERR_INVALID;
    if (lat_window && !afh::lat_bands_fit(lat_window, sc->horizon_s, n_groups, ~0ull, g_err)) return AF_ERR_INVALID;
    aflh::Tables T;
    std::vector<int32_t> alias;
    const bool all_rows = sw && replica_begin + n <= sw->n_rows;
    if (all_rows) alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    if (!aflh::build_tables(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0, all_rows ? alias.data() : nullptr, T, g_err)) return AF_ERR_INVALID;
    afl::Cfg& C = afl::h_cfg;
    memset(&C, 0, sizeof C);
    if (lane_bytes < aflh::min_lane_bytes(*sc, T)) lane_bytes = aflh::min_lane_bytes(*sc, T);
    if (!aflh::make_cfg(*sc, *opt, T, lane_bytes, afh::trace_tick_capacity(*sc), afl::LANES, C, aflh::pending_events_estimate(*sc, nullptr))) {
        g_err = "lane engine: tables do not fit the lane's shared memory"; return AF_ERR_INVALID;
    }
    std::vector<int32_t> need;
    if (sw && sw->n_columns > 0 && sw->n_rows > 0) {
        aflh::row_events_estimates(*sc, *sw, need);
        C.row_need = need.data(); C.need_first = 0; C.need_rows = sw->n_rows;
    }
    C.edges = T.edges.data(); C.servers = T.servers.data(); C.endpoints = T.endpoints.data(); C.steps = T.steps.data();
    C.spikes = T.spikes.data(); C.outages = T.outages.data(); C.lb_edges = T.lb.data(); C.cols = T.cols.data();
    if (sw) { C.sweep_vals = sw->values; C.sweep_first = 0; C.sweep_rows = sw->n_rows; }
    C.stats = stats; C.edge_sent = sent; C.edge_dropped = dropped; C.hist = hist; C.thr = thr;
    C.samp_sum = samp_sum; C.samp_max = samp_max; C.trace_clocks = trace_clocks; C.trace_series = trace_series;
    C.trace_counts = trace_counts;
    C.seed = seed; C.replica_begin = replica_begin; C.n_replicas = n;
    const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
    C.band_group = group_of; C.band_first = band_first; C.band_n = band_n; C.band_groups = (int32_t)n_groups;
    C.band_rows = band_rows; C.band_from = band_from;
    C.band_group_words = (1 + 2 * (uint64_t)C.n_series) * stride; C.band_stride = (int32_t)stride;
    C.lat_rows = lat_rows; C.lat_from = lat_from; C.lat_window = lat_window;
    C.lat_windows = lat_window ? (int32_t)afh::lat_windows(sc->horizon_s, lat_window) : 0;
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    uint64_t next = 0;
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    auto pull = [&]() -> uint64_t { return next < n ? next++ : ~0ull; };
    auto conv = [](bool alive) { return alive; };
    if (sampled && lat_window) afl::run_lane<true, true>(m, pull, conv);
    else if (sampled) afl::run_lane<true, false>(m, pull, conv);
    else if (lat_window) afl::run_lane<false, true>(m, pull, conv);
    else afl::run_lane<false, false>(m, pull, conv);
    if (C.collect_hist && stats)
        for (uint64_t r = 0; r < n; ++r) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    return AF_OK;
}

// The warp-per-replica engine over the local indices list[0 .. n_list) of a launch of replicas [replica_begin,
// replica_begin + n) (list = nullptr: every one, first-hand).  A re-run (band_from / lat_from != nullptr) continues each
// replica where the thread-per-replica pass stopped, as af_run's second pass (the outputs of those locals are overwritten).
extern "C" int af_lat_twin_run_warp(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t seed,
                                    uint64_t replica_begin, uint64_t n, const uint32_t* list, uint64_t n_list,
                                    int32_t sampled, int32_t lat_window, const uint32_t* group_of, uint64_t band_first,
                                    uint64_t band_n, uint32_t n_groups, uint64_t* band_rows, const uint32_t* band_from,
                                    uint64_t* lat_rows, const uint32_t* lat_from,
                                    AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                    uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                    uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
    uint32_t ticks = 0;
    if (sampled && !afh::band_ticks_fit(*sc, ticks, g_err)) return AF_ERR_INVALID;
    if (lat_window && !afh::lat_bands_fit(lat_window, sc->horizon_s, n_groups, ~0ull, g_err)) return AF_ERR_INVALID;
    afc::Layout& L = afc::h_L;
    memset(&L, 0, sizeof L);
    afh::make_layout(*sc, *opt, sw ? sw->n_columns : 0, L);
    afc::Globals& G = afc::h_G;
    memset(&G, 0, sizeof G);
    G.edges = sc->edges; G.servers = sc->servers;
    G.endpoints = sc->endpoints; G.steps = sc->steps;
    G.lb_edges = sc->lb_edges; G.spikes = sc->spike_marks; G.outages = sc->outage_marks;
    if (sw) { G.sweep_cols = sw->columns; G.sweep_vals = sw->values; G.sweep_first = 0; G.sweep_rows = sw->n_rows; }
    std::vector<double> sp_t((size_t)(L.ev_total - L.ev_smem) + 1);
    std::vector<uint64_t> sp_k((size_t)(L.ev_total - L.ev_smem) + 1);
    std::vector<afc::ReqRec> sp_r((size_t)(L.rq_total - L.rq_smem) + 1);
    std::vector<uint32_t> sp_n((size_t)(L.rq_total - L.rq_smem) + 1);
    G.spill_ev_time = sp_t.data(); G.spill_ev_key = sp_k.data(); G.spill_rq_rec = sp_r.data(); G.spill_rq_next = sp_n.data();
    G.stats = stats; G.edge_sent = sent; G.edge_dropped = dropped; G.hist = hist; G.thr = thr;
    G.samp_sum = samp_sum; G.samp_max = samp_max; G.trace_clocks = trace_clocks; G.trace_series = trace_series;
    G.trace_counts = trace_counts;
    G.seed = seed; G.replica_begin = replica_begin; G.n_replicas = n;
    uint32_t count = (uint32_t)n_list;
    if (band_from || lat_from) { G.redo_list = list; G.redo_count = &count; }
    afc::BandArgs band = {};
    band.group = group_of; band.first = band_first; band.n = band_n; band.groups = n_groups;
    if (sampled) {
        const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
        band.rows = band_rows; band.from = band_from;
        band.group_words = (1 + 2 * (uint64_t)L.n_series) * stride; band.stride = (uint32_t)stride;
        band.prev_off = L.warp_bytes;
        L.warp_bytes += afc::align_up(4 * L.n_series, 16);
    }
    if (lat_window) {
        band.lat_rows = lat_rows; band.lat_from = lat_from; band.lat_window = (uint32_t)lat_window;
        band.lat_windows = (uint32_t)afh::lat_windows(sc->horizon_s, lat_window);
    }
    std::vector<unsigned char> ws((size_t)L.warp_bytes + 64);
    unsigned char* base = (unsigned char*)(((uintptr_t)ws.data() + 15) & ~(uintptr_t)15);
    const uint64_t todo = list ? n_list : n;
    for (uint64_t k = 0; k < todo; ++k) {
        const uint64_t r = list ? list[k] : k;
        afc::State& W = *reinterpret_cast<afc::State*>(base);
        afc::bind(W, base, 0);
        afc::run_replica(W, r, band);
        if (L.collect_hist && stats) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    }
    return AF_OK;
}
