// CPU twin of both engines with PER-TICK DISTRIBUTION BANDS -- TEST INFRASTRUCTURE ONLY.
//
// af_run accumulates distribution bands (af_dist_bands_configure) as difference rows over (tick, value bin): the
// thread-per-replica engine moves a replica between bins at every change of a selected gauge (run_lane<*, *, *, true>),
// the warp-per-replica engine at every tick whose value differs from the last one (take_samples), and a replica the first
// pass flags is re-run by the second from the tick it stopped at.  This file drives both state machines that way, with
// the caller's capacities (small ones force stops), with or without the per-tick and latency bands and in the lean or the
// full build of the loop, so tests can pin the rows to the oracle and check that every other output stays the same.  The
// prefix scan is left to the caller.  Loaded by tests/dist_twin.py only.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_dist_twin_error() { return g_err.c_str(); }
extern "C" int af_dist_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" uint32_t af_dist_twin_ticks(const AfScenario* sc) { return afh::band_ticks(*sc); }
extern "C" uint32_t af_dist_twin_gauge_bin(uint32_t v) { return afr::gauge_bin(v); }
// the checks af_dist_bands_configure / af_bands_upload / af_run apply: 1 when the series are valid and the rows of
// n_groups groups fit a device of mem_total bytes (ticks and bins set), else 0 and why
extern "C" int af_dist_twin_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, const int32_t* series, int32_t n,
                                 uint64_t n_groups, uint64_t mem_total, uint32_t* ticks, uint32_t* bins, char* why, int why_cap) {
    std::string w;
    int32_t server = -1;
    const uint64_t ram = sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
    const bool ok = afh::dist_series_check(*sc, series, n, w)
                    && afh::dist_bands_fit(*sc, *opt, ram, server, n_groups, (uint64_t)n, mem_total, *ticks, *bins, w);
    snprintf(why, (size_t)why_cap, "%s", w.c_str());
    return ok ? 1 : 0;
}

template <bool S, bool L, bool Lean, class P, class V>
static void run_d(bool dist, const afl::Mem& m, P pull, V conv) {
    if (dist) afl::run_lane<S, L, Lean, true>(m, pull, conv);
    else afl::run_lane<S, L, Lean, false>(m, pull, conv);
}
template <bool S, bool L, class P, class V>
static void run_ld(bool lean, bool dist, const afl::Mem& m, P pull, V conv) {
    if (lean) run_d<S, L, true>(dist, m, pull, conv); else run_d<S, L, false>(dist, m, pull, conv);
}

// The shape of a launch's distribution rows, (n_groups + 1) x n x (ticks + 1) x bins u32 (zeroed by the caller; series[s]
// is the af_fetch_sampled index of slot s, slot[j] gets each series' slot).  af_run sizes the bins by the caller's
// request capacity in both passes: `capacity` stands for it when the twin runs a pass with another one (0: opt's).
static void dist_shape(const AfScenario* sc, const AfOptions* opt, const AfSweep* sw, int32_t n, int32_t capacity,
                       uint32_t& ticks, uint32_t& bins) {
    int32_t server = -1;
    const uint64_t ram = sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
    AfOptions o = *opt;
    if (capacity > 0) o.request_capacity = capacity;
    std::string w;
    afh::dist_bands_fit(*sc, o, ram, server, 0, (uint64_t)n, ~0ull, ticks, bins, w);
}

// The thread-per-replica engine, replicas [replica_begin, replica_begin + n).  sampled / lat_window != 0 select
// run_lane's bands; the groups are group_of[i] for replica band_first + i.  lat_rows: (n_groups + 1) x n_windows x
// afr::LAT_ROW u64, zeroed by the caller; lat_from[local] = the completions a stopped replica added.
extern "C" int af_dist_twin_run_lane(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t lane_bytes,
                                    uint64_t seed, uint64_t replica_begin, uint64_t n, int32_t sampled, int32_t lat_window,
                                    const uint32_t* group_of, uint64_t band_first, uint64_t band_n, uint32_t n_groups,
                                    uint64_t* band_rows, uint32_t* band_from, uint64_t* lat_rows, uint32_t* lat_from,
                                    int32_t lean, const int32_t* dist_series, int32_t n_dist, int32_t dist_capacity, int32_t* dist_slot, uint32_t* dist_rows,
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
    if (n_dist) {
        if (!afh::dist_series_check(*sc, dist_series, n_dist, g_err)) return AF_ERR_INVALID;
        uint32_t dt = 0, bins = 0;
        dist_shape(sc, opt, sw, n_dist, dist_capacity, dt, bins);
        for (int32_t j = 0; j < C.n_series; ++j) dist_slot[j] = -1;
        for (int32_t k = 0; k < n_dist; ++k) dist_slot[dist_series[k]] = k;
        C.dist_rows = dist_rows; C.dist_slot = dist_slot; C.dist_n = n_dist; C.dist_bins = (int32_t)bins;
        C.dist_series_words = ((uint64_t)dt + 1) * bins; C.dist_group_words = (uint64_t)n_dist * C.dist_series_words;
    }
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    uint64_t next = 0;
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    auto pull = [&]() -> uint64_t { return next < n ? next++ : ~0ull; };
    auto conv = [](bool alive) { return alive; };
    if (sampled && lat_window) run_ld<true, true>(lean, n_dist > 0, m, pull, conv);
    else if (sampled) run_ld<true, false>(lean, n_dist > 0, m, pull, conv);
    else if (lat_window) run_ld<false, true>(lean, n_dist > 0, m, pull, conv);
    else run_ld<false, false>(lean, n_dist > 0, m, pull, conv);
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
extern "C" int af_dist_twin_run_warp(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t seed,
                                    uint64_t replica_begin, uint64_t n, const uint32_t* list, uint64_t n_list,
                                    int32_t sampled, int32_t lat_window, const uint32_t* group_of, uint64_t band_first,
                                    uint64_t band_n, uint32_t n_groups, uint64_t* band_rows, const uint32_t* band_from,
                                    uint64_t* lat_rows, const uint32_t* lat_from,
                                    const int32_t* dist_series, int32_t n_dist, int32_t dist_capacity, int32_t* dist_slot,
                                    uint32_t* dist_rows,
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
    if (n_dist && !afh::dist_series_check(*sc, dist_series, n_dist, g_err)) return AF_ERR_INVALID;
    afc::BandArgs band = {};
    band.group = group_of; band.first = band_first; band.n = band_n; band.groups = n_groups;
    if (sampled) {
        const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
        band.rows = band_rows;
        band.group_words = (1 + 2 * (uint64_t)L.n_series) * stride; band.stride = (uint32_t)stride;
    }
    if (sampled || n_dist) {
        band.from = band_from;
        band.prev_off = L.warp_bytes;
        L.warp_bytes += afc::align_up(4 * L.n_series, 16);
    }
    if (n_dist) {
        uint32_t dt = 0, bins = 0;
        dist_shape(sc, opt, sw, n_dist, dist_capacity, dt, bins);
        for (int32_t j = 0; j < L.n_series; ++j) dist_slot[j] = -1;
        for (int32_t k = 0; k < n_dist; ++k) dist_slot[dist_series[k]] = k;
        band.dist_rows = dist_rows; band.dist_slot = dist_slot; band.dist_bins = bins;
        band.dist_series_words = ((uint64_t)dt + 1) * bins; band.dist_group_words = (uint64_t)n_dist * band.dist_series_words;
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
