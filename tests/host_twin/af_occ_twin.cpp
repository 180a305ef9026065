// CPU twin of both engines with OCCUPANCY INTEGRALS -- TEST INFRASTRUCTURE ONLY.
//
// af_run integrates, per replica, the requests in each state over the run (af_occupancy_configure): the
// thread-per-replica engine with run_lane<*, *, *, *, true>, the warp-per-replica engine behind State.occ, and a replica
// the first pass flags is re-run from the start by the second.  This file drives both state machines that way, with the
// caller's capacities (small ones force stops), with or without every kind of band and in the lean or the full build of
// the loop, so tests can pin the rows to the oracle and check that every other output stays the same.  Loaded by
// tests/occ_twin.py only.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_occ_twin_error() { return g_err.c_str(); }
extern "C" int af_occ_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" int32_t af_occ_twin_frac_bits(uint64_t bound, int32_t horizon_s) { return afh::occ_frac_bits(bound, horizon_s); }
extern "C" uint64_t af_occ_twin_fixed(double rest, int32_t frac_bits) { return afr::occ_fixed(rest, ldexp(1.0, frac_bits)); }
// the check af_run applies to a launch with f = frac_bits: 1 when it fits, else 0 and why
extern "C" int af_occ_twin_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t frac_bits, char* why,
                                int why_cap) {
    std::string w;
    int32_t server = -1;
    const uint64_t ram = sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
    const bool ok = afh::occ_fits(*sc, *opt, ram, server, frac_bits, w);
    snprintf(why, (size_t)why_cap, "%s", w.c_str());
    return ok ? 1 : 0;
}

template <bool S, bool L, bool Lean, bool D, class P, class V>
static void run_o(bool occ, const afl::Mem& m, P pull, V conv) {
    if (occ) afl::run_lane<S, L, Lean, D, true>(m, pull, conv);
    else afl::run_lane<S, L, Lean, D, false>(m, pull, conv);
}
template <bool S, bool L, class P, class V>
static void run_ldo(bool lean, bool dist, bool occ, const afl::Mem& m, P pull, V conv) {
    if (lean) { if (dist) run_o<S, L, true, true>(occ, m, pull, conv); else run_o<S, L, true, false>(occ, m, pull, conv); }
    else { if (dist) run_o<S, L, false, true>(occ, m, pull, conv); else run_o<S, L, false, false>(occ, m, pull, conv); }
}

// distribution bands of n series: ticks and bins as af_run sizes them for these options and sweep, each series' slot
static bool dist_setup(const AfScenario* sc, const AfOptions* opt, const AfSweep* sw, const int32_t* series, int32_t n,
                       int32_t n_series, int32_t* slot, uint32_t& ticks, uint32_t& bins) {
    if (!afh::dist_series_check(*sc, series, n, g_err)) return false;
    int32_t server = -1;
    const uint64_t ram = sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
    afh::dist_bands_fit(*sc, *opt, ram, server, 0, (uint64_t)n, ~0ull, ticks, bins, g_err);
    for (int32_t j = 0; j < n_series; ++j) slot[j] = -1;
    for (int32_t k = 0; k < n; ++k) slot[series[k]] = k;
    return true;
}

static void percentiles(AfReplicaStats* stats, const uint32_t* hist, uint64_t r) {
    stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
    stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
    stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
}

// The thread-per-replica engine, replicas [replica_begin, replica_begin + n).  occ_bits > 0: occupancy integrals with f =
// occ_bits into occ[n][5 n_servers + n_edges] (no check of f: af_run's is af_occ_twin_fits).  sampled / lat_window / n_dist
// select the bands over group_of[i] for replica band_first + i, into rows zeroed by the caller.
extern "C" int af_occ_twin_run_lane(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t lane_bytes,
                                    uint64_t seed, uint64_t replica_begin, uint64_t n, int32_t lean, int32_t occ_bits,
                                    uint64_t* occ, int32_t sampled, int32_t lat_window, const uint32_t* group_of,
                                    uint64_t band_first, uint64_t band_n, uint32_t n_groups, uint64_t* band_rows,
                                    uint32_t* band_from, uint64_t* lat_rows, uint32_t* lat_from, const int32_t* dist_series,
                                    int32_t n_dist, int32_t* dist_slot, uint32_t* dist_rows,
                                    AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                    uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                    uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
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
    if (occ_bits > 0) { aflh::add_occupancy(C, afl::LANES, afh::occ_cols(*sc), occ_bits); C.occ = occ; }
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
        uint32_t dt = 0, bins = 0;
        if (!dist_setup(sc, opt, sw, dist_series, n_dist, C.n_series, dist_slot, dt, bins)) return AF_ERR_INVALID;
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
    const bool dist = n_dist > 0, on = occ_bits > 0;
    if (sampled && lat_window) run_ldo<true, true>(lean, dist, on, m, pull, conv);
    else if (sampled) run_ldo<true, false>(lean, dist, on, m, pull, conv);
    else if (lat_window) run_ldo<false, true>(lean, dist, on, m, pull, conv);
    else run_ldo<false, false>(lean, dist, on, m, pull, conv);
    if (C.collect_hist && stats) for (uint64_t r = 0; r < n; ++r) percentiles(stats, hist, r);
    return AF_OK;
}

// The warp-per-replica engine over the local indices list[0 .. n_list) of a launch of replicas [replica_begin,
// replica_begin + n) (list = nullptr: every one, first-hand).  A re-run (band_from != nullptr) continues each replica's
// bands where the thread-per-replica pass stopped and overwrites its other outputs, occupancy included, as af_run's
// second pass.
extern "C" int af_occ_twin_run_warp(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t seed,
                                    uint64_t replica_begin, uint64_t n, const uint32_t* list, uint64_t n_list,
                                    int32_t occ_bits, uint64_t* occ, int32_t sampled, int32_t lat_window,
                                    const uint32_t* group_of, uint64_t band_first, uint64_t band_n, uint32_t n_groups,
                                    uint64_t* band_rows, const uint32_t* band_from, uint64_t* lat_rows,
                                    const uint32_t* lat_from, const int32_t* dist_series, int32_t n_dist, int32_t* dist_slot,
                                    uint32_t* dist_rows,
                                    AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                    uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                    uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
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
    if (list) { G.redo_list = list; G.redo_count = &count; }
    afc::BandArgs band = {};
    band.group = group_of; band.first = band_first; band.n = band_n; band.groups = n_groups;
    if (occ_bits > 0) { band.occ = occ; band.occ_scale = ldexp(1.0, occ_bits); }
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
        if (!dist_setup(sc, opt, sw, dist_series, n_dist, L.n_series, dist_slot, dt, bins)) return AF_ERR_INVALID;
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
        if (L.collect_hist && stats) percentiles(stats, hist, r);
    }
    return AF_OK;
}
