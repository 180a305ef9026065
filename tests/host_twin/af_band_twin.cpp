// CPU twin of both engines with PER-TICK BANDS -- TEST INFRASTRUCTURE ONLY.
//
// af_run accumulates per-tick bands (af_bands_upload) as difference rows: the thread-per-replica engine adds each gauge
// change at the tick index it happens before (run_lane<true>), the warp-per-replica engine each change between two
// ticks (take_samples), and a replica the first pass flags is re-run by the second from the tick it stopped at.  This
// file drives both state machines that way, with the caller's capacities (small ones force stops), so tests can pin the
// bands to the oracle and check the stitching of the two passes.  The prefix scan that turns the rows into per-tick
// values is left to the caller.  Loaded by tests/band_twin.py only; the product package cannot reach it.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_band_twin_error() { return g_err.c_str(); }
extern "C" int af_band_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" uint32_t af_band_twin_ticks(const AfScenario* sc) { return afh::band_ticks(*sc); }
// the tick-count check af_bands_upload / af_run apply: 1 when the band rows can hold every tick, else 0 and why
extern "C" int af_band_twin_ticks_fit(const AfScenario* sc, char* why, int why_cap) {
    uint32_t ticks = 0;
    std::string w;
    const bool ok = afh::band_ticks_fit(*sc, ticks, w);
    snprintf(why, (size_t)why_cap, "%s", w.c_str());
    return ok ? 1 : 0;
}

// the check af_bands_upload / af_run apply: 1 when a group of `group` replicas cannot wrap the u64 sums of squares,
// else 0 and the deciding bound in `what`
extern "C" int af_band_twin_sumsq_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t group,
                                       uint64_t* bound, char* what, int what_cap) {
    int32_t server = -1;
    const uint64_t ram = sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
    std::string w;
    *bound = afh::band_gauge_bound(*sc, *opt, ram, server, w);
    snprintf(what, (size_t)what_cap, "%s", w.c_str());
    return afh::band_sumsq_fits(group, *bound) ? 1 : 0;
}

// The thread-per-replica engine, replicas [replica_begin, replica_begin + n), each with its pool split as af_run splits
// it.  bands != 0: run_lane<true> into `band_rows` ((n_groups + 1) x (1 + 2 n_series) x (ticks + 1) u64, zeroed by the
// caller) with group_of[i] the group of replica band_first + i; `band_from[local]` = the tick a stopped replica stopped at.
extern "C" int af_band_twin_run_lane(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                                     int32_t lane_bytes, uint64_t seed, uint64_t replica_begin, uint64_t n,
                                     int32_t bands, const uint32_t* group_of, uint64_t band_first, uint64_t band_n,
                                     uint32_t n_groups, uint64_t* band_rows, uint32_t* band_from,
                                     AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                     uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                     uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
    uint32_t ticks = 0;
    if (bands && !afh::band_ticks_fit(*sc, ticks, g_err)) return AF_ERR_INVALID;
    aflh::Tables T;
    std::vector<int32_t> alias;
    const bool all_rows = sw && replica_begin >= sweep_first && replica_begin + n - sweep_first <= sw->n_rows;
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
        C.row_need = need.data(); C.need_first = sweep_first; C.need_rows = sw->n_rows;
    }
    C.edges = T.edges.data(); C.servers = T.servers.data(); C.endpoints = T.endpoints.data(); C.steps = T.steps.data();
    C.spikes = T.spikes.data(); C.outages = T.outages.data(); C.lb_edges = T.lb.data(); C.cols = T.cols.data();
    if (sw) { C.sweep_vals = sw->values; C.sweep_first = sweep_first; C.sweep_rows = sw->n_rows; }
    C.stats = stats; C.edge_sent = sent; C.edge_dropped = dropped; C.hist = hist; C.thr = thr;
    C.samp_sum = samp_sum; C.samp_max = samp_max; C.trace_clocks = trace_clocks; C.trace_series = trace_series;
    C.trace_counts = trace_counts;
    C.seed = seed; C.replica_begin = replica_begin; C.n_replicas = n;
    const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
    C.band_rows = band_rows; C.band_group = group_of; C.band_from = band_from;
    C.band_first = band_first; C.band_n = band_n; C.band_group_words = (1 + 2 * (uint64_t)C.n_series) * stride;
    C.band_groups = (int32_t)n_groups; C.band_stride = (int32_t)stride;
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    uint64_t next = 0;
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    auto pull = [&]() -> uint64_t { return next < n ? next++ : ~0ull; };
    auto conv = [](bool alive) { return alive; };
    if (bands) afl::run_lane<true>(m, pull, conv);
    else afl::run_lane<false>(m, pull, conv);
    if (C.collect_hist && stats)
        for (uint64_t r = 0; r < n; ++r) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    return AF_OK;
}

// The warp-per-replica engine over the local indices `list[0 .. n_list)` of a launch of replicas [replica_begin,
// replica_begin + n) (list = nullptr: every one, first-hand).  `band_from` != nullptr: a re-run of flagged replicas, as
// af_run's second pass -- each contributes from tick band_from[local] on (the outputs of those locals are overwritten).
extern "C" int af_band_twin_run_warp(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                                     uint64_t seed, uint64_t replica_begin, uint64_t n, const uint32_t* list, uint64_t n_list,
                                     int32_t bands, const uint32_t* group_of, uint64_t band_first, uint64_t band_n,
                                     uint32_t n_groups, uint64_t* band_rows, const uint32_t* band_from,
                                     AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                     uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                     uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
    uint32_t ticks = 0;
    if (bands && !afh::band_ticks_fit(*sc, ticks, g_err)) return AF_ERR_INVALID;
    afc::Layout& L = afc::h_L;
    memset(&L, 0, sizeof L);
    afh::make_layout(*sc, *opt, sw ? sw->n_columns : 0, L);
    afc::Globals& G = afc::h_G;
    memset(&G, 0, sizeof G);
    G.edges = sc->edges; G.servers = sc->servers;
    G.endpoints = sc->endpoints; G.steps = sc->steps;
    G.lb_edges = sc->lb_edges; G.spikes = sc->spike_marks; G.outages = sc->outage_marks;
    if (sw) { G.sweep_cols = sw->columns; G.sweep_vals = sw->values; G.sweep_first = sweep_first; G.sweep_rows = sw->n_rows; }
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
    if (band_from) { G.redo_list = list; G.redo_count = &count; }
    afc::BandArgs band = {};
    if (bands) {
        const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
        band.rows = band_rows; band.group = group_of; band.from = band_from;
        band.first = band_first; band.n = band_n; band.group_words = (1 + 2 * (uint64_t)L.n_series) * stride;
        band.groups = n_groups; band.stride = (uint32_t)stride;
        band.prev_off = L.warp_bytes;
        L.warp_bytes += afc::align_up(4 * L.n_series, 16);
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
