// CPU twin of the thread-per-replica engine with and without the LEAN build of its loop -- TEST INFRASTRUCTURE ONLY.
//
// af_run runs run_lane<S, L, true> (spikes, outages, traces, general edge samplers and endpoint draws compiled out)
// when aflh::lean_launch says the launch can reach none of them, run_lane<S, L, false> otherwise.  This file drives the
// same state machine both ways, with every band combination and per-replica pool splits, so that tests can require the
// two builds to give the same outputs bit for bit, and exposes the qualification rule.  Pool splits:
//   mode 0  every replica by the scenario's estimate
//   mode 1  as af_run: each replica with a sweep row by the row's estimate (aflh::row_events_estimates)
//   mode 2  a random split per replica (seeded by `split_seed` and the replica id), as tests/host_twin/af_split_twin.cpp
// Sweep rows describe replicas from 0.  Loaded by tests/test_lean_lane.py only; the product package cannot reach it.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_lean_twin_error() { return g_err.c_str(); }
extern "C" int af_lean_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" uint32_t af_lean_twin_ticks(const AfScenario* sc) { return afh::band_ticks(*sc); }
extern "C" int af_lean_twin_qualifies(const AfScenario* sc, int32_t trace_replicas) { return aflh::lean_launch(*sc, trace_replicas) ? 1 : 0; }

static uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

template <bool S, bool L, class P, class V>
static void run(bool lean, const afl::Mem& m, P pull, V conv) {
    if (lean) afl::run_lane<S, L, true>(m, pull, conv);
    else afl::run_lane<S, L, false>(m, pull, conv);
}

extern "C" int af_lean_twin_run_lane(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t lane_bytes,
                                     int32_t split_mode, uint64_t split_seed, uint64_t seed, uint64_t replica_begin,
                                     uint64_t n, int32_t lean, int32_t sampled, int32_t lat_window,
                                     const uint32_t* group_of, uint64_t band_first, uint64_t band_n, uint32_t n_groups,
                                     uint64_t* band_rows, uint32_t* band_from, uint64_t* lat_rows, uint32_t* lat_from,
                                     AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                     uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                     uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
    uint32_t ticks = 0;
    if (sampled && !afh::band_ticks_fit(*sc, ticks, g_err)) return AF_ERR_INVALID;
    if (lat_window && !afh::lat_bands_fit(lat_window, sc->horizon_s, n_groups, ~0ull, g_err)) return AF_ERR_INVALID;
    if (lean && !aflh::lean_launch(*sc, opt->trace_replicas)) { g_err = "the launch does not qualify for the lean loop"; return AF_ERR_INVALID; }
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
    if (split_mode == 1 && sw && sw->n_columns > 0 && sw->n_rows > 0) {
        aflh::row_events_estimates(*sc, *sw, need);
        C.row_need = need.data(); C.need_first = 0; C.need_rows = sw->n_rows;
    } else if (split_mode == 2) {
        need.resize((size_t)n);
        const int32_t rq_hi = C.pool - 1 < afl::RQ_BITS ? C.pool - 1 : afl::RQ_BITS;
        const int32_t span = rq_hi - C.rq_floor + 1;
        for (uint64_t r = 0; r < n; ++r) {
            const int32_t rq = span > 0 ? C.rq_floor + (int32_t)(splitmix64(split_seed * 0x100000001B3ull + replica_begin + r) % (uint64_t)span) : 1;
            need[(size_t)r] = C.pool - rq;
        }
        C.ev_lo = 1;
        C.row_need = need.data(); C.need_first = replica_begin; C.need_rows = n;
    } else if (split_mode != 0 && split_mode != 1) { g_err = "af_lean_twin_run_lane: unknown split mode"; return AF_ERR_INVALID; }
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
    if (sampled && lat_window) run<true, true>(lean != 0, m, pull, conv);
    else if (sampled) run<true, false>(lean != 0, m, pull, conv);
    else if (lat_window) run<false, true>(lean != 0, m, pull, conv);
    else run<false, false>(lean != 0, m, pull, conv);
    if (C.collect_hist && stats)
        for (uint64_t r = 0; r < n; ++r) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0);
        }
    return AF_OK;
}
