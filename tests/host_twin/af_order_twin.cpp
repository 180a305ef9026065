// CPU twin of the thread-per-replica engine with a PULL ORDER -- TEST INFRASTRUCTURE ONLY.
//
// af_run's lanes take local replica indices through a pull order (Cfg.order: heaviest replica first), not in id order.
// This file drives af_lane.cuh's run_lane the same way -- the lane pulls order[0], order[1], ... -- with each replica's
// pool split as af_run chooses it (its sweep row's pending-events estimate, else the scenario's), so tests can check that
// the order changes no output.  Loaded by tests/test_pull_order.py only; the product package cannot reach it.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_order_twin_error() { return g_err.c_str(); }
extern "C" int af_order_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }

// order: a permutation of [0, n) (nullptr: id order)
extern "C" int af_order_twin_run_lane(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                                      int32_t lane_bytes, uint64_t seed, uint64_t replica_begin, uint64_t n, const uint32_t* order,
                                      AfReplicaStats* stats, uint32_t* sent, uint32_t* dropped, uint32_t* hist,
                                      uint32_t* thr, uint64_t* samp_sum, uint32_t* samp_max, double* trace_clocks,
                                      uint32_t* trace_series, uint32_t* trace_counts) {
    if (!afh::validate(*sc, g_err)) return AF_ERR_INVALID;
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
    C.order = order;
    C.seed = seed; C.replica_begin = replica_begin; C.n_replicas = n;
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    uint64_t k = 0;                                   // the k-th pull gets local index order[k], as in af_lane_kernel
    afl::run_lane(m, [&]() -> uint64_t { if (k >= n) return ~0ull; const uint64_t i = C.order ? C.order[k] : k; ++k; return i; },
                  [](bool alive) { return alive; });
    if (C.collect_hist && stats)
        for (uint64_t r = 0; r < n; ++r) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    return AF_OK;
}
