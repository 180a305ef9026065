// CPU twin of the thread-per-replica engine with a pool split PER REPLICA -- TEST INFRASTRUCTURE ONLY.
//
// af_host_twin.cpp runs af_lane.cuh with one split for every replica of a launch (its pending-events estimate).  af_run
// splits each replica's shared-memory pool by the replica's own estimate (Cfg.row_need); this file drives the same
// state machine that way, so the CPU tests and tools/fuzz_campaign.py can pin per-replica splits to the oracle:
//   mode 1  as af_run: each replica with a sweep row by the row's estimate (aflh::row_events_estimates), the others by
//           the scenario's
//   mode 2  a random split per replica (seeded by `split_seed` and the replica id): rq_s uniform in
//           [2, min(pool - 1, 32)], the heap the rest
// Loaded by tests/split_twin.py only; the product package cannot reach it.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

static std::string g_err;
extern "C" const char* af_split_twin_error() { return g_err.c_str(); }
extern "C" int af_split_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }

static uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

extern "C" int af_split_twin_run_lane(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                                      int32_t lane_bytes, int32_t mode, uint64_t split_seed, uint64_t seed,
                                      uint64_t replica_begin, uint64_t n,
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
    if (mode == 1 && sw && sw->n_columns > 0 && sw->n_rows > 0) {
        aflh::row_events_estimates(*sc, *sw, need);
        C.row_need = need.data(); C.need_first = sweep_first; C.need_rows = sw->n_rows;
    } else if (mode == 2) {                            // the estimate that gives the drawn split (ev_lo = 1: any split)
        need.resize((size_t)n);
        const int32_t rq_hi = C.pool - 1 < afl::RQ_BITS ? C.pool - 1 : afl::RQ_BITS;
        const int32_t span = rq_hi - C.rq_floor + 1;
        for (uint64_t r = 0; r < n; ++r) {
            const int32_t rq = span > 0 ? C.rq_floor + (int32_t)(splitmix64(split_seed * 0x100000001B3ull + replica_begin + r) % (uint64_t)span) : 1;
            need[(size_t)r] = C.pool - rq;
        }
        C.ev_lo = 1;
        C.row_need = need.data(); C.need_first = replica_begin; C.need_rows = n;
    } else if (mode != 1) { g_err = "af_split_twin_run_lane: unknown mode"; return AF_ERR_INVALID; }
    C.edges = T.edges.data(); C.servers = T.servers.data(); C.endpoints = T.endpoints.data(); C.steps = T.steps.data();
    C.spikes = T.spikes.data(); C.outages = T.outages.data(); C.lb_edges = T.lb.data(); C.cols = T.cols.data();
    if (sw) { C.sweep_vals = sw->values; C.sweep_first = sweep_first; C.sweep_rows = sw->n_rows; }
    C.stats = stats; C.edge_sent = sent; C.edge_dropped = dropped; C.hist = hist; C.thr = thr;
    C.samp_sum = samp_sum; C.samp_max = samp_max; C.trace_clocks = trace_clocks; C.trace_series = trace_series;
    C.trace_counts = trace_counts;
    C.seed = seed; C.replica_begin = replica_begin; C.n_replicas = n;
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    uint64_t next = 0;
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    afl::run_lane(m, [&]() -> uint64_t { return next < n ? next++ : ~0ull; }, [](bool alive) { return alive; });
    if (C.collect_hist && stats)
        for (uint64_t r = 0; r < n; ++r) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    return AF_OK;
}

// The split af_run gives each row of `sw` for a lane of `lane_bytes` (the CUDA engine's capacities), and the one it
// reports for the launch (AfRunPasses: the heaviest row's).  out[0] = pool, out[1], out[2] = the reported split,
// out[3 + 3r ...] = {estimate, ev_s, rq_s} of row r
extern "C" int af_split_twin_row_splits(const AfScenario* sc, const AfSweep* sw, int32_t lane_bytes, int32_t* out) {
    aflh::Tables T; std::string err;
    std::vector<int32_t> alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    if (!aflh::build_tables(*sc, sw->columns, sw->n_columns, alias.data(), T, err)) return -1;
    AfOptions o; memset(&o, 0, sizeof o); o.event_capacity = aflh::LANE_EVENT_CAPACITY; o.request_capacity = aflh::LANE_REQUEST_CAPACITY;
    afl::Cfg C; memset(&C, 0, sizeof C);
    if (!aflh::make_cfg(*sc, o, T, lane_bytes, 0, 32, C, aflh::pending_events_estimate(*sc, nullptr))) return -2;
    std::vector<int32_t> rows;
    const int32_t heaviest = aflh::row_events_estimates(*sc, *sw, rows);
    out[0] = C.pool;
    aflh::pool_split(C, heaviest, out[1], out[2]);
    for (size_t r = 0; r < rows.size(); ++r) {
        out[3 + 3 * r] = rows[r];
        aflh::pool_split(C, rows[r], out[4 + 3 * r], out[5 + 3 * r]);
    }
    return 0;
}
