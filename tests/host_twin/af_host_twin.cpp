// CPU debugging twin of the replica engine -- TEST INFRASTRUCTURE ONLY.
//
// Compiles asyncflow_b200/csrc/af_core.cuh (the SAME state machine the CUDA kernel
// runs) for the host with a "warp" of one lane, so that the engine's event
// semantics can be checked against oracle/des_port.py in the CPU-only test tier
// (`pytest -m "not gpu"`) of a container that has no GPU.  It is built into
// tests/host_twin/_build/ and loaded only by tests/; the product package
// (asyncflow_b200/) cannot reach it and has no CPU fallback.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

extern "C" const char* af_twin_last_error() {
    static thread_local std::string e;
    return e.c_str();
}
static std::string g_err;
extern "C" const char* af_twin_error() { return g_err.c_str(); }

extern "C" int af_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }

extern "C" double af_twin_hist_percentile(const uint32_t* hist, uint64_t n, double q, double lat_min, double lat_max) {
    return afh::hist_percentile(hist, n, q, lat_min, lat_max);
}

extern "C" int af_twin_run(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                           uint64_t seed, uint64_t replica_begin, uint64_t n,
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
    std::vector<unsigned char> ws((size_t)L.warp_bytes + 64);
    unsigned char* base = (unsigned char*)(((uintptr_t)ws.data() + 15) & ~(uintptr_t)15);
    for (uint64_t r = 0; r < n; ++r) {
        afc::State& W = *reinterpret_cast<afc::State*>(base);
        afc::bind(W, base, 0);
        afc::run_replica(W, r);
        if (L.collect_hist && stats) {
            stats[r].p50 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 50.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p95 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 95.0, stats[r].lat_min, stats[r].lat_max);
            stats[r].p99 = afh::hist_percentile(hist + r * AF_HIST_BINS, stats[r].completed, 99.0, stats[r].lat_min, stats[r].lat_max);
        }
    }
    return AF_OK;
}

// af_run splits a lane's shared memory by aflh::pending_events_estimate(); the twin splits evenly unless a test sets
// the estimate it wants the next af_twin_run_lane calls to use (0 = even split)
static int32_t g_ev_need = 0;
extern "C" void af_twin_set_ev_need(int32_t ev_need) { g_ev_need = ev_need < 0 ? 0 : ev_need; }

// The thread-per-replica engine (af_lane.cuh) as a "warp" of one lane.  `lane_bytes` = the lane's share of
// shared memory: small values push the tiered tables (events, requests, now-queue) into their second tier.
extern "C" int af_twin_run_lane(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfOptions* opt,
                                int32_t lane_bytes, uint64_t seed, uint64_t replica_begin, uint64_t n,
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
    if (lane_bytes < aflh::min_lane_bytes(*sc, T)) lane_bytes = aflh::min_lane_bytes(*sc, T);   // (the engine lowers its occupancy instead)
    if (!aflh::make_cfg(*sc, *opt, T, lane_bytes, afh::trace_tick_capacity(*sc), afl::LANES, C, g_ev_need)) { g_err = "lane engine: tables do not fit the lane's shared memory"; return AF_ERR_INVALID; }
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

// the host-side estimate that splits a lane's shared memory between events and request records (af_run)
extern "C" int af_twin_pending_events_estimate(const AfScenario* sc, const AfSweep* sw) { return aflh::pending_events_estimate(*sc, sw); }
// ... and the split it leads to for a given per-lane budget: out = {ev_s, rq_s}
extern "C" int af_twin_lane_split(const AfScenario* sc, const AfSweep* sw, int32_t lane_bytes, int32_t use_estimate, int32_t* out) {
    aflh::Tables T; std::string err;
    std::vector<int32_t> alias;
    if (sw) alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    if (!aflh::build_tables(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0, sw ? alias.data() : nullptr, T, err)) return -1;
    AfOptions o; memset(&o, 0, sizeof o); o.event_capacity = aflh::LANE_EVENT_CAPACITY; o.request_capacity = aflh::LANE_REQUEST_CAPACITY;
    afl::Cfg C; memset(&C, 0, sizeof C);
    if (!aflh::make_cfg(*sc, o, T, lane_bytes, 0, 32, C, use_estimate ? aflh::pending_events_estimate(*sc, sw) : 0)) return -2;
    out[0] = C.ev_s; out[1] = C.rq_s;
    return 0;
}

// sizeof() of every ABI struct as the C++ compiler lays it out (tests/test_capi.py)
extern "C" int af_twin_sizeof(int which) {
    switch (which) {
    case 0: return (int)sizeof(AfEdge);
    case 1: return (int)sizeof(AfServer);
    case 2: return (int)sizeof(AfEndpoint);
    case 3: return (int)sizeof(AfStep);
    case 4: return (int)sizeof(AfSpikeMark);
    case 5: return (int)sizeof(AfOutageMark);
    case 6: return (int)sizeof(AfScenario);
    case 7: return (int)sizeof(AfSweepColumn);
    case 8: return (int)sizeof(AfSweep);
    case 9: return (int)sizeof(AfOptions);
    case 10: return (int)sizeof(AfReplicaStats);
    default: return -1;
    }
}
