// CPU twin of both replica engines -- TEST INFRASTRUCTURE ONLY.
//
// Compiles the state machines the CUDA kernels run -- af_lane.cuh (thread per replica) and af_core.cuh (warp per
// replica) -- for the host, with a "warp" of one lane, so that the CPU-only test tier can check them against
// oracle/des_port.py and the GPU tier can check the device against them.  Each runner sets up one launch the way af_run
// does (pool splits, pull order, per-tick / latency / distribution bands, occupancy integrals, the lean build of the
// loop, the second pass's re-run of flagged replicas) from its own restatement of that arithmetic, never af_run's code:
// it is the independent reference af_run is compared against.  Built into tests/host_twin/_build/ and loaded by
// tests/twin.py only; the product package cannot reach it and has no CPU fallback.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

// One launch's knobs (tests/twin.py mirrors it).  Band rows are zeroed by the caller; groups are group_of[i] for replica
// band_first + i.
struct TwinLaunch {
    uint64_t sweep_first;       // the replica sweep row 0 describes
    int32_t lane_bytes;         // lane engine: the lane's share of shared memory (raised to what the tables need)
    int32_t ev_need;            // lane engine: the pending-events estimate the pool is split by (< 0: the scenario's)
    int32_t split;              // lane engine: 0 every replica by ev_need, 1 each sweep row by its own estimate (as
                                // af_run), 2 a random split per replica drawn from split_seed and the replica id
    int32_t lean;               // lane engine: the lean build of the loop
    uint64_t split_seed;
    const uint32_t* order;      // lane engine: the pull order, a permutation of [0, n) (nullptr: id order)
    int32_t sampled;            // per-tick bands into band_rows: (n_groups + 1) x (1 + 2 n_series) x (ticks + 1) u64
    int32_t lat_window;         // latency bands of this many seconds into lat_rows: (n_groups + 1) x windows x LAT_ROW
    const uint32_t* group_of;
    uint64_t band_first, band_n;
    uint32_t n_groups;
    int32_t n_dist;             // distribution bands of dist_series[0 .. n_dist) into dist_rows
    uint64_t* band_rows;
    uint32_t* band_from;        // per local replica: the tick a stopped one stopped at (the lane engine writes it)
    uint64_t* lat_rows;
    uint32_t* lat_from;         // per local replica: the completions a stopped one added (the lane engine writes it)
    const int32_t* dist_series;
    int32_t dist_capacity;      // the request capacity the bins are sized by (0: opt's), as af_run sizes both passes'
    int32_t occ_bits;           // > 0: occupancy integrals with this many fraction bits into occ[n][5 n_servers + n_edges]
    uint32_t* dist_rows;
    uint64_t* occ;
    const uint32_t* redo;       // warp engine: re-run these local indices as af_run's second pass (nullptr: every
    uint64_t n_redo;            // replica, first-hand); their bands continue from band_from / lat_from
};

struct TwinOutputs {
    AfReplicaStats* stats; uint32_t* sent; uint32_t* dropped; uint32_t* hist; uint32_t* thr;
    uint64_t* samp_sum; uint32_t* samp_max; double* trace_clocks; uint32_t* trace_series; uint32_t* trace_counts;
};

static std::string g_err;
extern "C" const char* af_twin_error() { return g_err.c_str(); }

static int report(bool ok, const std::string& w, char* why, int why_cap) {
    snprintf(why, (size_t)why_cap, "%s", w.c_str());
    return ok ? 1 : 0;
}

static uint64_t swept_ram(const AfSweep* sw, int32_t& server) {
    server = -1;
    return sw ? afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, server) : 0;
}

static uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// ---- the launch checks af_bands_upload / af_bands_configure / af_dist_bands_configure / af_run apply ----------------
extern "C" int af_twin_trace_tick_capacity(const AfScenario* sc) { return afh::trace_tick_capacity(*sc); }
extern "C" uint32_t af_twin_ticks(const AfScenario* sc) { return afh::band_ticks(*sc); }
// 1 when the band rows can hold every tick, else 0 and why
extern "C" int af_twin_ticks_fit(const AfScenario* sc, char* why, int why_cap) {
    uint32_t ticks = 0;
    std::string w;
    const bool ok = afh::band_ticks_fit(*sc, ticks, w);
    return report(ok, w, why, why_cap);
}
// 1 when a group of `group` replicas cannot wrap the u64 sums of squares, else 0 and the deciding bound in `what`
extern "C" int af_twin_sumsq_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t group,
                                  uint64_t* bound, char* what, int what_cap) {
    int32_t server;
    const uint64_t ram = swept_ram(sw, server);
    std::string w;
    *bound = afh::band_gauge_bound(*sc, *opt, ram, server, w);
    return report(afh::band_sumsq_fits(group, *bound), w, what, what_cap);
}
// 1 when latency bands of `window_s` seconds over n_groups groups fit a device of mem_total bytes, else 0 and why
extern "C" int af_twin_lat_fits(int32_t window_s, int32_t horizon_s, uint64_t n_groups, uint64_t mem_total, char* why,
                                int why_cap) {
    std::string w;
    const bool ok = afh::lat_bands_fit(window_s, horizon_s, n_groups, mem_total, w);
    return report(ok, w, why, why_cap);
}
// 1 when the series are valid and the rows of n_groups groups fit a device of mem_total bytes (ticks and bins set)
extern "C" int af_twin_dist_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, const int32_t* series,
                                 int32_t n, uint64_t n_groups, uint64_t mem_total, uint32_t* ticks, uint32_t* bins,
                                 char* why, int why_cap) {
    std::string w;
    int32_t server;
    const uint64_t ram = swept_ram(sw, server);
    const bool ok = afh::dist_series_check(*sc, series, n, w)
                    && afh::dist_bands_fit(*sc, *opt, ram, server, n_groups, (uint64_t)n, mem_total, *ticks, *bins, w);
    return report(ok, w, why, why_cap);
}
// 1 when occupancy integrals of frac_bits fraction bits fit the launch, else 0 and why
extern "C" int af_twin_occ_fits(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, int32_t frac_bits,
                                char* why, int why_cap) {
    std::string w;
    int32_t server;
    const uint64_t ram = swept_ram(sw, server);
    const bool ok = afh::occ_fits(*sc, *opt, ram, server, frac_bits, w);
    return report(ok, w, why, why_cap);
}

// ---- the device's number formats, on the host ----------------------------------------------------------------------
extern "C" uint32_t af_twin_gauge_bin(uint32_t v) { return afr::gauge_bin(v); }
extern "C" uint64_t af_twin_fixed32(double lat) { return afr::lat_fixed32(lat); }
extern "C" int32_t af_twin_hist_bin(double lat) { return afr::hist_bin(lat); }
extern "C" int32_t af_twin_frac_bits(uint64_t bound, int32_t horizon_s) { return afh::occ_frac_bits(bound, horizon_s); }
extern "C" uint64_t af_twin_occ_fixed(double rest, int32_t frac_bits) { return afr::occ_fixed(rest, ldexp(1.0, frac_bits)); }
extern "C" double af_twin_hist_percentile(const uint32_t* hist, uint64_t n, double q, double lat_min, double lat_max) {
    return afh::hist_percentile(hist, n, q, lat_min, lat_max);
}
extern "C" int af_twin_lean_qualifies(const AfScenario* sc, int32_t trace_replicas) {
    return aflh::lean_launch(*sc, trace_replicas) ? 1 : 0;
}

// ---- the lane engine's shared-memory pool split, as af_run chooses it ------------------------------------------------
extern "C" int af_twin_pending_events_estimate(const AfScenario* sc, const AfSweep* sw) { return aflh::pending_events_estimate(*sc, sw); }

static bool split_cfg(const AfScenario* sc, const AfSweep* sw, int32_t lane_bytes, int32_t ev_need, aflh::Tables& T,
                      afl::Cfg& C) {
    std::string err;
    std::vector<int32_t> alias;
    if (sw) alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    if (!aflh::build_tables(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0, sw ? alias.data() : nullptr, T, err))
        return false;
    AfOptions o; memset(&o, 0, sizeof o); o.event_capacity = aflh::LANE_EVENT_CAPACITY; o.request_capacity = aflh::LANE_REQUEST_CAPACITY;
    memset(&C, 0, sizeof C);
    return aflh::make_cfg(*sc, o, T, lane_bytes, 0, 32, C, ev_need);
}
// the split a per-lane budget leads to (the CUDA engine's capacities): out = {ev_s, rq_s}
extern "C" int af_twin_lane_split(const AfScenario* sc, const AfSweep* sw, int32_t lane_bytes, int32_t use_estimate, int32_t* out) {
    aflh::Tables T; afl::Cfg C;
    if (!split_cfg(sc, sw, lane_bytes, use_estimate ? aflh::pending_events_estimate(*sc, sw) : 0, T, C)) return -1;
    out[0] = C.ev_s; out[1] = C.rq_s;
    return 0;
}
// The split af_run gives each row of `sw` for a lane of `lane_bytes`, and the one it reports for the launch
// (AfRunPasses: the heaviest row's).  out[0] = pool, out[1], out[2] = the reported split, out[3 + 3r ...] = {estimate,
// ev_s, rq_s} of row r
extern "C" int af_twin_row_splits(const AfScenario* sc, const AfSweep* sw, int32_t lane_bytes, int32_t* out) {
    aflh::Tables T; afl::Cfg C;
    if (!split_cfg(sc, sw, lane_bytes, aflh::pending_events_estimate(*sc, nullptr), T, C)) return -1;
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

// ---- the runners ------------------------------------------------------------------------------------------------------
static bool band_checks(const AfScenario* sc, const TwinLaunch& k) {
    uint32_t ticks = 0;
    if (k.sampled && !afh::band_ticks_fit(*sc, ticks, g_err)) return false;
    if (k.lat_window && !afh::lat_bands_fit(k.lat_window, sc->horizon_s, k.n_groups, ~0ull, g_err)) return false;
    return true;
}

// Distribution bands: each series' slot (-1: not banded), the bins af_run sizes for these options and sweep, and the
// words of one series' rows.
static bool dist_setup(const AfScenario* sc, const AfOptions* opt, const AfSweep* sw, const TwinLaunch& k,
                       int32_t n_series, std::vector<int32_t>& slot, uint32_t& bins, uint64_t& series_words) {
    if (!afh::dist_series_check(*sc, k.dist_series, k.n_dist, g_err)) return false;
    int32_t server;
    const uint64_t ram = swept_ram(sw, server);
    AfOptions o = *opt;
    if (k.dist_capacity > 0) o.request_capacity = k.dist_capacity;
    uint32_t ticks = 0;
    std::string w;
    afh::dist_bands_fit(*sc, o, ram, server, 0, (uint64_t)k.n_dist, ~0ull, ticks, bins, w);
    slot.assign((size_t)n_series, -1);
    for (int32_t j = 0; j < k.n_dist; ++j) slot[(size_t)k.dist_series[j]] = j;
    series_words = ((uint64_t)ticks + 1) * bins;
    return true;
}

static void percentiles(const TwinOutputs& o, uint64_t r) {
    AfReplicaStats& s = o.stats[r];
    const uint32_t* h = o.hist + r * AF_HIST_BINS;
    s.p50 = afh::hist_percentile(h, s.completed, 50.0, s.lat_min, s.lat_max);
    s.p95 = afh::hist_percentile(h, s.completed, 95.0, s.lat_min, s.lat_max);
    s.p99 = afh::hist_percentile(h, s.completed, 99.0, s.lat_min, s.lat_max);
}

// run_lane<sampled, latency, lean, dist, occ> with the flags f[0 .. 5) as its template arguments
template <bool... B, class P>
static void run_lane_as(const afl::Mem& m, P pull, const bool (&f)[5]) {
    if constexpr (sizeof...(B) == 5) afl::run_lane<B...>(m, pull, [](bool alive) { return alive; });
    else if (f[sizeof...(B)]) run_lane_as<B..., true>(m, pull, f);
    else run_lane_as<B..., false>(m, pull, f);
}

// The thread-per-replica engine over replicas [begin, begin + n), as one lane pulling them.
extern "C" int af_twin_run_lane(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t seed,
                                uint64_t begin, uint64_t n, const TwinLaunch* launch, const TwinOutputs* out) {
    const TwinLaunch& k = *launch;
    const TwinOutputs& o = *out;
    if (!afh::validate(*sc, g_err) || !band_checks(sc, k)) return AF_ERR_INVALID;
    aflh::Tables T;
    std::vector<int32_t> alias;
    const bool all_rows = sw && begin >= k.sweep_first && begin + n - k.sweep_first <= sw->n_rows;
    if (all_rows) alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    if (!aflh::build_tables(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0, all_rows ? alias.data() : nullptr, T, g_err)) return AF_ERR_INVALID;
    afl::Cfg& C = afl::h_cfg;
    memset(&C, 0, sizeof C);
    const int32_t lane_bytes = k.lane_bytes < aflh::min_lane_bytes(*sc, T) ? aflh::min_lane_bytes(*sc, T) : k.lane_bytes;   // (the engine lowers its occupancy instead)
    const int32_t ev_need = k.ev_need < 0 ? aflh::pending_events_estimate(*sc, nullptr) : k.ev_need;
    if (!aflh::make_cfg(*sc, *opt, T, lane_bytes, afh::trace_tick_capacity(*sc), afl::LANES, C, ev_need)) {
        g_err = "lane engine: tables do not fit the lane's shared memory"; return AF_ERR_INVALID;
    }
    if (k.occ_bits > 0) { aflh::add_occupancy(C, afl::LANES, afh::occ_cols(*sc), k.occ_bits); C.occ = k.occ; }
    std::vector<int32_t> need;
    if (k.split == 1) {
        if (sw && sw->n_columns > 0 && sw->n_rows > 0) {
            aflh::row_events_estimates(*sc, *sw, need);
            C.row_need = need.data(); C.need_first = k.sweep_first; C.need_rows = sw->n_rows;
        }
    } else if (k.split == 2) {                        // the estimate that gives the drawn split (ev_lo = 1: any split)
        need.resize((size_t)n);
        const int32_t rq_hi = C.pool - 1 < afl::RQ_BITS ? C.pool - 1 : afl::RQ_BITS;
        const int32_t span = rq_hi - C.rq_floor + 1;
        for (uint64_t r = 0; r < n; ++r) {
            const int32_t rq = span > 0 ? C.rq_floor + (int32_t)(splitmix64(k.split_seed * 0x100000001B3ull + begin + r) % (uint64_t)span) : 1;
            need[(size_t)r] = C.pool - rq;
        }
        C.ev_lo = 1;
        C.row_need = need.data(); C.need_first = begin; C.need_rows = n;
    } else if (k.split != 0) { g_err = "af_twin_run_lane: unknown split mode"; return AF_ERR_INVALID; }
    C.edges = T.edges.data(); C.servers = T.servers.data(); C.endpoints = T.endpoints.data(); C.steps = T.steps.data();
    C.spikes = T.spikes.data(); C.outages = T.outages.data(); C.lb_edges = T.lb.data(); C.cols = T.cols.data();
    if (sw) { C.sweep_vals = sw->values; C.sweep_first = k.sweep_first; C.sweep_rows = sw->n_rows; }
    C.stats = o.stats; C.edge_sent = o.sent; C.edge_dropped = o.dropped; C.hist = o.hist; C.thr = o.thr;
    C.samp_sum = o.samp_sum; C.samp_max = o.samp_max; C.trace_clocks = o.trace_clocks; C.trace_series = o.trace_series;
    C.trace_counts = o.trace_counts;
    C.order = k.order;
    C.seed = seed; C.replica_begin = begin; C.n_replicas = n;
    const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
    C.band_group = k.group_of; C.band_first = k.band_first; C.band_n = k.band_n; C.band_groups = (int32_t)k.n_groups;
    C.band_rows = k.band_rows; C.band_from = k.band_from;
    C.band_group_words = (1 + 2 * (uint64_t)C.n_series) * stride; C.band_stride = (int32_t)stride;
    C.lat_rows = k.lat_rows; C.lat_from = k.lat_from; C.lat_window = k.lat_window;
    C.lat_windows = k.lat_window ? (int32_t)afh::lat_windows(sc->horizon_s, k.lat_window) : 0;
    std::vector<int32_t> slot;
    if (k.n_dist) {
        uint32_t bins = 0;
        if (!dist_setup(sc, opt, sw, k, C.n_series, slot, bins, C.dist_series_words)) return AF_ERR_INVALID;
        C.dist_rows = k.dist_rows; C.dist_slot = slot.data(); C.dist_n = k.n_dist; C.dist_bins = (int32_t)bins;
        C.dist_group_words = (uint64_t)k.n_dist * C.dist_series_words;
    }
    std::vector<uint64_t> smem((size_t)C.warp_bytes / 8 + 2), glob((size_t)(C.gwarp_bytes / 8) + 2);
    afl::afl_smem_host = (unsigned char*)smem.data();
    afl::Mem m;
    m.s128 = 0u; m.s64 = (uint32_t)((size_t)C.n128 * afl::STRIDE128); m.s32 = m.s64 + (uint32_t)((size_t)C.n64 * afl::STRIDE64);
    m.g128 = (unsigned char*)glob.data(); m.g64 = m.g128 + (size_t)C.gn128 * afl::STRIDE128; m.g32 = m.g64 + (size_t)C.gn64 * afl::STRIDE64;
    uint64_t next = 0;                                // the next-th pull gets local index order[next], as in af_lane_kernel
    auto pull = [&]() -> uint64_t { if (next >= n) return ~0ull; const uint64_t i = C.order ? C.order[next] : next; ++next; return i; };
    const bool flags[5] = {k.sampled != 0, k.lat_window != 0, k.lean != 0, k.n_dist > 0, k.occ_bits > 0};
    run_lane_as<>(m, pull, flags);
    if (C.collect_hist && o.stats) for (uint64_t r = 0; r < n; ++r) percentiles(o, r);
    return AF_OK;
}

// The warp-per-replica engine over replicas [begin, begin + n): every one first-hand, or the re-run of k.redo.
extern "C" int af_twin_run_warp(const AfScenario* sc, const AfSweep* sw, const AfOptions* opt, uint64_t seed,
                                uint64_t begin, uint64_t n, const TwinLaunch* launch, const TwinOutputs* out) {
    const TwinLaunch& k = *launch;
    const TwinOutputs& o = *out;
    if (!afh::validate(*sc, g_err) || !band_checks(sc, k)) return AF_ERR_INVALID;
    afc::Layout& L = afc::h_L;
    memset(&L, 0, sizeof L);
    afh::make_layout(*sc, *opt, sw ? sw->n_columns : 0, L);
    afc::Globals& G = afc::h_G;
    memset(&G, 0, sizeof G);
    G.edges = sc->edges; G.servers = sc->servers;
    G.endpoints = sc->endpoints; G.steps = sc->steps;
    G.lb_edges = sc->lb_edges; G.spikes = sc->spike_marks; G.outages = sc->outage_marks;
    if (sw) { G.sweep_cols = sw->columns; G.sweep_vals = sw->values; G.sweep_first = k.sweep_first; G.sweep_rows = sw->n_rows; }
    std::vector<double> sp_t((size_t)(L.ev_total - L.ev_smem) + 1);
    std::vector<uint64_t> sp_k((size_t)(L.ev_total - L.ev_smem) + 1);
    std::vector<afc::ReqRec> sp_r((size_t)(L.rq_total - L.rq_smem) + 1);
    std::vector<uint32_t> sp_n((size_t)(L.rq_total - L.rq_smem) + 1);
    G.spill_ev_time = sp_t.data(); G.spill_ev_key = sp_k.data(); G.spill_rq_rec = sp_r.data(); G.spill_rq_next = sp_n.data();
    G.stats = o.stats; G.edge_sent = o.sent; G.edge_dropped = o.dropped; G.hist = o.hist; G.thr = o.thr;
    G.samp_sum = o.samp_sum; G.samp_max = o.samp_max; G.trace_clocks = o.trace_clocks; G.trace_series = o.trace_series;
    G.trace_counts = o.trace_counts;
    G.seed = seed; G.replica_begin = begin; G.n_replicas = n;
    uint32_t count = (uint32_t)k.n_redo;
    if (k.redo) { G.redo_list = k.redo; G.redo_count = &count; }
    afc::BandArgs band = {};
    band.group = k.group_of; band.first = k.band_first; band.n = k.band_n; band.groups = k.n_groups;
    if (k.occ_bits > 0) { band.occ = k.occ; band.occ_scale = ldexp(1.0, k.occ_bits); }
    if (k.sampled) {
        const uint64_t stride = (uint64_t)afh::band_ticks(*sc) + 1;
        band.rows = k.band_rows;
        band.group_words = (1 + 2 * (uint64_t)L.n_series) * stride; band.stride = (uint32_t)stride;
    }
    if (k.sampled || k.n_dist) {                      // each series' last emitted value, behind the warp's tables
        band.from = k.band_from;
        band.prev_off = L.warp_bytes;
        L.warp_bytes += afc::align_up(4 * L.n_series, 16);
    }
    std::vector<int32_t> slot;
    if (k.n_dist) {
        if (!dist_setup(sc, opt, sw, k, L.n_series, slot, band.dist_bins, band.dist_series_words)) return AF_ERR_INVALID;
        band.dist_rows = k.dist_rows; band.dist_slot = slot.data();
        band.dist_group_words = (uint64_t)k.n_dist * band.dist_series_words;
    }
    if (k.lat_window) {
        band.lat_rows = k.lat_rows; band.lat_from = k.lat_from; band.lat_window = (uint32_t)k.lat_window;
        band.lat_windows = (uint32_t)afh::lat_windows(sc->horizon_s, k.lat_window);
    }
    std::vector<unsigned char> ws((size_t)L.warp_bytes + 64);
    unsigned char* base = (unsigned char*)(((uintptr_t)ws.data() + 15) & ~(uintptr_t)15);
    const uint64_t todo = k.redo ? k.n_redo : n;
    for (uint64_t i = 0; i < todo; ++i) {
        const uint64_t r = k.redo ? k.redo[i] : i;
        afc::State& W = *reinterpret_cast<afc::State*>(base);
        afc::bind(W, base, 0);
        afc::run_replica(W, r, band);
        if (L.collect_hist && o.stats) percentiles(o, r);
    }
    return AF_OK;
}
