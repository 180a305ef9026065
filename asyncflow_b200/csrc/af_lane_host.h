// Host side of the thread-per-replica engine (af_lane.cuh): the read-only scenario tables with the
// sweep's column map folded in, and the launch configuration (shared-memory layout of a warp, tier
// sizes).  Shared by the CUDA engine (af_engine.cu) and the CPU-only debugging twin (tests/host_twin).
#pragma once
#include <string>
#include <vector>
#include "af_lane.cuh"

namespace aflh {

struct Tables {
    std::vector<afl::EdgeP> edges; std::vector<afl::ServerP> servers; std::vector<afl::EndpointP> endpoints;
    std::vector<afl::StepP> steps; std::vector<afl::SpikeP> spikes; std::vector<afl::OutageP> outages;
    std::vector<int32_t> lb; std::vector<afl::ColP> cols;
    int32_t n_row = 0;
};

// Scenario (+ the sweep's columns) -> the kernel's read-only tables.  A column over a field the kernel
// looks up during the run (edge latency parameters, step durations, endpoint RAM, spike amplitudes) gets a
// slot in the lane's row copy; a column over a field consumed at the start of a replica (users, cores, RAM)
// does not.  Two columns over the same (field, index): the later one wins, as in af_core.cuh::load_params.
inline bool build_tables(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols, const int32_t* alias, Tables& t, std::string& err) {
    t = Tables();
    t.edges.resize((size_t)s.n_edges);
    for (int i = 0; i < s.n_edges; ++i) {
        const AfEdge& a = s.edges[i]; afl::EdgeP& e = t.edges[(size_t)i];
        e.mean = a.mean; e.sigma = a.sigma; e.dropout = a.dropout;
        e.meta = (uint32_t)a.dist | ((uint32_t)a.target_kind << 3) | ((uint32_t)a.target_index << 5);
        e.c_mean = e.c_sigma = e.c_drop = -1; e.pad = 0; e.pad2[0] = e.pad2[1] = 0;
    }
    t.servers.resize((size_t)s.n_servers);
    for (int i = 0; i < s.n_servers; ++i) {
        const AfServer& a = s.servers[i]; afl::ServerP& v = t.servers[(size_t)i];
        v.cpu_cores = a.cpu_cores; v.ram_mb = a.ram_mb; v.out_edge = (uint32_t)a.out_edge;
        v.ep_begin = (uint32_t)a.endpoint_begin; v.n_ep = (uint32_t)a.n_endpoints; v.c_cores = v.c_ram = -1; v.pad = 0;
    }
    t.endpoints.resize((size_t)s.n_endpoints);
    for (int i = 0; i < s.n_endpoints; ++i) {
        const AfEndpoint& a = s.endpoints[i]; afl::EndpointP& p = t.endpoints[(size_t)i];
        p.step_begin = (uint32_t)a.step_begin; p.n_steps = (uint32_t)a.n_steps; p.total_ram = (uint32_t)a.total_ram; p.c_ram = -1;
    }
    t.steps.resize((size_t)s.n_steps);
    for (int i = 0; i < s.n_steps; ++i) { t.steps[(size_t)i].dur = s.steps[i].duration; t.steps[(size_t)i].kind = (uint32_t)s.steps[i].kind; t.steps[(size_t)i].c_dur = -1; }
    t.spikes.resize((size_t)s.n_spike_marks);
    for (int i = 0; i < s.n_spike_marks; ++i) {
        afl::SpikeP& p = t.spikes[(size_t)i];
        p.fire = s.spike_marks[i].fire_time; p.delta = s.spike_marks[i].delta; p.edge = (uint32_t)s.spike_marks[i].edge; p.c_delta = -1; p.pad[0] = p.pad[1] = 0;
    }
    t.outages.resize((size_t)s.n_outage_marks);
    for (int i = 0; i < s.n_outage_marks; ++i) { t.outages[(size_t)i].fire = s.outage_marks[i].fire_time; t.outages[(size_t)i].lb_edge = s.outage_marks[i].lb_edge; t.outages[(size_t)i].down = s.outage_marks[i].down; }
    t.lb.assign(s.lb_edges, s.lb_edges + s.n_lb_edges);
    t.cols.resize((size_t)n_cols);
    int32_t n_row = 0;
    for (int32_t c = 0; c < n_cols; ++c) {
        afl::ColP& k = t.cols[(size_t)c];
        k.field = cols[c].field; k.index = cols[c].index; k.slot = -1; k.pad = 0; k.base = 0.0;
        const int32_t i = k.index;
        // a column whose values repeat an earlier looked-up column's in every row shares that column's slot
        // (configs[2] sweeps all six edges with one RTT array and one jitter array: 2 slots, not 12)
        const int32_t shared = alias && alias[c] >= 0 ? t.cols[(size_t)alias[c]].slot : -1;
#define AFLH_SLOT() (shared >= 0 ? shared : n_row++)
        switch (k.field) {
        case AF_FIELD_USERS_MEAN: k.base = s.users_mean; break;
        case AF_FIELD_USERS_SIGMA: k.base = s.users_sigma; break;
        case AF_FIELD_RATE_PER_USER: k.base = s.rate_per_user; break;
        case AF_FIELD_SERVER_CPU_CORES: k.base = s.servers[i].cpu_cores; break;
        case AF_FIELD_SERVER_RAM_MB: k.base = s.servers[i].ram_mb; break;
        case AF_FIELD_EDGE_MEAN: k.slot = AFLH_SLOT(); k.base = s.edges[i].mean; t.edges[(size_t)i].c_mean = (int16_t)k.slot; break;
        case AF_FIELD_EDGE_SIGMA: k.slot = AFLH_SLOT(); k.base = s.edges[i].sigma; t.edges[(size_t)i].c_sigma = (int16_t)k.slot; break;
        case AF_FIELD_EDGE_DROPOUT: k.slot = AFLH_SLOT(); k.base = s.edges[i].dropout; t.edges[(size_t)i].c_drop = (int16_t)k.slot; break;
        case AF_FIELD_STEP_DURATION: k.slot = AFLH_SLOT(); k.base = s.steps[i].duration; t.steps[(size_t)i].c_dur = k.slot; break;
        case AF_FIELD_ENDPOINT_RAM: k.slot = AFLH_SLOT(); k.base = s.endpoints[i].total_ram; t.endpoints[(size_t)i].c_ram = k.slot; break;
        case AF_FIELD_SPIKE_DELTA: k.slot = AFLH_SLOT(); k.base = s.spike_marks[i].delta < 0.0 ? -s.spike_marks[i].delta : s.spike_marks[i].delta;
                                   t.spikes[(size_t)i].c_delta = k.slot; break;
        default: err = "sweep: unknown field id"; return false;
        }
#undef AFLH_SLOT
    }
    if (n_row > 32000) { err = "sweep: too many looked-up columns for the lane engine"; return false; }
    t.n_row = n_row;
    return true;
}

// alias[c] = the first earlier column whose values equal column c's in every row, or -1
inline std::vector<int32_t> column_aliases(const double* values, uint64_t n_rows, int32_t n_cols) {
    std::vector<int32_t> alias((size_t)n_cols, -1);
    for (int32_t c = 1; c < n_cols; ++c)
        for (int32_t a = 0; a < c && alias[(size_t)c] < 0; ++a) {
            if (alias[(size_t)a] >= 0) continue;                 // compare with class representatives only
            uint64_t r = 0;
            while (r < n_rows && values[r * (uint64_t)n_cols + (uint64_t)c] == values[r * (uint64_t)n_cols + (uint64_t)a]) ++r;
            if (r == n_rows) alias[(size_t)c] = a;
        }
    return alias;
}

// How many pending events a replica typically holds: Little's law -- requests in flight = arrival rate x time in
// system (`edge`: the longest mean edge latency, `steps`: the longest endpoint), one pending event each, plus the
// generator's and the injection timelines' own.  Only used to split a lane's shared memory (a wrong guess costs speed,
// not results).
inline int32_t littles_law_events(const AfScenario& s, double users, double rate, double edge, double steps) {
    const int hops = s.n_lb_edges > 0 ? 4 : 3;           // generator -> client -> [LB ->] server -> client
    const double in_flight = users * rate * (hops * edge + steps);
    const double need = in_flight + 6.0;
    return need > 100000.0 ? 100000 : (int32_t)need;
}
inline double longest_edge(const AfScenario& s) {
    double edge = 0.0;
    for (int i = 0; i < s.n_edges; ++i) if (s.edges[i].mean > edge && s.edges[i].dist != AF_DIST_LOG_NORMAL) edge = s.edges[i].mean;
    return edge;
}
// the longest endpoint: step durations from `dur` (one per step)
inline double longest_endpoint(const AfScenario& s, const double* dur) {
    double steps = 0.0;
    for (int e = 0; e < s.n_endpoints; ++e) {
        double d = 0.0;
        for (int k = 0; k < s.endpoints[e].n_steps; ++k) d += dur[s.endpoints[e].step_begin + k];
        if (d > steps) steps = d;
    }
    return steps;
}
// ... of the scenario, with the sweep's largest users, rates and edge means (the launch's heaviest replica at most)
inline int32_t pending_events_estimate(const AfScenario& s, const AfSweep* sw) {
    double users = s.users_mean, rate = s.rate_per_user, edge = longest_edge(s);
    std::vector<double> dur((size_t)s.n_steps);
    for (int k = 0; k < s.n_steps; ++k) dur[(size_t)k] = s.steps[k].duration;
    const double steps = longest_endpoint(s, dur.data());
    if (sw)
        for (int c = 0; c < sw->n_columns; ++c) {
            const int f = sw->columns[c].field;
            if (f != AF_FIELD_USERS_MEAN && f != AF_FIELD_RATE_PER_USER && f != AF_FIELD_EDGE_MEAN) continue;
            double mx = 0.0;
            for (uint64_t r = 0; r < sw->n_rows; ++r) { const double v = sw->values[r * (uint64_t)sw->n_columns + (uint64_t)c]; if (v > mx) mx = v; }
            if (f == AF_FIELD_USERS_MEAN) users = mx; else if (f == AF_FIELD_RATE_PER_USER) rate = mx; else if (mx > edge) edge = mx;
        }
    return littles_law_events(s, users, rate, edge, steps);
}
// ... of every row of the sweep, on the row's own values (swept users, rate, edge means, step durations): out[r].
// The lane kernel splits each replica's pool by its row's estimate.  Returns the largest.
inline int32_t row_events_estimates(const AfScenario& s, const AfSweep& sw, std::vector<int32_t>& out) {
    out.assign((size_t)sw.n_rows, 0);
    std::vector<double> mean((size_t)s.n_edges), dur((size_t)s.n_steps);
    bool per_row_steps = false;
    for (int c = 0; c < sw.n_columns; ++c) per_row_steps = per_row_steps || sw.columns[c].field == AF_FIELD_STEP_DURATION;
    for (int k = 0; k < s.n_steps; ++k) dur[(size_t)k] = s.steps[k].duration;
    double steps = longest_endpoint(s, dur.data());
    int32_t mx = 0;
    for (uint64_t r = 0; r < sw.n_rows; ++r) {
        const double* row = sw.values + r * (uint64_t)sw.n_columns;
        double users = s.users_mean, rate = s.rate_per_user;
        for (int i = 0; i < s.n_edges; ++i) mean[(size_t)i] = s.edges[i].mean;
        if (per_row_steps) for (int k = 0; k < s.n_steps; ++k) dur[(size_t)k] = s.steps[k].duration;
        for (int c = 0; c < sw.n_columns; ++c) {            // (two columns over one field: the later one wins, as in the kernels)
            const int i = sw.columns[c].index;
            switch (sw.columns[c].field) {
            case AF_FIELD_USERS_MEAN: users = row[c]; break;
            case AF_FIELD_RATE_PER_USER: rate = row[c]; break;
            case AF_FIELD_EDGE_MEAN: mean[(size_t)i] = row[c]; break;
            case AF_FIELD_STEP_DURATION: dur[(size_t)i] = row[c]; break;
            default: break;
            }
        }
        double edge = 0.0;
        for (int i = 0; i < s.n_edges; ++i) if (mean[(size_t)i] > edge && s.edges[i].dist != AF_DIST_LOG_NORMAL) edge = mean[(size_t)i];
        if (per_row_steps) steps = longest_endpoint(s, dur.data());
        const int32_t need = littles_law_events(s, users, rate, edge, steps);
        out[(size_t)r] = need;
        if (need > mx) mx = need;
    }
    return mx;
}

constexpr int32_t LANE_EVENT_CAPACITY = 512;      // defaults of the lane engine's global tiers (AfOptions fields <= 0)
constexpr int32_t LANE_REQUEST_CAPACITY = 2048;

// smallest per-lane budget make_cfg() accepts for this scenario (4 events, 2 requests + the hot fixed tables)
// the lane's fixed tables in shared memory: spike offsets + sweep-row copy (64-bit), connection counts, server levels,
// LB order, the gauges' dirty bits (32-bit).  (The gauges' sums / maxima and the send counters are write-only: global tier.)
inline int32_t fixed_lane_bytes(const AfScenario& s, const Tables& t) {
    const int32_t n_series = 3 * s.n_servers + s.n_edges;
    const int32_t fix64 = (s.n_spike_marks > 0 ? s.n_edges : 0) + t.n_row;
    const int32_t fix32 = s.n_edges + afl::SV_WORDS * s.n_servers + s.n_lb_edges + (n_series + 31) / 32;
    return 8 * fix64 + 4 * fix32;
}
constexpr int32_t MIN_DYNAMIC_BYTES = 16 * 4 + 36 * 2;      // (a pool of 8 elements: 4 heap entries, 2 records and more)
// smallest per-lane budget make_cfg() accepts for this scenario
inline int32_t min_lane_bytes(const AfScenario& s, const Tables& t) { return fixed_lane_bytes(s, t) + MIN_DYNAMIC_BYTES; }

// The split of the lane's pool a replica with an estimated `need` pending events gets: {ev_s, rq_s}
inline void pool_split(const afl::Cfg& C, int32_t need, int32_t& ev_s, int32_t& rq_s) {
    ev_s = afl::pool_events(C.pool, C.ev_lo, C.rq_floor, C.ev_total, C.rq_total, need);
    rq_s = C.pool - ev_s;
}

// `ev_need`: pending-events estimate of the replicas the launch has no per-replica estimate for (Cfg.row_need; 0: the
// even split -- the twin's default); `rq_min`: the record slots that stay in shared memory when the events take more
// than the even split.
// The launch configuration for a budget of `lane_bytes` of shared memory per lane (= per replica in
// flight).  Returns false when even the smallest tiers do not fit: the topology is too wide for this
// engine at this occupancy (the caller lowers the occupancy or takes the warp-per-replica engine).
// `lanes` = lanes of a warp in the code that will RUN the configuration: 32 for the CUDA kernel, 1 for the host twin
// (afl::LANES is a property of the compilation pass, and the host pass of a .cu file sees 1).
inline bool make_cfg(const AfScenario& s, const AfOptions& o, const Tables& t, int32_t lane_bytes, int32_t trace_tick_cap, int32_t lanes, afl::Cfg& C, int32_t ev_need = 0, int32_t rq_min = 2) {
    C.n_edges = s.n_edges; C.n_servers = s.n_servers; C.n_endpoints = s.n_endpoints; C.n_steps = s.n_steps;
    C.n_lb_edges = s.n_lb_edges; C.lb_algo = s.lb_algo; C.gen_edge = s.gen_edge; C.client_edge = s.client_edge;
    C.n_spike = s.n_spike_marks; C.n_outage = s.n_outage_marks;
    C.users_dist = s.users_dist; C.window_s = s.window_s; C.horizon_s = s.horizon_s; C.metrics_mask = s.metrics_mask;
    C.users_mean = s.users_mean; C.users_sigma = s.users_sigma; C.rate_per_user = s.rate_per_user; C.sample_period = s.sample_period;
    C.n_series = 3 * s.n_servers + s.n_edges;
    C.n_sweep_cols = (int32_t)t.cols.size(); C.n_row = t.n_row;
    C.collect_hist = o.collect_histogram; C.collect_thr = o.collect_throughput;
    C.trace_replicas = o.trace_replicas; C.trace_clock_cap = o.trace_clock_capacity; C.trace_tick_cap = trace_tick_cap;
    C.redo = 0;
    int32_t ev_total = o.event_capacity > 0 ? o.event_capacity : LANE_EVENT_CAPACITY;
    int32_t rq_total = o.request_capacity > 0 ? o.request_capacity : LANE_REQUEST_CAPACITY;
    if (rq_total > (int32_t)afl::SLOT_MASK) rq_total = (int32_t)afl::SLOT_MASK;
    // fixed part of a lane's shared memory
    const int32_t fix64 = (C.n_spike > 0 ? C.n_edges : 0) + C.n_row;
    C.n_dirty = (C.n_series + 31) / 32;
    const int32_t fix32 = C.n_edges + afl::SV_WORDS * C.n_servers + C.n_lb_edges + C.n_dirty;
    int32_t nq_s = 0;                                // zero-delay items: ties only -- the ring starts in the global tier
    const int32_t rest = lane_bytes - 8 * fix64 - 4 * fix32;
    // the rest is the pool: 16-byte elements shared by the heap and the request records, split per replica
    // (afl::pool_events); it never holds more than both tables can use
    const int32_t rq_cap = rq_total < afl::RQ_BITS ? rq_total : afl::RQ_BITS;
    int32_t pool = rest < 0 ? 0 : rest / 16;
    if (pool > ev_total + rq_cap) {                  // everything fits: what is left over takes the front of the now-queue
        pool = ev_total + rq_cap;
        nq_s = (rest - 16 * pool) / 8;
        if (nq_s > afl::NQ_TOTAL) nq_s = afl::NQ_TOTAL;
    }
    if (pool < (ev_total < 4 ? ev_total : 4) + (rq_total < 2 ? rq_total : 2)) return false;
    // The even split -- at nominal load a request in flight owns one pending event, plus the arrival and the two
    // timelines -- is the fewest heap entries a replica gets: a replica whose events fit does not need the record slots
    // beyond it.  Above it the heap takes what the replica's estimate asks for, down to `rq_min` (>= 2) record slots.
    C.pool = pool; C.ev_lo = pool - (pool - 4) / 2; C.rq_floor = rq_min < 2 ? 2 : rq_min;
    C.row_need = nullptr; C.need_first = 0; C.need_rows = 0;
    C.ev_total = ev_total; C.rq_total = rq_total; C.nq_s = nq_s;
    pool_split(C, ev_need, C.ev_s, C.rq_s);
    C.n128 = pool;
    int32_t e = 0;
    C.o64_nq = e; e += nq_s;
    C.o64_spike = e; e += C.n_spike > 0 ? C.n_edges : 0;
    C.o64_row = e; e += C.n_row;
    C.n64 = e;
    int32_t w = 0;
    C.o32_conn = w; w += C.n_edges;
    C.o32_srv = w; w += afl::SV_WORDS * C.n_servers;
    C.o32_lb = w; w += C.n_lb_edges;
    C.o32_dirty = w; w += C.n_dirty;
    C.n32 = w;
    C.warp_bytes = (C.n128 * 16 + C.n64 * 8 + C.n32 * 4) * lanes;
    // global tier: 128-bit region (events, request records), 64-bit region (now-queue), 32-bit region (links, cold words).
    // A replica keeps ev_s + rq_s = pool entries in shared memory whatever its split: heap entries [ev_s, ev_total) at
    // elements [0, ev_total - ev_s), record slots [rq_s, rq_total) right after them
    C.gi_rq = ev_total - pool;
    C.gn128 = ev_total + rq_total - pool;
    C.gi_nq = 0 - nq_s;
    C.gi_acc = afl::NQ_TOTAL - nq_s;
    C.gn64 = C.gi_acc + C.n_series;
    int32_t hcount = rq_total;                       // the `next` link of every record slot
    C.g32_cold = hcount;
    C.c_srvq = 0; C.c_inbox = C.c_srvq + afl::SQ_WORDS * C.n_servers; C.c_drop = C.c_inbox + afl::IB_WORDS * (C.n_servers + 2);
    hcount += C.c_drop + C.n_edges;
    C.gi_smax = hcount; hcount += C.n_series;
    C.gi_sent = hcount; hcount += C.n_edges;
    C.gn32 = hcount;
    C.gwarp_bytes = ((uint64_t)C.gn128 * 16 + (uint64_t)C.gn64 * 8 + (uint64_t)C.gn32 * 4) * (uint64_t)lanes;
    return true;
}

}  // namespace aflh
