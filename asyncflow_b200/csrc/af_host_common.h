// Host-side helpers shared by the CUDA engine (af_engine.cu) and the CPU-only
// debugging twin (tests/host_twin): scenario validation, workspace layout and the
// serial histogram-quantile used to cross-check the device percentile kernel.
#pragma once
#include <math.h>
#include <stdio.h>
#include <algorithm>
#include <string>
#include <vector>
#include "af_core.cuh"

namespace afh {

constexpr int32_t DEFAULT_EVENT_CAPACITY = 2048;
constexpr int32_t DEFAULT_REQUEST_CAPACITY = 16384;
constexpr int32_t DEFAULT_EV_SMEM = 64;
constexpr int32_t DEFAULT_RQ_SMEM = 64;

inline bool validate(const AfScenario& s, std::string& err) {
    char buf[256];
#define AF_CHECK(cond, ...) do { if (!(cond)) { snprintf(buf, sizeof buf, __VA_ARGS__); err = buf; return false; } } while (0)
    AF_CHECK(s.n_edges > 0 && s.n_edges <= (int)afc::AUX_MASK, "n_edges=%d out of range [1,%u]", s.n_edges, afc::AUX_MASK);
    AF_CHECK(s.n_servers > 0 && s.n_servers <= 120, "n_servers=%d out of range [1,120]", s.n_servers);
    AF_CHECK(s.n_endpoints > 0 && s.n_endpoints < 4096, "n_endpoints=%d out of range", s.n_endpoints);
    AF_CHECK(s.n_steps >= 0 && s.n_steps < (1 << 20), "n_steps=%d out of range", s.n_steps);
    AF_CHECK(s.horizon_s >= 1, "horizon_s=%d must be >= 1", s.horizon_s);
    AF_CHECK(s.window_s >= 1, "window_s=%d must be >= 1", s.window_s);
    AF_CHECK(s.sample_period > 0.0, "sample_period must be > 0");
    AF_CHECK(s.users_dist == AF_DIST_POISSON || s.users_dist == AF_DIST_NORMAL, "users_dist=%d unsupported", s.users_dist);
    // a non-finite mean never ends a draw (a Poisson mean of +inf would loop forever in afr::poisson)
    AF_CHECK(isfinite(s.users_mean) && isfinite(s.users_sigma) && isfinite(s.rate_per_user),
             "users: mean=%g sigma=%g rate=%g must be finite", s.users_mean, s.users_sigma, s.rate_per_user);
    AF_CHECK(s.gen_edge >= 0 && s.gen_edge < s.n_edges, "gen_edge out of range");
    AF_CHECK(s.client_edge >= 0 && s.client_edge < s.n_edges, "client_edge out of range");
    AF_CHECK(s.edges && s.servers && s.endpoints, "null topology arrays");
    AF_CHECK(s.n_steps == 0 || s.steps, "null steps");
    bool has_lb_target = false;
    for (int i = 0; i < s.n_edges; ++i) {
        const AfEdge& e = s.edges[i];
        AF_CHECK(e.dist >= 0 && e.dist <= 4, "edge %d: dist=%d", i, e.dist);
        AF_CHECK(e.target_kind >= 0 && e.target_kind <= 2, "edge %d: target_kind=%d", i, e.target_kind);
        if (e.target_kind == AF_TARGET_SERVER)
            AF_CHECK(e.target_index >= 0 && e.target_index < s.n_servers, "edge %d: target server %d", i, e.target_index);
        if (e.target_kind == AF_TARGET_LB) has_lb_target = true;
        AF_CHECK(e.dropout >= 0.0 && e.dropout <= 1.0, "edge %d: dropout", i);
        AF_CHECK(isfinite(e.mean) && isfinite(e.sigma), "edge %d: mean=%g sigma=%g must be finite", i, e.mean, e.sigma);
        AF_CHECK(e.dist != AF_DIST_POISSON || e.mean <= afr::EDGE_POISSON_MEAN_MAX,
                 "edge %d: Poisson mean %g above %g, the largest a request's random-number blocks cover", i, e.mean,
                 afr::EDGE_POISSON_MEAN_MAX);
    }
    if (has_lb_target) {
        AF_CHECK(s.n_lb_edges > 0 && s.lb_edges, "an edge targets the LB but n_lb_edges == 0");
        AF_CHECK(s.lb_algo == AF_LB_ROUND_ROBIN || s.lb_algo == AF_LB_LEAST_CONNECTIONS, "lb_algo=%d", s.lb_algo);
    }
    for (int i = 0; i < s.n_lb_edges; ++i)
        AF_CHECK(s.lb_edges[i] >= 0 && s.lb_edges[i] < s.n_edges, "lb_edges[%d] out of range", i);
    for (int i = 0; i < s.n_servers; ++i) {
        const AfServer& v = s.servers[i];
        AF_CHECK(v.cpu_cores >= 1 && v.ram_mb >= 1, "server %d: resources", i);
        AF_CHECK(v.out_edge >= 0 && v.out_edge < s.n_edges, "server %d: out_edge", i);
        AF_CHECK(v.n_endpoints >= 1 && v.endpoint_begin >= 0 && v.endpoint_begin + v.n_endpoints <= s.n_endpoints,
                 "server %d: endpoint range", i);
        AF_CHECK(v.max_in_service >= 0, "server %d: max_in_service=%d must be >= 0 (0 = no admission limit)", i, v.max_in_service);
        AF_CHECK(isfinite(v.deadline) && v.deadline >= 0.0, "server %d: deadline=%g must be finite and >= 0 (0 = none)", i, v.deadline);
        AF_CHECK(isfinite(v.rate_limit) && v.rate_limit >= 0.0, "server %d: rate_limit=%g must be finite and >= 0 (0 = none)",
                 i, v.rate_limit);
        AF_CHECK(v.burst >= 0, "server %d: burst=%d must be >= 0 (0 reads as 1)", i, v.burst);
    }
    AF_CHECK(isfinite(s.lb_rate_limit) && s.lb_rate_limit >= 0.0, "lb_rate_limit=%g must be finite and >= 0 (0 = none)",
             s.lb_rate_limit);
    AF_CHECK(s.lb_burst >= 0, "lb_burst=%d must be >= 0 (0 reads as 1)", s.lb_burst);
    AF_CHECK(s.lb_rate_limit == 0.0 || s.n_lb_edges > 0, "lb_rate_limit=%g: the scenario has no load balancer", s.lb_rate_limit);
    AF_CHECK(isfinite(s.client_timeout) && s.client_timeout >= 0.0, "client_timeout=%g must be finite and >= 0 (0 = none)",
             s.client_timeout);
    for (int i = 0; i < s.n_endpoints; ++i) {
        const AfEndpoint& p = s.endpoints[i];
        AF_CHECK(p.n_steps >= 0 && p.n_steps <= 255 && p.step_begin >= 0 && p.step_begin + p.n_steps <= s.n_steps,
                 "endpoint %d: step range", i);
        AF_CHECK(p.total_ram >= 0, "endpoint %d: total_ram", i);
    }
    for (int i = 0; i < s.n_steps; ++i)
        AF_CHECK((s.steps[i].kind == AF_STEP_CPU || s.steps[i].kind == AF_STEP_IO) && s.steps[i].duration >= 0.0,
                 "step %d invalid", i);
    for (int i = 0; i < s.n_spike_marks; ++i) {
        AF_CHECK(s.spike_marks[i].edge >= 0 && s.spike_marks[i].edge < s.n_edges, "spike mark %d: edge", i);
        AF_CHECK(i == 0 || s.spike_marks[i].fire_time >= s.spike_marks[i - 1].fire_time, "spike marks unsorted");
    }
    for (int i = 0; i < s.n_outage_marks; ++i) {
        AF_CHECK(s.outage_marks[i].lb_edge < s.n_edges, "outage mark %d: edge", i);
        AF_CHECK(i == 0 || s.outage_marks[i].fire_time >= s.outage_marks[i - 1].fire_time, "outage marks unsorted");
    }
#undef AF_CHECK
    return true;
}

// The per-replica timeline rows of af_timeline_upload get the checks validate() applies to the scenario's tables, row by
// row: spike edges in range, fire times non-decreasing, an outage's lb_edge -1 or one of the scenario's LB edges.
inline bool validate_timeline(const AfScenario& s, const AfTimeline& t, std::string& err) {
    char buf[256];
#define AF_CHECK(cond, ...) do { if (!(cond)) { snprintf(buf, sizeof buf, __VA_ARGS__); err = buf; return false; } } while (0)
    AF_CHECK((s.n_spike_marks == 0 || t.spikes) && (s.n_outage_marks == 0 || t.outages), "timeline: null mark rows");
    for (uint64_t r = 0; r < t.n_rows; ++r) {
        const AfSpikeMark* sp = t.spikes + r * (uint64_t)s.n_spike_marks;
        for (int i = 0; i < s.n_spike_marks; ++i) {
            AF_CHECK(sp[i].edge >= 0 && sp[i].edge < s.n_edges, "timeline row %llu: spike mark %d: edge %d out of range",
                     (unsigned long long)r, i, sp[i].edge);
            AF_CHECK(i == 0 || sp[i].fire_time >= sp[i - 1].fire_time, "timeline row %llu: spike marks unsorted at mark %d",
                     (unsigned long long)r, i);
        }
        const AfOutageMark* om = t.outages + r * (uint64_t)s.n_outage_marks;
        for (int i = 0; i < s.n_outage_marks; ++i) {
            bool lb = om[i].lb_edge == -1;
            for (int k = 0; k < s.n_lb_edges && !lb; ++k) lb = s.lb_edges[k] == om[i].lb_edge;
            AF_CHECK(lb, "timeline row %llu: outage mark %d: lb_edge %d is neither -1 nor an edge of the load balancer",
                     (unsigned long long)r, i, om[i].lb_edge);
            AF_CHECK(i == 0 || om[i].fire_time >= om[i - 1].fire_time, "timeline row %llu: outage marks unsorted at mark %d",
                     (unsigned long long)r, i);
        }
    }
#undef AF_CHECK
    return true;
}

// Does a launch shed requests at an admission limit somewhere (DESIGN.md §3.12)?  A scenario limit, or a sweep column
// over AF_FIELD_SERVER_MAX_IN_SERVICE (even one of zeros): only such launches lay out the kernels' admission words.
inline bool admission_launch(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols) {
    for (int32_t i = 0; i < s.n_servers; ++i) if (s.servers[i].max_in_service > 0) return true;
    for (int32_t c = 0; c < n_cols; ++c) if (cols[c].field == AF_FIELD_SERVER_MAX_IN_SERVICE) return true;
    return false;
}

// af_sweep_upload's check of the AF_FIELD_SERVER_MAX_IN_SERVICE columns: every value an integer in [0, 2^31) (naming
// the row).  Index ranges are checked with the other fields'.
inline bool admission_sweep_fits(const AfSweepColumn* cols, int32_t n_cols, const double* vals, uint64_t n_rows, std::string& err) {
    for (int32_t c = 0; c < n_cols; ++c) {
        if (cols[c].field != AF_FIELD_SERVER_MAX_IN_SERVICE) continue;
        for (uint64_t r = 0; r < n_rows; ++r) {
            const double v = vals[r * (uint64_t)n_cols + (uint64_t)c];
            if (!(v >= 0.0 && v <= 2147483647.0 && v == floor(v))) {      // (NaN fails the first test)
                char b[200];
                snprintf(b, sizeof b, "sweep: row %llu column %d (server_max_in_service, server %d): value %g is not an "
                         "integer in [0, 2^31)", (unsigned long long)r, c, cols[c].index, v);
                err = b;
                return false;
            }
        }
    }
    return true;
}

// Does a launch have a request deadline or a client timeout somewhere (DESIGN.md §3.13)?  A scenario value, or a sweep
// column over AF_FIELD_SERVER_DEADLINE / AF_FIELD_CLIENT_TIMEOUT (even one of zeros): only such launches lay out the
// kernels' deadline words and fill the expired / late outputs.
inline bool deadline_launch(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols) {
    if (s.client_timeout > 0.0) return true;
    for (int32_t i = 0; i < s.n_servers; ++i) if (s.servers[i].deadline > 0.0) return true;
    for (int32_t c = 0; c < n_cols; ++c)
        if (cols[c].field == AF_FIELD_SERVER_DEADLINE || cols[c].field == AF_FIELD_CLIENT_TIMEOUT) return true;
    return false;
}

// af_sweep_upload's check of the AF_FIELD_SERVER_DEADLINE / AF_FIELD_CLIENT_TIMEOUT columns: every value finite and
// >= 0 (naming the row).  Index ranges are checked with the other fields'.
inline bool deadline_sweep_fits(const AfSweepColumn* cols, int32_t n_cols, const double* vals, uint64_t n_rows, std::string& err) {
    for (int32_t c = 0; c < n_cols; ++c) {
        const int32_t f = cols[c].field;
        if (f != AF_FIELD_SERVER_DEADLINE && f != AF_FIELD_CLIENT_TIMEOUT) continue;
        for (uint64_t r = 0; r < n_rows; ++r) {
            const double v = vals[r * (uint64_t)n_cols + (uint64_t)c];
            if (!(v >= 0.0 && isfinite(v))) {                               // (NaN fails the first test)
                char b[200];
                snprintf(b, sizeof b, "sweep: row %llu column %d (%s %d): value %g is not a finite number of seconds >= 0",
                         (unsigned long long)r, c, f == AF_FIELD_SERVER_DEADLINE ? "server_deadline, server" : "client_timeout, index",
                         cols[c].index, v);
                err = b;
                return false;
            }
        }
    }
    return true;
}

// Does a launch have a rate limit somewhere (DESIGN.md §3.14)?  A scenario rate, or a sweep column over
// AF_FIELD_SERVER_RATE / AF_FIELD_SERVER_BURST / AF_FIELD_LB_RATE / AF_FIELD_LB_BURST (even one of zeros): only such
// launches lay out the kernels' token buckets and fill the throttled output.
inline bool ratelimit_launch(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols) {
    if (s.lb_rate_limit > 0.0) return true;
    for (int32_t i = 0; i < s.n_servers; ++i) if (s.servers[i].rate_limit > 0.0) return true;
    for (int32_t c = 0; c < n_cols; ++c)
        if (cols[c].field >= AF_FIELD_SERVER_RATE && cols[c].field <= AF_FIELD_LB_BURST) return true;
    return false;
}

// af_sweep_upload's check of the rate-limit columns: a rate finite and >= 0, a burst an integer in [1, 2^31) (naming the
// row), and no LB column on a scenario without a load balancer.  Index ranges are checked with the other fields'.
inline bool ratelimit_sweep_fits(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols, const double* vals,
                                 uint64_t n_rows, std::string& err) {
    static const char* const names[] = {"server_rate, server", "server_burst, server", "lb_rate, index", "lb_burst, index"};
    char b[200];
    for (int32_t c = 0; c < n_cols; ++c) {
        const int32_t f = cols[c].field;
        if (f < AF_FIELD_SERVER_RATE || f > AF_FIELD_LB_BURST) continue;
        const char* name = names[f - AF_FIELD_SERVER_RATE];
        if ((f == AF_FIELD_LB_RATE || f == AF_FIELD_LB_BURST) && s.n_lb_edges == 0) {
            snprintf(b, sizeof b, "sweep: column %d (%s %d): the scenario has no load balancer", c, name, cols[c].index);
            err = b;
            return false;
        }
        const bool rate = f == AF_FIELD_SERVER_RATE || f == AF_FIELD_LB_RATE;
        for (uint64_t r = 0; r < n_rows; ++r) {
            const double v = vals[r * (uint64_t)n_cols + (uint64_t)c];
            const bool ok = rate ? v >= 0.0 && isfinite(v) : v >= 1.0 && v <= 2147483647.0 && v == floor(v);   // (NaN fails)
            if (!ok) {
                snprintf(b, sizeof b, "sweep: row %llu column %d (%s %d): value %g is not %s", (unsigned long long)r, c, name,
                         cols[c].index, v, rate ? "a finite rate >= 0 (0 = none)" : "an integer burst in [1, 2^31)");
                err = b;
                return false;
            }
        }
    }
    return true;
}

// af_run's rule for a launch with timeline rows: no AF_FIELD_SPIKE_DELTA column (it indexes a mark in the scenario's
// order, which a row may change; a row carries its own amplitudes).
inline bool timeline_sweep_fits(const AfSweepColumn* cols, int32_t n_cols, std::string& err) {
    for (int32_t c = 0; c < n_cols; ++c)
        if (cols[c].field == AF_FIELD_SPIKE_DELTA) {
            err = "af_run: sweep column " + std::to_string(c) + " sweeps a spike amplitude (AF_FIELD_SPIKE_DELTA) while timeline "
                  "rows are uploaded; put the amplitudes in the rows' spike deltas";
            return false;
        }
    return true;
}

// af_sweep_upload's checks of the load-balancer columns (AF_FIELD_LB_COVERED / AF_FIELD_LB_ALGORITHM): a load balancer
// to sweep, values 0 or 1, and in every row at least one covered LB edge (two columns over one position: the later wins,
// as in the kernels).  Index ranges are checked with the other fields'.
inline bool lb_sweep_fits(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols, const double* vals, uint64_t n_rows,
                          std::string& err) {
    char buf[256];
#define AF_CHECK(cond, ...) do { if (!(cond)) { snprintf(buf, sizeof buf, __VA_ARGS__); err = buf; return false; } } while (0)
    bool cover = false;
    for (int32_t c = 0; c < n_cols; ++c) {
        const int32_t f = cols[c].field;
        if (f != AF_FIELD_LB_COVERED && f != AF_FIELD_LB_ALGORITHM) continue;
        AF_CHECK(s.n_lb_edges > 0 && s.lb_algo != AF_LB_NONE, "sweep: column %d sweeps the load balancer of a scenario without one", c);
        cover = cover || f == AF_FIELD_LB_COVERED;
        for (uint64_t r = 0; r < n_rows; ++r) {
            const double v = vals[r * (uint64_t)n_cols + (uint64_t)c];
            AF_CHECK(v == 0.0 || v == 1.0, "sweep: row %llu column %d (%s): value %g is neither 0 nor 1", (unsigned long long)r, c,
                     f == AF_FIELD_LB_COVERED ? "lb_covered" : "lb_algorithm", v);
        }
    }
    if (!cover) return true;
    std::vector<char> on((size_t)s.n_lb_edges);
    for (uint64_t r = 0; r < n_rows; ++r) {
        std::fill(on.begin(), on.end(), (char)1);
        for (int32_t c = 0; c < n_cols; ++c)
            if (cols[c].field == AF_FIELD_LB_COVERED) on[(size_t)cols[c].index] = vals[r * (uint64_t)n_cols + (uint64_t)c] != 0.0;
        bool any = false;
        for (char x : on) any = any || x;
        AF_CHECK(any, "sweep: row %llu covers no edge of the load balancer (AF_FIELD_LB_COVERED is 0 for all %d)",
                 (unsigned long long)r, s.n_lb_edges);
    }
#undef AF_CHECK
    return true;
}

// af_run's rule for a launch with AF_FIELD_LB_COVERED columns: no replica of [begin, end) with a sweep row (sweep row r
// describes replica sweep_first + r) may uncover an LB edge that the outage marks it runs with still name -- its
// timeline row (row r of `tl` describes replica tl_first + r) if it has one, else the scenario's.  Such a mark would
// put the edge back behind the load balancer at its SERVER_UP.  `cols` / `vals` may hold the LB_COVERED columns alone.
inline bool lb_cover_fits(const AfScenario& s, const AfSweepColumn* cols, int32_t n_cols, const double* vals,
                          uint64_t sweep_first, uint64_t sweep_rows, const AfTimeline* tl, uint64_t tl_first,
                          uint64_t begin, uint64_t end, std::string& err) {
    std::vector<int32_t> cover;
    for (int32_t c = 0; c < n_cols; ++c) if (cols[c].field == AF_FIELD_LB_COVERED) cover.push_back(c);
    if (cover.empty() || s.n_lb_edges == 0) return true;
    std::vector<char> on((size_t)s.n_lb_edges);
    const uint64_t lo = begin > sweep_first ? begin : sweep_first;
    const uint64_t hi = end < sweep_first + sweep_rows ? end : sweep_first + sweep_rows;
    for (uint64_t id = lo; id < hi; ++id) {
        const double* row = vals + (id - sweep_first) * (uint64_t)n_cols;
        std::fill(on.begin(), on.end(), (char)1);
        bool cut = false;
        for (int32_t c : cover) { const bool v = row[c] != 0.0; on[(size_t)cols[c].index] = v; cut = cut || !v; }
        if (!cut) continue;
        const bool own = tl != nullptr && id - tl_first < tl->n_rows;
        const AfOutageMark* om = own ? tl->outages + (id - tl_first) * (uint64_t)s.n_outage_marks : s.outage_marks;
        for (int32_t i = 0; i < s.n_outage_marks; ++i) {
            if (om[i].lb_edge < 0) continue;
            for (int32_t k = 0; k < s.n_lb_edges; ++k)
                if (!on[(size_t)k] && s.lb_edges[k] == om[i].lb_edge) {
                    char b[320];
                    snprintf(b, sizeof b, "af_run: replica %llu uncovers load-balancer edge %d (AF_FIELD_LB_COVERED position %d) "
                             "while outage mark %d of its %s names it; give the row a timeline row whose marks of that "
                             "server have lb_edge = -1", (unsigned long long)id, s.lb_edges[k], k, i,
                             own ? "timeline row" : "scenario's timeline");
                    err = b;
                    return false;
                }
        }
    }
    return true;
}

inline int32_t trace_tick_capacity(const AfScenario& s) {
    double n = (double)s.horizon_s / s.sample_period;
    if (n > 50.0e6) n = 50.0e6;
    return (int32_t)n + 2;
}

// Ticks the collector takes before the horizon: n_ticks of every replica that reaches it (the kernels' own repeated
// addition of the sample period; sample_period is not sweepable, so it is the same for every replica of a scenario).
// Counted up to BAND_TICK_LIMIT: a result of BAND_TICK_LIMIT means "at least that many" (band_ticks_fit refuses it).
constexpr uint32_t BAND_TICK_LIMIT = 50000000u;
inline uint32_t band_ticks(const AfScenario& s) {
    const double horizon = (double)s.horizon_s;
    if (horizon / s.sample_period > (double)BAND_TICK_LIMIT + 2.0) return BAND_TICK_LIMIT;
    uint32_t n = 0;
    for (double tick = 0.0 + s.sample_period; tick < horizon && n < BAND_TICK_LIMIT; tick = tick + s.sample_period) ++n;
    return n;
}
// The band rows hold one word per tick and the kernels index them by the replica's tick count without a bounds check:
// every tick a replica can take must have its word, so a scenario that reaches the limit is refused.
inline bool band_ticks_fit(const AfScenario& s, uint32_t& ticks, std::string& why) {
    ticks = band_ticks(s);
    if (ticks < BAND_TICK_LIMIT) return true;
    why = "bands: horizon " + std::to_string(s.horizon_s) + " s at a sample period of " + std::to_string(s.sample_period) +
          " s takes " + std::to_string(BAND_TICK_LIMIT) + " ticks or more; per-tick bands hold fewer";
    return false;
}
// bytes of the difference rows of n_groups groups plus the one of the replicas without a group
inline unsigned __int128 band_row_bytes(uint64_t n_groups, int32_t n_series, uint32_t ticks) {
    return ((unsigned __int128)n_groups + 1) * (unsigned __int128)(1 + 2 * (uint64_t)n_series) * ((unsigned __int128)ticks + 1) * 8u;
}

// Per-window latency bands: ceil(horizon / window) windows of `window_s` seconds, the last one cut at the horizon.
inline uint64_t lat_windows(int32_t horizon_s, int32_t window_s) {
    return ((uint64_t)(horizon_s > 0 ? horizon_s : 0) + (uint64_t)window_s - 1) / (uint64_t)window_s;
}
// bytes of the windows of n_groups groups plus the one of the replicas without a group
inline unsigned __int128 lat_row_bytes(uint64_t n_groups, uint64_t windows) {
    return ((unsigned __int128)n_groups + 1) * (unsigned __int128)windows * afr::LAT_ROW * 8u;
}
// The checks af_bands_configure, af_bands_upload and af_run apply to latency bands of `window_s` seconds over n_groups
// groups: a positive window, and rows the device (mem_total bytes) can hold.
inline bool lat_bands_fit(int32_t window_s, int32_t horizon_s, uint64_t n_groups, uint64_t mem_total, std::string& why) {
    if (window_s < 1) {
        why = "latency bands: window of " + std::to_string(window_s) + " s; the width is a whole number of seconds >= 1";
        return false;
    }
    const uint64_t w = lat_windows(horizon_s, window_s);
    const unsigned __int128 bytes = lat_row_bytes(n_groups, w);
    if (bytes <= (unsigned __int128)mem_total) return true;
    char b[256];
    snprintf(b, sizeof b, "latency bands: %llu groups x %llu windows of %d s need %.3g GB of rows, more than the device's %.3g GB",
             (unsigned long long)n_groups, (unsigned long long)w, window_s, (double)bytes / 1e9, (double)mem_total / 1e9);
    why = b;
    return false;
}

// The largest ram_mb a sweep sets (0: none), and the server it belongs to.
inline uint64_t swept_ram_max(const AfSweepColumn* cols, int32_t n_cols, const double* vals, uint64_t n_rows, int32_t& server) {
    uint64_t b = 0;
    server = -1;
    for (int32_t c = 0; c < n_cols; ++c) {
        if (cols[c].field != AF_FIELD_SERVER_RAM_MB) continue;
        for (uint64_t r = 0; r < n_rows; ++r) {
            const double v = vals[r * (uint64_t)n_cols + (uint64_t)c];
            if (v > (double)b) { b = (uint64_t)v; server = cols[c].index; }
        }
    }
    return b;
}

// The largest value any sampled gauge of a replica can take: a queue length or an edge's connection count is at most
// the requests in flight (the request capacity of either engine), RAM in use at most the largest ram_mb, swept values
// (`swept_ram` of server `swept_server`) included.  `what` names the bound that decides.
inline uint64_t band_gauge_bound(const AfScenario& s, const AfOptions& o, uint64_t swept_ram, int32_t swept_server, std::string& what) {
    int32_t rq = o.request_capacity > 0 ? o.request_capacity : DEFAULT_REQUEST_CAPACITY;
    if (rq > (int32_t)afc::SLOT_MASK) rq = (int32_t)afc::SLOT_MASK;
    uint64_t b = (uint64_t)rq;
    what = "request capacity " + std::to_string(rq);
    for (int i = 0; i < s.n_servers; ++i)
        if ((uint64_t)s.servers[i].ram_mb > b) { b = (uint64_t)s.servers[i].ram_mb; what = "ram_mb " + std::to_string(b) + " of server " + std::to_string(i); }
    if (swept_ram > b) { b = swept_ram; what = "swept ram_mb " + std::to_string(b) + " of server " + std::to_string(swept_server); }
    return b;
}

// sumsq of a group of `group` replicas cannot wrap u64: group * bound^2 < 2^64
inline bool band_sumsq_fits(uint64_t group, uint64_t bound) {
    return (unsigned __int128)group * bound * bound < ((unsigned __int128)1 << 64);
}

// Per-tick distribution bands (DESIGN.md §3.7).  The series af_dist_bands_configure selects, by their af_fetch_sampled
// index: each in range, sampled by the scenario, listed once.
inline bool dist_series_check(const AfScenario& s, const int32_t* series, int32_t n, std::string& why) {
    const int32_t ns3 = 3 * s.n_servers, n_series = ns3 + s.n_edges;
    std::vector<char> seen((size_t)n_series, 0);
    for (int32_t i = 0; i < n; ++i) {
        const int32_t j = series[i];
        const char* bad = nullptr;
        if (j < 0 || j >= n_series) bad = "is not a sampled series of the scenario (index out of range)";
        else if (j < ns3 ? (s.metrics_mask & 7u) != 7u : (s.metrics_mask & AF_METRIC_EDGE_CONN) == 0) bad = "is not sampled by the scenario";
        else if (seen[(size_t)j]) bad = "is listed twice";
        if (bad) {
            char b[200];
            snprintf(b, sizeof b, "distribution bands: series[%d] = %d %s (%d series)", i, j, bad, n_series);
            why = b;
            return false;
        }
        seen[(size_t)j] = 1;
    }
    return true;
}
// The checks af_dist_bands_configure, af_bands_upload and af_run apply to distribution bands of n_dist series over
// n_groups groups: fewer than BAND_TICK_LIMIT ticks, and rows of (n_groups + 1) x n_dist x (ticks + 1) x bins u32 the
// device (mem_total bytes) can hold.  bins = gauge_bin(bound) + 1 for the band_gauge_bound of the scenario, options and
// sweep.  Sets ticks and bins.
inline bool dist_bands_fit(const AfScenario& s, const AfOptions& o, uint64_t swept_ram, int32_t swept_server, uint64_t n_groups,
                           uint64_t n_dist, uint64_t mem_total, uint32_t& ticks, uint32_t& bins, std::string& why) {
    std::string what;
    const uint64_t bound = band_gauge_bound(s, o, swept_ram, swept_server, what);
    bins = afr::gauge_bin((uint32_t)(bound < 0xFFFFFFFFull ? bound : 0xFFFFFFFFull)) + 1u;
    if (!band_ticks_fit(s, ticks, why)) { why = "distribution " + why; return false; }
    const unsigned __int128 bytes = ((unsigned __int128)n_groups + 1) * n_dist * ((unsigned __int128)ticks + 1) * bins * 4u;
    if (bytes <= (unsigned __int128)mem_total) return true;
    char b[320];
    snprintf(b, sizeof b, "distribution bands: %llu groups x %llu series x %u ticks x %u bins (bound on a gauge %llu: %s) need "
             "%.3g GB of rows, more than the device's %.3g GB", (unsigned long long)n_groups, (unsigned long long)n_dist,
             ticks, bins, (unsigned long long)bound, what.c_str(), (double)bytes / 1e9, (double)mem_total / 1e9);
    why = b;
    return false;
}

// Occupancy integrals (DESIGN.md §3.8): 5 columns per server (afl::OC_*), one per edge.
inline int32_t occ_cols(const AfScenario& s) { return 5 * s.n_servers + s.n_edges; }
// The most fraction bits f (at most 32) for which a column bounded by `bound` x `horizon_s` seconds stays below 2^64:
// floor(log2((2^64 - 1) / (bound x horizon))); -1 when not even f = 0 fits.
inline int32_t occ_frac_bits(uint64_t bound, int32_t horizon_s) {
    const unsigned __int128 bh = (unsigned __int128)(bound ? bound : 1) * (uint64_t)(horizon_s > 0 ? horizon_s : 1);
    if (bh > ~0ull) return -1;
    const uint64_t q = ~0ull / (uint64_t)bh;
    int32_t f = 63 - __builtin_clzll(q);
    return f < 32 ? f : 32;
}
// The check af_occupancy_configure and af_run apply: 8 <= f <= 32, and bound x horizon x 2^f <= 2^64 - 1 for the
// band_gauge_bound of the scenario, options and sweep (a count of requests is at most the request capacity, MB in use
// at most the largest ram_mb).
inline bool occ_fits(const AfScenario& s, const AfOptions& o, uint64_t swept_ram, int32_t swept_server, int32_t frac_bits,
                     std::string& why) {
    std::string what;
    const uint64_t bound = band_gauge_bound(s, o, swept_ram, swept_server, what);
    char b[400];
    if (frac_bits < 8 || frac_bits > 32) {
        snprintf(b, sizeof b, "occupancy: %d fraction bits; 8 to 32 are supported", frac_bits);
        why = b;
        return false;
    }
    if (((unsigned __int128)bound * (uint64_t)s.horizon_s << frac_bits) <= (unsigned __int128)~0ull) return true;
    snprintf(b, sizeof b, "occupancy: a column of up to B = %llu (%s) x H = %d s in fixed point with f = %d fraction bits "
             "could reach 2^64; this bound and horizon allow f <= %d", (unsigned long long)bound, what.c_str(), s.horizon_s,
             frac_bits, occ_frac_bits(bound, s.horizon_s));
    why = b;
    return false;
}

inline void make_layout(const AfScenario& s, const AfOptions& o, int32_t n_sweep_cols, afc::Layout& L) {
    L.n_edges = s.n_edges; L.n_servers = s.n_servers; L.n_endpoints = s.n_endpoints; L.n_steps = s.n_steps;
    L.n_lb_edges = s.n_lb_edges; L.lb_algo = s.lb_algo; L.gen_edge = s.gen_edge; L.client_edge = s.client_edge;
    L.n_spike = s.n_spike_marks; L.n_outage = s.n_outage_marks;
    L.users_dist = s.users_dist; L.window_s = s.window_s; L.horizon_s = s.horizon_s; L.metrics_mask = s.metrics_mask;
    L.users_mean = s.users_mean; L.users_sigma = s.users_sigma; L.rate_per_user = s.rate_per_user;
    L.sample_period = s.sample_period;
    int32_t ev = o.event_capacity > 0 ? o.event_capacity : DEFAULT_EVENT_CAPACITY;
    int32_t rq = o.request_capacity > 0 ? o.request_capacity : DEFAULT_REQUEST_CAPACITY;
    if (rq > (int32_t)afc::SLOT_MASK) rq = (int32_t)afc::SLOT_MASK;
    L.ev_total = ev; L.ev_smem = ev < DEFAULT_EV_SMEM ? ev : DEFAULT_EV_SMEM;
    L.rq_total = rq; L.rq_smem = rq < DEFAULT_RQ_SMEM ? rq : DEFAULT_RQ_SMEM;
    L.n_series = 3 * s.n_servers + s.n_edges;
    L.n_sweep_cols = n_sweep_cols;
    L.collect_hist = o.collect_histogram; L.collect_thr = o.collect_throughput;
    L.trace_replicas = o.trace_replicas; L.trace_clock_cap = o.trace_clock_capacity;
    L.trace_tick_cap = trace_tick_capacity(s);
    afc::layout_finalize(L);
}

// lower edge (seconds) of histogram bin `idx`
inline double hist_bin_edge(int32_t idx) {
    uint64_t bits = ((uint64_t)(idx + ((1023 + AF_HIST_MIN_EXP) << AF_HIST_SUB_BITS))) << (52 - AF_HIST_SUB_BITS);
    double x; memcpy(&x, &bits, 8); return x;
}

// value of the order statistic `rank` (0-based) read off the histogram.  The end bins also hold the latencies the
// histogram clamps into them: bin 0 spans [min(edge(0), lat_min), edge(1)), the last bin [edge(B-1), max(edge(B),
// lat_max)], lat_min / lat_max being the replica's exact extremes
inline double hist_order_stat(const uint32_t* hist, uint64_t rank, double lat_min, double lat_max) {
    uint64_t cum = 0;
    for (int32_t b = 0; b < AF_HIST_BINS; ++b) {
        uint64_t c = hist[b];
        if (c && rank < cum + c) {
            double lo = hist_bin_edge(b), hi = hist_bin_edge(b + 1);
            if (b == 0 && lat_min < lo) lo = lat_min;
            if (b == AF_HIST_BINS - 1 && lat_max > hi) hi = lat_max;
            double frac = ((double)(rank - cum) + 0.5) / (double)c;
            return lo + frac * (hi - lo);
        }
        cum += c;
    }
    return NAN;
}

// numpy.percentile(..., method="linear") evaluated on the histogram of a replica whose latencies span [lat_min, lat_max].
// Without the extremes (a histogram summed over replicas has none) every bin keeps its own edges.
inline double hist_percentile(const uint32_t* hist, uint64_t n, double q, double lat_min = INFINITY, double lat_max = 0.0) {
    if (n == 0) return NAN;
    double pos = q / 100.0 * (double)(n - 1);
    uint64_t lo = (uint64_t)floor(pos);
    double frac = pos - (double)lo;
    double a = hist_order_stat(hist, lo, lat_min, lat_max);
    if (frac == 0.0 || lo + 1 >= n) return a;
    double b = hist_order_stat(hist, lo + 1, lat_min, lat_max);
    return a + frac * (b - a);
}

}  // namespace afh
