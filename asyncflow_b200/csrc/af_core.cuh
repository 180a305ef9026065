// af_core.cuh -- the per-replica next-event engine (one replica per warp).
//
// This is the H100-native replacement of the reference's hot loop: SimPy's
// Environment.step() (external simpy 4.1.1, called from reference
// src/asyncflow/runtime/simulation_runner.py:369) popping (time, prio, eid)
// tuples and resuming the AsyncFlow actor generators.  Here every actor is a
// branch of one state machine and only events that carry simulated delay are
// queued in the pending-event pool (6-7 per request instead of SimPy's 25-30,
// SURVEY.md 8a); SimPy's zero-delay events (Store put/get, Container put/get,
// process resume) are continuation items of a small FIFO that is bypassed
// whenever nothing else shares the instant (see the ordering rule below):
//
//   code here           reference being replaced
//   ------------------  ---------------------------------------------------------
//   gen_next_gap        samplers/poisson_poisson.py:52-82, gaussian_poisson.py:64-94
//   on_arrival          runtime/actors/rqs_generator.py:97-119
//   edge_send           runtime/actors/edge.py:73-107 (dropout, latency, spike)
//   on_deliver          edge.py:110-116 (timeout fired: connection closes, Store.put)
//   node_got            client.py:43-71, load_balancer.py:60-72 + routing/lb_algorithms.py:10-36,
//                       server.py:303-313 (the node's consumer process resumes)
//   server_got          runtime/actors/server.py:88-149 (endpoint pick, RAM first)
//   run_steps           server.py:197-276 (lazy CPU lock, IO queue, release, forward)
//   cpu_walk, ram_walk  simpy Container._trigger_get (FIFO, head-of-line blocking)
//   on_spike/on_outage  runtime/events/injection.py:167-226
//   take_samples        metrics/collector.py:50-66
//   complete            client.py:62-69 + metrics/analyzer.py:83-125
//
// Ordering rule (DESIGN.md "tie rule").  SimPy orders by (time, priority, eid).  Timed
// events live in the pending-event pool and pop by (time, seq), seq being the per-replica
// scheduling counter (SimPy's eid).  Step durations are deterministic, so different
// requests DO reach the same instant (e.g. 3 ms CPU + 8 ms IO + 1 ms CPU == 12 ms IO), and
// what happens at such an instant depends on SimPy's zero-delay events: a Store put, a
// Container get/put or a process resume is itself an event that is queued BEHIND everything
// already scheduled for that instant.  The engine therefore keeps a small FIFO of zero-delay
// continuation items (the "now-queue": I_PUT, I_GOT, I_CLIENT_LOOP, I_RAM_OK, I_CPU_OK,
// I_CPU_PUT, I_RAM_PUT -- one per SimPy event that carries an observable effect), each with
// its own seq, and always runs the smallest seq among {now-queue front, pool events of the
// current instant}.  URGENT events (process Initialize) run at the end of the item that
// created them, as in SimPy.  Collector ticks are not queued: state is piecewise constant
// between timed events, so the samples that fall before an event are emitted lazily just
// before it (they carry a seq too).
//
// Execution model: ALL 32 lanes of the warp run this code redundantly on the
// same replica (warp-uniform control flow, identical values in every lane).
// Lanes differ only inside the few helpers that say so: the pending-event pool
// is an unsorted, lane-strided array and pop-min is a warp arg-min
// (redux.sync on the time words, then seq); per-entity loops (sampling, final
// write-back, parameter load) are lane-strided.
//
// Code-size rule (round-1 profile): with everything inlined
// the kernel was 14 k instructions and 67 % of warp stalls were instruction-cache
// misses -- every warp sits in a different handler.  So the replica's scalar
// state lives in a per-warp struct in SHARED memory (`State`), the scenario
// sizes / device pointers live in __constant__ memory, and every helper with
// more than one call site is a real function (__noinline__) taking only
// `State&`: one copy of each body, few live registers, more resident warps.
//
// The same source compiles for the host with a warp of ONE lane
// (tests/host_twin -- a debugging twin used by the CPU-only tests; it is NOT
// reachable from the product API).
//
// Round 2: this engine is the fall-back of af_run (topologies too wide for a useful occupancy of the thread-per-replica
// engine, replicas that overflow its tiers).  Its round-1 build variants (memoised variates, sorted front ring, pinned
// request slots) were never promoted -- the thread-per-replica engine made the question moot -- and are gone.
#pragma once
#include "af_rng.cuh"
#include "../../include/asyncflow_b200.h"

#if defined(__CUDA_ARCH__)
#define AF_DEVICE_CODE 1
#else
#define AF_DEVICE_CODE 0
#endif

#if defined(__CUDACC__)
#define AF_FN __host__ __device__ __noinline__       /* one shared body            */
#define AF_IN __host__ __device__ __forceinline__    /* small, or single call site */
#else
#define AF_FN static
#define AF_IN static inline
#endif

// Tell the compiler that a pointer is into shared memory so that the helpers (which only
// see a generic `State&`) emit LDS/STS instead of generic LD/ST.
#if AF_DEVICE_CODE
#define AF_SHARED(p) __builtin_assume(__isShared(p))
#else
#define AF_SHARED(p) ((void)0)
#endif

// Host-twin debugging aid: compile the twin with -DAF_TRACE_HOST to log every handled event.
#if defined(AF_TRACE_HOST) && !AF_DEVICE_CODE
#include <stdio.h>
#define AF_TRACE(...) fprintf(stderr, __VA_ARGS__)
#else
#define AF_TRACE(...) ((void)0)
#endif

#define AF_LIKELY(x) __builtin_expect(!!(x), 1)
#define AF_UNLIKELY(x) __builtin_expect(!!(x), 0)

namespace afc {

// flags that end a replica early (its partial results are written back with the flag set)
constexpr uint32_t STOP_FLAGS = AF_FLAG_EVENT_OVERFLOW | AF_FLAG_REQUEST_OVERFLOW | AF_FLAG_NOWQ_OVERFLOW | AF_FLAG_LB_EMPTY;
constexpr uint32_t NIL = 0xFFFFFFFFu;
constexpr uint64_t INF_BITS = 0x7FF0000000000000ull;

// ---- event payload: kind[29:32) | aux[20:29) | slot[0:20) -------------------
enum : uint32_t { K_ARRIVAL = 0, K_DELIVER = 1, K_STEP_END = 2, K_SPIKE = 3, K_OUTAGE = 4 };
constexpr uint32_t SLOT_BITS = 20, AUX_BITS = 9;
constexpr uint32_t SLOT_MASK = (1u << SLOT_BITS) - 1, AUX_MASK = (1u << AUX_BITS) - 1;
AF_IN uint32_t mk_payload(uint32_t kind, uint32_t aux, uint32_t slot) {
    return (kind << 29) | (aux << SLOT_BITS) | slot;
}

// ---- request record pack: hops[0:8) step[8:16) ep[16:28) core[28] io[29] wait[30] expired[31] ----
constexpr uint32_t PK_CORE = 1u << 28, PK_IO = 1u << 29;
constexpr uint32_t PK_EXPIRED = 1u << 31;   // past its server's deadline: the handler's tail runs, no forward (§3.13)
constexpr double INF_DEADLINE = __builtin_huge_val();   // ServerS.deadline / State.timeout of "none"
AF_IN uint32_t pk_hops(uint32_t p) { return p & 0xFFu; }
AF_IN uint32_t pk_step(uint32_t p) { return (p >> 8) & 0xFFu; }
AF_IN uint32_t pk_ep(uint32_t p) { return (p >> 16) & 0xFFFu; }

struct ReqRec { double t0; uint32_t rid; uint32_t pack; };          // 16 B


// ---- per-warp private tables (shared memory on the device) -------------------
struct EdgeS {            // 48 B
    double mean, sigma, dropout, spike;
    uint32_t meta;        // dist[0:3) | target_kind[3:5) | target_index[5:)
    uint32_t conn, sent, dropped;
};
struct ServerS {          // 64 B
    int32_t cpu_free, ram_free, ready_q, io_q, ram_in_use;
    uint32_t ramq_head, ramq_tail, cpuq_head, cpuq_tail;
    uint32_t out_edge, ep_begin, n_ep;
    uint32_t ramq_head_need;   // total_ram of the request at the head of the RAM queue (valid when ramq_head != NIL)
    // admission limit (DESIGN.md §3.12): admissions left before the server sheds (0xFFFFFFFF: no limit; one per request
    // in service), requests shed
    uint32_t adm_left, rejected;
    // requests dropped past the server's deadline (DESIGN.md §3.13; the deadline itself: tbl_deadline)
    uint32_t expired;
};
struct EndpointS { uint32_t step_begin, n_steps, total_ram, pad; }; // 16 B
struct StepS { double dur; uint32_t kind, pad; };                   // 16 B
struct SpikeS { double fire, delta; uint32_t edge, pad; };           // 24 B
struct OutageS { double fire; int32_t lb_edge, down; };              // 16 B
struct InboxS { uint32_t head, tail, pending, pad; };                // 16 B: a node's Store + its consumer's pending get()
// a server's rate limit (DESIGN.md §3.14; tbl_rate): its GCRA bucket's theoretical arrival time, tau and tolerance L
// (tau = 0: no limit), and the requests it throttled
struct RateS { double tat, tau, lim; uint32_t throttled, pad; };     // 32 B

// The replica's scalar state: one per warp, at the start of the warp's workspace.
struct State {
    // this warp's HBM spill regions (the shared-memory tables sit at fixed offsets
    // behind this struct: see tbl_*() below -- 32-bit shared addresses, no pointer loads)
    double* sp_ev_time; uint64_t* sp_ev_key; ReqRec* sp_rq_rec; uint32_t* sp_rq_next;
    // identity
    uint64_t replica, local;                // replica: the stream its draws are keyed by; local: its output slot
    // clock + pending-event pool
    double now, horizon;
    uint32_t seq;
    int32_t ev_hw, ev_live, ev_last_free, ev_hole;
    uint32_t peak_ev;
    // zero-delay continuation FIFO (ring of NQ_CAP items) + "the pool may hold an event of this instant"
    uint32_t nq_head, nq_tail, busy;   // busy = 2 * (items in the now-queue) + (pool may hold an event of this instant)
    // request table
    uint32_t rq_free, rq_hw, rq_live, peak_rq;
    // generator (two clocks: the sampler's virtual one and the simulation's)
    double g_vnow, g_window_end, g_lam;
    uint32_t g_pos, generated, g_done, need_arrival, arm_seq;
    // parameters that may be swept
    double users_mean, users_sigma, rate_per_user;
    // load balancer / timelines
    int32_t lb_n, spike_cur, outage_cur;
    // sampler
    uint32_t tick_seq, n_ticks;
    double tick_time;
    // results
    uint32_t completed, flags, traced;
    int32_t lb_algo;                        // the replica's AF_LB_* (its sweep row's, else the scenario's)
    uint64_t n_events;
    double lat_sum, lat_sumsq, lat_min, lat_max;
    // per-tick bands: the replica's group's difference rows (nullptr: bands off), the first tick it contributes, the
    // words per difference row, the byte offset of the table of each series' last emitted value (u32, behind the tables)
    uint64_t* band;
    uint32_t band_from, band_stride, band_prev_off, band_pad;
    // per-window latency bands: the replica's group's windows (nullptr: off), the completions the thread-per-replica
    // pass already added (a re-run adds from there on), the window width in seconds
    uint64_t* lat;
    uint32_t lat_from, lat_window;
    // per-tick distribution bands: the replica's group's rows (nullptr: off; the first tick is band_from, the last
    // emitted values are the band_prev table), each series' slot (-1: not selected), bins per tick row, words per series
    uint32_t* dist; const int32_t* dist_slot;
    uint64_t dist_series_words;
    uint32_t dist_bins, dist_pad;
    // occupancy integrals: the replica's output row (nullptr: off; afl::occ_add, DESIGN.md §3.8), 2^f
    uint64_t* occ; double occ_scale;
    // client timeout (DESIGN.md §3.13; +inf: none) and the completions later than it
    double timeout;
    uint32_t late, late_pad;
    // the load balancer's rate limit and the requests it throttled (DESIGN.md §3.14)
    RateS lb_rl;
};

// Everything the kernel needs to know about sizes; built on the host.
struct Layout {
    int32_t n_edges, n_servers, n_endpoints, n_steps, n_lb_edges, lb_algo;
    int32_t gen_edge, client_edge, n_spike, n_outage;
    int32_t users_dist, window_s, horizon_s;
    uint32_t metrics_mask;
    double users_mean, users_sigma, rate_per_user, sample_period;
    int32_t ev_smem, ev_total;     // pending-event pool: slots in smem / in total
    int32_t rq_smem, rq_total;     // request table: slots in smem / in total
    int32_t n_series;              // 3*n_servers + n_edges
    int32_t n_sweep_cols;
    int32_t collect_hist, collect_thr;
    int32_t trace_replicas, trace_clock_cap, trace_tick_cap;
    // byte offsets inside the per-warp workspace
    int32_t off_ev_time, off_ev_key, off_rq_rec, off_rq_next, off_edge, off_server,
            off_endpoint, off_step, off_lb, off_spike, off_outage, off_samp_sum, off_samp_max, off_nq, off_inbox;
    int32_t warp_bytes;
};

// Per-tick bands of a launch (af_sim_kernel's parameter; stride == 0: off).  As afl::Cfg's band_* (af_lane.cuh):
// group g's difference rows start at rows + g * group_words; from[local] = the tick from which a re-run of a flagged
// replica contributes (the thread-per-replica pass contributed the ticks before it); prev_off = byte offset of the
// table of each series' last emitted value in the warp's workspace (4 * n_series bytes behind Layout.warp_bytes).
// Per-window latency bands (lat_window == 0: off), over the same groups: group g's windows start at
// lat_rows + g * lat_windows * afr::LAT_ROW; lat_from[local] = the completions the thread-per-replica pass added.
struct BandArgs {
    uint64_t* rows; const uint32_t* group; const uint32_t* from;
    uint64_t first, n, group_words;
    uint32_t groups, stride; int32_t prev_off, pad;
    uint64_t* lat_rows; const uint32_t* lat_from;
    uint32_t lat_window, lat_windows;
    // per-tick distribution bands (dist_rows == nullptr: off), over the same groups and with the same from[] as the
    // per-tick bands: afl::Cfg's dist_* (af_lane.cuh); they need the prev_off table too
    uint32_t* dist_rows; const int32_t* dist_slot;
    uint64_t dist_group_words, dist_series_words;
    uint32_t dist_bins, dist_pad;
    // occupancy integrals (occ == nullptr: off): [n_replicas][5 n_servers + n_edges] u64, occ_scale = 2^f
    uint64_t* occ; double occ_scale;
    // requests each server shed at its admission limit (nullptr: the launch has no limit; DESIGN.md §3.12):
    // [n_replicas][n_servers] u32, written with the replica's other outputs
    uint32_t* server_rejected;
    // requests each server dropped past its deadline, [n_replicas][n_servers] u32, and completions later than the client
    // timeout, [n_replicas] u32 (nullptr: the launch has neither; DESIGN.md §3.13)
    uint32_t* server_expired; uint32_t* late;
    double client_timeout;         // the scenario's (0: none)
    // requests each site throttled at its rate limit, [n_replicas][n_servers + 1] u32, column n_servers the load
    // balancer (nullptr: the launch has no rate limit; DESIGN.md §3.14), and the scenario's LB rate (0: none) and burst
    uint32_t* throttled;
    double lb_rate;
    int32_t lb_burst, rl_pad;
};

// Per-replica timelines of a launch (af_sim_kernel's parameter; rows == 0: none): replica first + r, r < rows, copies its
// marks from spikes + r * n_spike and outages + r * n_outage instead of Globals' tables (DESIGN.md §3.9).
struct TimelineArgs {
    const AfSpikeMark* spikes; const AfOutageMark* outages;
    uint64_t first, rows;
};

// Random streams of a launch (af_sim_kernel's parameter; rows == 0: none): replica first + i, i < rows, draws as
// stream_of[i], every other replica as its own id (DESIGN.md §3.10).
struct StreamArgs {
    const uint64_t* stream_of;
    uint64_t first, rows;
};

constexpr int32_t NQ_CAP = 128;   // now-queue capacity (power of two)

AF_IN int32_t align_up(int32_t x, int32_t a) { return (x + a - 1) / a * a; }

inline void layout_finalize(Layout& L) {
    int32_t o = align_up((int32_t)sizeof(State), 16);
    L.off_ev_time = o;  o += 8 * L.ev_smem;
    L.off_ev_key = o;   o += 8 * L.ev_smem;
    L.off_nq = o;       o += 8 * NQ_CAP;
    L.off_inbox = o;    o += 16 * (L.n_servers + 2);
    L.off_rq_rec = o;   o += 16 * L.rq_smem;
    L.off_edge = o;     o += 48 * L.n_edges;
    L.off_server = o;   o += 64 * L.n_servers;
    L.off_endpoint = o; o += 16 * L.n_endpoints;
    L.off_step = o;     o += 16 * L.n_steps;
    L.off_spike = o;    o += 24 * L.n_spike;
    L.off_outage = o;   o += 16 * L.n_outage;
    L.off_samp_sum = o; o += 8 * L.n_series;
    L.off_rq_next = o;  o += 4 * L.rq_smem;
    L.off_samp_max = o; o += 4 * L.n_series;
    L.off_lb = o;       o += 4 * L.n_lb_edges;
    o = align_up(o, 8) + 8 * L.n_servers;  // each server's deadline (tbl_deadline: no Layout field, so that no
                                            // __constant__ offset of the lane kernel's moves)
    o += 32 * L.n_servers;                  // each server's rate limit (tbl_rate; likewise)
    L.warp_bytes = align_up(o, 16);
}

// Device-global pointers (read-only scenario, sweep rows, spill tiers, outputs).
struct Globals {
    const AfEdge* edges; const AfServer* servers; const AfEndpoint* endpoints;
    const AfStep* steps; const int32_t* lb_edges; const AfSpikeMark* spikes;
    const AfOutageMark* outages;
    const AfSweepColumn* sweep_cols; const double* sweep_vals; uint64_t sweep_first, sweep_rows;
    // spill tiers, one region per resident warp slot
    double* spill_ev_time; uint64_t* spill_ev_key; ReqRec* spill_rq_rec; uint32_t* spill_rq_next;
    // outputs, indexed by local replica
    AfReplicaStats* stats; uint32_t* edge_sent; uint32_t* edge_dropped;
    uint32_t* hist; uint32_t* thr; uint64_t* samp_sum; uint32_t* samp_max;
    double* trace_clocks; uint32_t* trace_series; uint32_t* trace_counts;
    unsigned long long* work_counter;
    const uint32_t* order;           // first pass: the k-th replica a warp pulls is local index order[k] (af_run)
    // second pass (af_engine.cu): the replicas the thread-per-replica pass flagged; NULL = every replica of the launch
    const uint32_t* redo_list; const uint32_t* redo_count;
    uint64_t seed, replica_begin, n_replicas;
};

// Launch-wide constants: __constant__ memory on the device (every helper reads them
// through the constant cache), plain globals in the host twin.
#if defined(__CUDACC__)
__constant__ Layout c_L;
__constant__ Globals c_G;
#endif
#if AF_DEVICE_CODE
#define AF_L c_L
#define AF_G c_G
#else
static Layout h_L;
static Globals h_G;
#define AF_L h_L
#define AF_G h_G
#endif


// Shared-memory tables of the warp: fixed byte offsets (Layout) behind its State.
#define AF_TBL(name, type, off)                                                    \
    AF_IN type* name(State& W) { return reinterpret_cast<type*>(reinterpret_cast<unsigned char*>(&W) + AF_L.off); } \
    AF_IN const type* name(const State& W) { return reinterpret_cast<const type*>(reinterpret_cast<const unsigned char*>(&W) + AF_L.off); }
AF_TBL(tbl_ev_time, double, off_ev_time)
AF_TBL(tbl_ev_key, uint64_t, off_ev_key)
AF_TBL(tbl_rq_rec, ReqRec, off_rq_rec)
AF_TBL(tbl_rq_next, uint32_t, off_rq_next)
AF_TBL(tbl_edge, EdgeS, off_edge)
AF_TBL(tbl_server, ServerS, off_server)
AF_TBL(tbl_endpoint, EndpointS, off_endpoint)
AF_TBL(tbl_step, StepS, off_step)
AF_TBL(tbl_lb, uint32_t, off_lb)
AF_TBL(tbl_spike, SpikeS, off_spike)
AF_TBL(tbl_outage, OutageS, off_outage)
AF_TBL(tbl_samp_sum, uint64_t, off_samp_sum)
AF_TBL(tbl_samp_max, uint32_t, off_samp_max)
// each server's deadline in seconds (+inf: none; DESIGN.md §3.13), f64, right after the LB order
AF_IN double* tbl_deadline(State& W) {
    return reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(&W) + align_up(AF_L.off_lb + 4 * AF_L.n_lb_edges, 8));
}
// each server's rate limit (RateS; DESIGN.md §3.14), right after the deadlines
AF_IN RateS* tbl_rate(State& W) {
    return reinterpret_cast<RateS*>(reinterpret_cast<unsigned char*>(&W) + align_up(AF_L.off_lb + 4 * AF_L.n_lb_edges, 8)
                                    + 8 * AF_L.n_servers);
}
AF_TBL(tbl_nq, uint64_t, off_nq)
AF_TBL(tbl_inbox, InboxS, off_inbox)
AF_IN uint32_t* tbl_band_prev(State& W) { return reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(&W) + W.band_prev_off); }

// ---- warp primitives (a warp of ONE lane on the host) ------------------------
#if AF_DEVICE_CODE
constexpr int WARP = 32;
#define AF_FULL 0xFFFFFFFFu
__device__ __forceinline__ int lane_id() { return (int)(threadIdx.x & 31u); }
__device__ __forceinline__ uint32_t w_min(uint32_t v) { return __reduce_min_sync(AF_FULL, v); }
__device__ __forceinline__ uint32_t w_ballot(bool p) { return __ballot_sync(AF_FULL, p); }
__device__ __forceinline__ uint32_t w_shfl(uint32_t v, int src) { return __shfl_sync(AF_FULL, v, src); }
__device__ __forceinline__ void w_sync() { __syncwarp(); }
__device__ __forceinline__ void red_add_u32(uint32_t* p, uint32_t v) { atomicAdd(p, v); }
__device__ __forceinline__ void red_add_u64(uint64_t* p, uint64_t v) { atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); }
#else
constexpr int WARP = 1;
static inline int lane_id() { return 0; }
static inline uint32_t w_min(uint32_t v) { return v; }
static inline uint32_t w_ballot(bool p) { return p ? 1u : 0u; }
static inline uint32_t w_shfl(uint32_t v, int) { return v; }
static inline void w_sync() {}
static inline void red_add_u32(uint32_t* p, uint32_t v) { *p += v; }
static inline void red_add_u64(uint64_t* p, uint64_t v) { *p += v; }
#endif

// occupancy integrals (afl::occ_add): a count of requests in some state changes by delta at W.now -- lane 0 adds
// delta * fixed(H - now) to the column of the replica's row (every lane runs this code)
enum : int32_t { OC_RAM_WAIT = 0, OC_CPU_WAIT, OC_CPU, OC_IO, OC_RAM_MB, OC_WORDS };
AF_IN void occ_add(const State& W, int32_t col, int32_t delta) {
    if (W.occ != nullptr && lane_id() == 0)
        red_add_u64(W.occ + col, (uint64_t)(int64_t)delta * afr::occ_fixed(W.horizon - W.now, W.occ_scale));
}
AF_IN void occ_srv(const State& W, uint32_t sidx, int32_t state, int32_t delta) { occ_add(W, OC_WORDS * (int32_t)sidx + state, delta); }

// ---------------------------------------------------------------------------------
// storage tiers: low slot numbers live in shared memory, the rest in the warp's HBM
// spill region (overloaded replicas queue 10^4-10^5 requests, SURVEY.md 8d C2)
// ---------------------------------------------------------------------------------
#define AF_IN_SMEM(idx, cap) AF_LIKELY((int32_t)(idx) < (cap))
AF_IN ReqRec rq_load(const State& W, uint32_t s) {
    return AF_IN_SMEM(s, AF_L.rq_smem) ? tbl_rq_rec(W)[s] : W.sp_rq_rec[s - AF_L.rq_smem];
}
AF_IN void rq_store(State& W, uint32_t s, const ReqRec& r) {
    if (AF_IN_SMEM(s, AF_L.rq_smem)) tbl_rq_rec(W)[s] = r; else W.sp_rq_rec[s - AF_L.rq_smem] = r;
}
AF_IN void rq_set_pack(State& W, uint32_t s, uint32_t pack) {
    if (AF_IN_SMEM(s, AF_L.rq_smem)) tbl_rq_rec(W)[s].pack = pack; else W.sp_rq_rec[s - AF_L.rq_smem].pack = pack;
}
AF_IN uint32_t nx_load(const State& W, uint32_t s) {
    return AF_IN_SMEM(s, AF_L.rq_smem) ? tbl_rq_next(W)[s] : W.sp_rq_next[s - AF_L.rq_smem];
}
AF_IN void nx_store(State& W, uint32_t s, uint32_t v) {
    if (AF_IN_SMEM(s, AF_L.rq_smem)) tbl_rq_next(W)[s] = v; else W.sp_rq_next[s - AF_L.rq_smem] = v;
}
AF_IN uint64_t evt_load(const State& W, int32_t k) {
    return afr::d2u(AF_IN_SMEM(k, AF_L.ev_smem) ? tbl_ev_time(W)[k] : W.sp_ev_time[k - AF_L.ev_smem]);
}
AF_IN uint64_t evk_load(const State& W, int32_t k) {
    return AF_IN_SMEM(k, AF_L.ev_smem) ? tbl_ev_key(W)[k] : W.sp_ev_key[k - AF_L.ev_smem];
}

// ---- request slots (free list threaded through rq_next) ------------------------
AF_IN uint32_t rq_alloc(State& W) {
    uint32_t s;
    if (W.rq_free != NIL) { s = W.rq_free; W.rq_free = nx_load(W, s); }
    else if ((int32_t)W.rq_hw < AF_L.rq_total) { s = W.rq_hw++; }
    else { W.flags |= AF_FLAG_REQUEST_OVERFLOW; return NIL; }
    uint32_t live = ++W.rq_live;
    if (live > W.peak_rq) W.peak_rq = live;
    return s;
}
AF_IN void rq_release(State& W, uint32_t s) { nx_store(W, s, W.rq_free); W.rq_free = s; --W.rq_live; }


// intrusive FIFOs (RAM waiters, CPU waiters) through the same `next` links
AF_FN void fifo_push(State& W, uint32_t& head, uint32_t& tail, uint32_t s) {
    AF_SHARED(&W); AF_SHARED(&head); AF_SHARED(&tail);
    nx_store(W, s, NIL);
    if (tail == NIL) head = s; else nx_store(W, tail, s);
    tail = s;
}
AF_FN uint32_t fifo_pop(State& W, uint32_t& head, uint32_t& tail) {
    AF_SHARED(&W); AF_SHARED(&head); AF_SHARED(&tail);
    uint32_t s = head;
    head = nx_load(W, s);
    if (head == NIL) tail = NIL;
    return s;
}

// ---------------------------------------------------------------------------------
// pending-event pool: an unsorted, lane-strided array; slot k belongs to lane k % 32.
// push is O(1) -- it reuses the slot freed by the last pop, else a hole the last pop's
// scan noticed, else appends; pop is a warp arg-min over (time, seq).  Every lane
// executes push (same slot, same values); only the owner lane reads the slot back.
// ---------------------------------------------------------------------------------
// Pool hygiene (both out of line, both rare).  push takes the slot of the last pop, then a hole the
// last scan noticed, then APPENDS; under bursts that lets the high-water mark run ahead of the live
// count and -- because fresh events keep landing at the top -- it never comes back: overloaded
// replicas were scanning ~750 slots for ~20 live events (round-1 finding).  So: once the slack
// exceeds POOL_SLACK, push fills the lowest hole instead, and popping the top slot pulls the mark
// down to the highest occupied slot.
constexpr int32_t POOL_SLACK = 8;
AF_FN int32_t pool_top(State& W) {
    AF_SHARED(&W);
    const int lane = lane_id();
    const int32_t hw = W.ev_hw;
    int32_t mine = -1;
#pragma unroll 1
    for (int32_t k = lane; k < hw; k += WARP)
        if (evt_load(W, k) != INF_BITS) mine = k;
#if AF_DEVICE_CODE
    mine = (int32_t)__reduce_max_sync(AF_FULL, (uint32_t)(mine + 1)) - 1;
#endif
    return mine;
}
AF_FN int32_t pool_find_hole(State& W) {
    AF_SHARED(&W);
    const int lane = lane_id();
    const int32_t hw = W.ev_hw;
    int32_t mine = 0x7FFFFFFF;
#pragma unroll 1
    for (int32_t k = lane; k < hw; k += WARP)
        if (evt_load(W, k) == INF_BITS) { mine = k; break; }
    mine = (int32_t)w_min((uint32_t)mine);
    return mine == 0x7FFFFFFF ? -1 : mine;
}

AF_FN void push_seq(State& W, double t, uint32_t payload, uint32_t s) {
    AF_SHARED(&W);
    if (!(t < W.horizon)) return;       // env.run(until=T): events at >= T never fire
    if (AF_UNLIKELY(t == W.now)) W.busy |= 1u;   // a zero-delay timeout: it competes with the now-queue
    int32_t slot;
    if (W.ev_last_free >= 0) { slot = W.ev_last_free; W.ev_last_free = -1; }
    else if (W.ev_hole >= 0) { slot = W.ev_hole; W.ev_hole = -1; }
    else {
        slot = W.ev_hw;
        if (AF_UNLIKELY(slot - W.ev_live > POOL_SLACK)) {
            slot = pool_find_hole(W);                // fragmented: fill the lowest hole instead of appending --
        } else {                                     // a fresh event at the top would keep every later scan long
            if (AF_UNLIKELY(slot >= AF_L.ev_total)) { W.flags |= AF_FLAG_EVENT_OVERFLOW; return; }
            W.ev_hw = slot + 1;
        }
    }
    uint64_t key = ((uint64_t)s << 32) | payload;
    if (AF_IN_SMEM(slot, AF_L.ev_smem)) { tbl_ev_time(W)[slot] = t; tbl_ev_key(W)[slot] = key; }
    else { W.sp_ev_time[slot - AF_L.ev_smem] = t; W.sp_ev_key[slot - AF_L.ev_smem] = key; }
    uint32_t live = (uint32_t)(++W.ev_live);
    if (live > W.peak_ev) W.peak_ev = live;
}
AF_IN void push(State& W, double t, uint32_t payload) { push_seq(W, t, payload, W.seq++); }

// The (time, seq)-minimum of the pool, without removing it.  `more` = at least one other
// event carries the same time.  False when the pool is empty.  (single call site)
struct PoolMin { uint64_t tbits, key; int32_t slot, hole; bool more; };
AF_IN bool pool_scan(State& W, PoolMin& m) {
    if (W.ev_live == 0) return false;
    const int lane = lane_id();
    const int32_t hw = W.ev_hw;
    uint64_t bt = ~0ull, bk = ~0ull; int32_t bi = -1; int32_t hole = 0x7FFFFFFF;
    bool dup = false;                 // this lane holds two events at ITS earliest time
#pragma unroll 1
    for (int32_t k = lane; k < hw; k += WARP) {
        uint64_t tb = evt_load(W, k);
        if (tb == INF_BITS) { if (k < hole) hole = k; continue; }
        uint64_t kk = evk_load(W, k);
        if (tb < bt) { bt = tb; bk = kk; bi = k; dup = false; }
        else if (tb == bt) { dup = true; if (kk < bk) { bk = kk; bi = k; } }
    }
#if AF_DEVICE_CODE
    uint32_t hi = (uint32_t)(bt >> 32), lo = (uint32_t)bt;
    uint32_t mhi = w_min(hi);
    bool cand = (hi == mhi) && bi >= 0;
    uint32_t mlo = w_min(cand ? lo : 0xFFFFFFFFu);
    cand = cand && lo == mlo;
    uint32_t b = w_ballot(cand);
    const bool more = __popc(b) > 1 || w_ballot(cand && dup) != 0;
    if (__popc(b) > 1) {              // equal times: the earlier push wins (SimPy eid order)
        uint32_t sq = (uint32_t)(bk >> 32);
        uint32_t msq = w_min(cand ? sq : 0xFFFFFFFFu);
        cand = cand && sq == msq;
        b = w_ballot(cand);
    }
    int owner = __ffs((int)b) - 1;
    uint32_t k_hi = w_shfl((uint32_t)(bk >> 32), owner), k_lo = w_shfl((uint32_t)bk, owner);
    m.slot = (int32_t)w_shfl((uint32_t)bi, owner);
    m.tbits = ((uint64_t)mhi << 32) | mlo;
    m.key = ((uint64_t)k_hi << 32) | k_lo;
    m.hole = (int32_t)w_min((uint32_t)hole);
    m.more = more;
#else
    m.slot = bi; m.tbits = bt; m.key = bk; m.hole = hole; m.more = dup;
#endif
    return true;
}
AF_IN void pool_remove(State& W, const PoolMin& m) {
    const int32_t hw = W.ev_hw, slot = m.slot;
    if (AF_IN_SMEM(slot, AF_L.ev_smem)) tbl_ev_time(W)[slot] = afr::u2d(INF_BITS);
    else W.sp_ev_time[slot - AF_L.ev_smem] = afr::u2d(INF_BITS);
    W.ev_live -= 1;
    int32_t nhw = hw;
    if (slot == hw - 1) {
        nhw = hw - 1;
        W.ev_hw = nhw;
        if (AF_UNLIKELY(nhw - W.ev_live > POOL_SLACK)) { nhw = pool_top(W) + 1; W.ev_hw = nhw; }
        W.ev_last_free = -1;
    }
    else W.ev_last_free = slot;
    W.ev_hole = m.hole < nhw ? m.hole : -1;
}


// ---- now-queue: FIFO of zero-delay continuation items (seq << 32 | kind:3 aux:9 slot:20) ----
enum : uint32_t { I_PUT = 0, I_GOT = 1, I_CLIENT_LOOP = 2, I_RAM_OK = 3, I_CPU_OK = 4, I_CPU_PUT = 5, I_RAM_PUT = 6 };
constexpr uint32_t NODE_CLIENT = 0, NODE_LB = 1, NODE_SERVER0 = 2;   // `aux` of I_PUT / I_GOT
// Fast path.  When the now-queue is empty and no pool event shares the current instant, an
// item pushed as the LAST action of the running item would be the very next thing to run:
// its effect may be applied at once (same state transitions, no ring round trip).  This is
// what keeps the common no-tie case as cheap as an inlined cascade.
AF_IN bool can_fuse(const State& W) { return AF_LIKELY(W.busy == 0); }

AF_FN void nq_push(State& W, uint32_t kind, uint32_t aux, uint32_t slot) {
    AF_SHARED(&W);
    uint32_t tail = W.nq_tail;
    if (tail - W.nq_head >= (uint32_t)NQ_CAP) { W.flags |= AF_FLAG_NOWQ_OVERFLOW; return; }
    tbl_nq(W)[tail & (NQ_CAP - 1)] = ((uint64_t)(W.seq++) << 32) | mk_payload(kind, aux, slot);
    W.nq_tail = tail + 1;
    W.busy += 2u;
}

// ---------------------------------------------------------------------------------
// generator: samplers/poisson_poisson.py:52-82 / gaussian_poisson.py:64-94.
// Returns false when the sampler is exhausted; otherwise the next yielded gap.
// ---------------------------------------------------------------------------------

AF_IN bool gen_next_gap(State& W, double& gap) {
    const double T = W.horizon;
    double vnow = W.g_vnow, wend = W.g_window_end, lam = W.g_lam;
    uint32_t pos = W.g_pos;
    bool ok = false;
    for (;;) {
        if (!(vnow < T)) break;
        if (vnow >= wend) {
            wend = vnow + (double)AF_L.window_s;
            afr::GenDraw d = afr::gen_users(AF_G.seed, W.replica, pos, AF_L.users_dist, W.users_mean, W.users_sigma);
            pos = d.pos;
            lam = d.value * W.rate_per_user;
        }
        if (lam <= 0.0) { vnow = wend; continue; }
        afr::Src s = afr::make_gen(AF_G.seed, W.replica, pos);
        double u = s.next53();
        pos = s.pos;
        if (u < 1e-15) u = 1e-15;                   // max(u, 1e-15)
        double dt = afr::af_div(-afr::af_log(1.0 - u), lam);
        if (vnow + dt > T) break;
        if (vnow + dt >= wend) { vnow = wend; continue; }
        vnow += dt;
        gap = dt;
        ok = true;
        break;
    }
    W.g_vnow = vnow; W.g_window_end = wend; W.g_lam = lam; W.g_pos = pos;
    return ok;
}

AF_IN void arm_generator(State& W) {
    W.need_arrival = 0;
    double gap;
    if (!W.g_done && gen_next_gap(W, gap)) push_seq(W, W.now + gap, mk_payload(K_ARRIVAL, 0, 0), W.arm_seq);
    else W.g_done = 1;
}

// ---------------------------------------------------------------------------------
// edges: EdgeRuntime.transport -> Initialize (URGENT) -> _deliver up to its timeout
// (edge.py:73-107).  Called at the END of the item that called transport().
// ---------------------------------------------------------------------------------

AF_FN void edge_send(State& W, uint32_t slot, uint32_t e, uint32_t rid, uint32_t hops) {
    AF_SHARED(&W);
    EdgeS& E = tbl_edge(W)[e];
    uint32_t s = W.seq++;                            // the timeout's place in SimPy's eid order
    const double dropout = E.dropout;
    afr::EdgeDraw d = afr::edge_draw(AF_G.seed, W.replica, rid, hops, (int)(E.meta & 7u), E.mean, E.sigma, dropout);
    E.sent += 1;
    if (d.u < dropout) {                            // the request vanishes (edge.py:79-86)
        E.dropped += 1;
        rq_release(W, slot);
        return;
    }
    E.conn += 1;
    occ_add(W, OC_WORDS * AF_L.n_servers + (int32_t)e, 1);
    double effective = d.transit + E.spike;        // spike read at SEND time (edge.py:94-106)
    push_seq(W, W.now + effective, mk_payload(K_DELIVER, e, slot), s);
}

// ---------------------------------------------------------------------------------
// Stores (mailboxes).  Store.put appends at once and schedules the put event (I_PUT); the
// consumer's pending get() is served when THAT event is processed (-> I_GOT); a consumer
// that calls get() on a non-empty store is served at once (-> I_GOT).   SURVEY.md App. A
// ---------------------------------------------------------------------------------
// `yield box.get()` of the node's consumer process
AF_FN void consumer_get_slow(State& W, uint32_t node) {
    AF_SHARED(&W);
    InboxS& b = tbl_inbox(W)[node];
    uint32_t it = fifo_pop(W, b.head, b.tail);
    nq_push(W, I_GOT, node, it);
}
AF_IN void consumer_get(State& W, uint32_t node) {
    InboxS& b = tbl_inbox(W)[node];
    if (AF_UNLIKELY(b.head != NIL)) consumer_get_slow(W, node); else b.pending = 1;
}

// ---------------------------------------------------------------------------------
// server: Container semantics (FIFO, head-of-line blocking; level changes at CALL time,
// waiters are woken when the put/get EVENT is processed or a new request walks the queue)
// ---------------------------------------------------------------------------------
// Container._trigger_get over the CPU queue: grant heads while a core is free
// (returns true when `watch` was among the granted: its get is "triggered" at the call)
AF_FN bool cpu_walk(State& W, ServerS& S, uint32_t sidx, uint32_t watch) {
    AF_SHARED(&W); AF_SHARED(&S);
    bool hit = false;
#pragma unroll 1
    while (S.cpuq_head != NIL && S.cpu_free > 0) {
        uint32_t w = fifo_pop(W, S.cpuq_head, S.cpuq_tail);
        S.cpu_free -= 1;
        occ_srv(W, sidx, OC_CPU, 1);
        hit = hit || w == watch;
        nq_push(W, I_CPU_OK, sidx, w);
    }
    return hit;
}
// ... over the RAM queue: grant heads while they fit, stop at the first that does not
AF_FN void ram_walk(State& W, ServerS& S, uint32_t sidx) {
    AF_SHARED(&W); AF_SHARED(&S);
#pragma unroll 1
    while (S.ramq_head != NIL) {
        const uint32_t need = S.ramq_head_need;      // kept beside the queue: no trip to the waiter's record
        if ((int32_t)need > S.ram_free) break;
        uint32_t w = fifo_pop(W, S.ramq_head, S.ramq_tail);
        occ_srv(W, sidx, OC_RAM_WAIT, -1);
        if (S.ramq_head != NIL) S.ramq_head_need = tbl_endpoint(W)[pk_ep(rq_load(W, S.ramq_head).pack)].total_ram;
        S.ram_free -= (int32_t)need;
        nq_push(W, I_RAM_OK, sidx, w);
    }
}
// RAM.get(total_ram) of a request that cannot be served at once: join the queue, walk it
AF_IN void ram_enqueue(State& W, ServerS& S, uint32_t sidx, uint32_t slot, uint32_t total_ram) {
    if (S.ramq_head == NIL) S.ramq_head_need = total_ram;
    fifo_push(W, S.ramq_head, S.ramq_tail, slot);
    occ_srv(W, sidx, OC_RAM_WAIT, 1);
    ram_walk(W, S, sidx);
}

constexpr uint32_t PK_WAIT = 1u << 30;   // the request sits in the ready queue (server.py:215-217)

// The `for step in selected_endpoint.steps` loop (server.py:197-255) from the request's current
// step up to its next yield, and the tail of the handler (server.py:257-276).
AF_FN void run_steps(State& W, uint32_t slot, uint32_t sidx, uint32_t rid, uint32_t pack) {
    AF_SHARED(&W);
    ServerS& S = tbl_server(W)[sidx];
    const EndpointS ep = tbl_endpoint(W)[pk_ep(pack)];
    for (;;) {
        const uint32_t st = pk_step(pack);
        if (st < ep.n_steps) {
            const StepS sp = tbl_step(W)[ep.step_begin + st];
            if (sp.kind == AF_STEP_CPU) {
                if (pack & PK_IO) { pack &= ~PK_IO; S.io_q -= 1; occ_srv(W, sidx, OC_IO, -1); }
                if (!(pack & PK_CORE)) {             // cpu_req = CPU.get(1); yield cpu_req
                    if (S.cpuq_head == NIL && S.cpu_free > 0 && can_fuse(W)) {
                        S.cpu_free -= 1;             // granted, and its get event would run next
                        occ_srv(W, sidx, OC_CPU, 1);
                        pack |= PK_CORE;
                    } else {
                        fifo_push(W, S.cpuq_head, S.cpuq_tail, slot);
                        if (!cpu_walk(W, S, sidx, slot)) { pack |= PK_WAIT; S.ready_q += 1; occ_srv(W, sidx, OC_CPU_WAIT, 1); }   // not cpu_req.triggered
                        rq_set_pack(W, slot, pack);
                        return;
                    }
                }
                // the request holds a core: past its server's deadline it abandons -- the tail of the handler as it
                // stands (core, then RAM), no forward (DESIGN.md §3.13)
                // (the start time is read from the record only for a server with a deadline: a register across every
                //  call of run_steps costs af_sim_kernel a spill)
                if (AF_UNLIKELY(tbl_deadline(W)[sidx] < INF_DEADLINE) && W.now - rq_load(W, slot).t0 > tbl_deadline(W)[sidx]) {
                    pack = (pack & ~0xFF00u) | (ep.n_steps << 8) | PK_EXPIRED;
                    continue;
                }
                rq_set_pack(W, slot, pack);
                push(W, W.now + sp.dur, mk_payload(K_STEP_END, sidx, slot));
                return;
            }
            if (pack & PK_CORE) {                    // yield CPU.put(1): level rises NOW
                S.cpu_free += 1;
                occ_srv(W, sidx, OC_CPU, -1);
                if (can_fuse(W)) { if (AF_UNLIKELY(S.cpuq_head != NIL)) cpu_walk(W, S, sidx, NIL); pack &= ~PK_CORE; continue; }
                rq_set_pack(W, slot, pack);
                nq_push(W, I_CPU_PUT, sidx, slot);
                return;
            }
            if (!(pack & PK_IO)) { pack |= PK_IO; S.io_q += 1; occ_srv(W, sidx, OC_IO, 1); }
            rq_set_pack(W, slot, pack);
            push(W, W.now + sp.dur, mk_payload(K_STEP_END, sidx, slot));
            return;
        }
        // end of the endpoint (server.py:257-276)
        if (pack & PK_CORE) {                        // yield CPU.put(1)
            S.cpu_free += 1;
            occ_srv(W, sidx, OC_CPU, -1);
            if (can_fuse(W)) { if (AF_UNLIKELY(S.cpuq_head != NIL)) cpu_walk(W, S, sidx, NIL); pack &= ~PK_CORE; continue; }
            rq_set_pack(W, slot, pack);
            nq_push(W, I_CPU_PUT, sidx, slot);
            return;
        }
        if (pack & PK_IO) { pack &= ~PK_IO; S.io_q -= 1; occ_srv(W, sidx, OC_IO, -1); }
        rq_set_pack(W, slot, pack);
        if (ep.total_ram) {                          // yield RAM.put(total_ram): level rises NOW
            S.ram_in_use -= (int32_t)ep.total_ram;
            occ_srv(W, sidx, OC_RAM_MB, -(int32_t)ep.total_ram);
            S.ram_free += (int32_t)ep.total_ram;
            if (!can_fuse(W)) { nq_push(W, I_RAM_PUT, sidx, slot); return; }
            if (AF_UNLIKELY(S.ramq_head != NIL)) ram_walk(W, S, sidx);   // the put event would run next: waiters, then forward
        }
        S.adm_left += 1;                             // out of service: handed to the out-edge, or dropped past its deadline
        if (AF_UNLIKELY(pack & PK_EXPIRED)) { S.expired += 1; rq_release(W, slot); return; }
        edge_send(W, slot, S.out_edge, rid, pk_hops(pack));
        return;
    }
}

// the CPU.put(1) event of `slot` is processed: waiters are re-examined, then the request goes on
AF_IN void on_cpu_put(State& W, uint32_t slot, uint32_t sidx) {
    ServerS& S = tbl_server(W)[sidx];
    cpu_walk(W, S, sidx, NIL);
    ReqRec r = rq_load(W, slot);
    run_steps(W, slot, sidx, r.rid, r.pack & ~PK_CORE);   // core_locked = False; same step again
}

// A site's process takes a request at W.now: true when its rate limit R throttles it (counted), else it spends a token
// (afr::rl_pass; DESIGN.md §3.14).  Out of line: the check is off the path of launches without a limit.
AF_FN bool rl_throttle(State& W, RateS& R) {
    double tat = R.tat;
    if (afr::rl_pass(tat, W.now, R.tau, R.lim)) { R.tat = tat; return false; }
    R.throttled += 1;
    return true;
}

// ServerRuntime._dispatcher resumed with `slot` (server.py:303-313), then the head of
// _handle_request (server.py:88-149), which runs as an URGENT Initialize right after
AF_IN void server_got(State& W, uint32_t slot, uint32_t sidx, const ReqRec& r) {
    consumer_get(W, NODE_SERVER0 + sidx);            // the dispatcher loops back to get() first
    // throttled at its rate limit, before the admission limit (§3.14): gone as a shed request is
    if (AF_UNLIKELY(tbl_rate(W)[sidx].tau != 0.0) && rl_throttle(W, tbl_rate(W)[sidx])) { rq_release(W, slot); return; }
    ServerS& S = tbl_server(W)[sidx];
    if (AF_UNLIKELY(S.adm_left == 0)) {              // at its admission limit: shed at the door, no handler
        S.rejected += 1;
        rq_release(W, slot);
        return;
    }
    S.adm_left -= 1;
    uint32_t pack = r.pack + 1;                      // record_hop(SERVER)
    uint32_t epi = 0;
    const uint32_t n_ep = S.n_ep;
    if (n_ep > 1) {
        afr::Src src = afr::make_request(AF_G.seed, W.replica, afr::P_SERVER, r.rid, pk_hops(pack));
        src.load(0);
        epi = (uint32_t)(((uint64_t)src.w.x * n_ep) >> 32);
    }
    const uint32_t ep_global = S.ep_begin + epi;
    pack = (pack & 0xFFu) | (ep_global << 16);       // step 0, flags clear
    rq_set_pack(W, slot, pack);
    const uint32_t total_ram = tbl_endpoint(W)[ep_global].total_ram;
    if (total_ram) {                                 // yield RAM.get(total_ram)
        if (!(S.ramq_head == NIL && (int32_t)total_ram <= S.ram_free && can_fuse(W))) {
            ram_enqueue(W, S, sidx, slot, total_ram);
            return;
        }
        S.ram_free -= (int32_t)total_ram;            // granted, and its get event would run next
        S.ram_in_use += (int32_t)total_ram;
        occ_srv(W, sidx, OC_RAM_MB, (int32_t)total_ram);
    }
    run_steps(W, slot, sidx, r.rid, pack);
}

// ---------------------------------------------------------------------------------
// client: completion (client.py:62-69 + analyzer.py:83-125)
// ---------------------------------------------------------------------------------
// per-window latency bands: one to the latency's bin and the latency in 32.32 fixed point to the two sum words of the
// finish window (af_lane.cuh's lat_add; the caller has checked that this completion counts)
AF_IN void lat_add(const State& W, double now, double lat) {
    int32_t b = (int32_t)ceil(now) - 1;
    b = b < 0 ? 0 : b;
    if (b >= AF_L.horizon_s) return;
    uint64_t* row = W.lat + (uint64_t)((uint32_t)b / W.lat_window) * afr::LAT_ROW;
    red_add_u64(row + afr::hist_bin(lat), 1u);
    const uint64_t u = afr::lat_fixed32(lat);
    if (u >> 32) red_add_u64(row + AF_HIST_BINS, u >> 32);
    red_add_u64(row + AF_HIST_BINS + 1, u & 0xFFFFFFFFull);
}

AF_IN void complete(State& W, uint32_t slot, double t0) {
    const double now = W.now;
    const double lat = now - t0;                     // finish - start (analyzer.py:86-89)
    const uint32_t done = ++W.completed;
    W.lat_sum += lat;
    W.lat_sumsq += lat * lat;
    if (lat < W.lat_min) W.lat_min = lat;
    if (lat > W.lat_max) W.lat_max = lat;
    if (lat > W.timeout) W.late += 1;                // later than the client timeout (DESIGN.md §3.13)
    const bool traced = W.traced != 0;
    if (traced && (int32_t)(done - 1) >= AF_L.trace_clock_cap) W.flags |= AF_FLAG_TRACE_TRUNCATED;
    if (lane_id() == 0) {
        const uint64_t local = W.local;
        if (AF_L.collect_hist) red_add_u32(&AF_G.hist[local * AF_HIST_BINS + (uint32_t)afr::hist_bin(lat)], 1u);
        // a completion counts in the latency bands while no stop flag is set (what follows a flag may differ from a
        // re-run), and in a re-run only from the first one the thread-per-replica pass did not add
        if (W.lat != nullptr && done > W.lat_from && !(W.flags & STOP_FLAGS)) lat_add(W, now, lat);
        if (AF_L.collect_thr) {
            // bucket k counts (k, k+1] (analyzer.py:108-125)
            int32_t b = (int32_t)ceil(now) - 1;
            b = b < 0 ? 0 : b;
            if (b < AF_L.horizon_s) red_add_u32(&AF_G.thr[local * (uint64_t)AF_L.horizon_s + (uint32_t)b], 1u);
        }
        if (traced && (int32_t)(done - 1) < AF_L.trace_clock_cap) {
            double* p = AF_G.trace_clocks + (local * (uint64_t)AF_L.trace_clock_cap + (done - 1)) * 2;
            p[0] = t0; p[1] = now;
        }
    }
    w_sync();
    rq_release(W, slot);
}

// ---------------------------------------------------------------------------------
// a node's consumer process resumes with `slot` (the StoreGet event is processed):
// client.py:43-71, load_balancer.py:60-72 + routing/lb_algorithms.py:10-36, server.py:303-313
// ---------------------------------------------------------------------------------
AF_FN void node_got(State& W, uint32_t node, uint32_t slot, double t0, uint32_t rid, uint32_t pack_in) {
    AF_SHARED(&W);
    ReqRec r; r.t0 = t0; r.rid = rid; r.pack = pack_in;   // the record as the caller already holds it
    if (node >= NODE_SERVER0) { server_got(W, slot, node - NODE_SERVER0, r); return; }
    r.pack += 1;                                     // record_hop(client / LB)
    if (node == NODE_CLIENT) {
        if (pk_hops(r.pack) > 3) {                   // client.py:62: back from the servers
            complete(W, slot, r.t0);
            if (can_fuse(W)) consumer_get(W, NODE_CLIENT);
            else nq_push(W, I_CLIENT_LOOP, 0, 0);    // yield completed_box.put(state)
            return;
        }
        rq_set_pack(W, slot, r.pack);
        consumer_get(W, NODE_CLIENT);
        edge_send(W, slot, (uint32_t)AF_L.client_edge, r.rid, pk_hops(r.pack));
        return;
    }
    rq_set_pack(W, slot, r.pack);
    if (AF_UNLIKELY(W.lb_rl.tau != 0.0) && rl_throttle(W, W.lb_rl)) {   // throttled at the LB's rate limit: gone
        consumer_get(W, NODE_LB);                                          // before the pick (§3.14)
        rq_release(W, slot);
        return;
    }
    uint32_t* lb = tbl_lb(W);
    const int32_t n = W.lb_n;
    // every covered server is down: the reference dies here (StopIteration inside round_robin); the replica
    // stops and says so (flatten() rejects timelines that can reach this state)
    if (AF_UNLIKELY(n <= 0)) { W.flags |= AF_FLAG_LB_EMPTY; return; }
    uint32_t pick = lb[0];
    if (W.lb_algo == AF_LB_ROUND_ROBIN) {            // lb_algorithms.py:22-36
#pragma unroll 1
        for (int32_t i = 1; i < n; ++i) lb[i - 1] = lb[i];
        lb[n - 1] = pick;
    } else {                                         // least_connections, :10-20 (first min wins)
        uint32_t best = tbl_edge(W)[pick].conn;
#pragma unroll 1
        for (int32_t i = 1; i < n; ++i) {
            uint32_t c = tbl_edge(W)[lb[i]].conn;
            if (c < best) { best = c; pick = lb[i]; }
        }
    }
    consumer_get(W, NODE_LB);
    edge_send(W, slot, pick, r.rid, pk_hops(r.pack));
}

// ---------------------------------------------------------------------------------
// one zero-delay item (single call site in run_replica)
// ---------------------------------------------------------------------------------
AF_IN void run_item(State& W, uint32_t item) {
    const uint32_t kind = item >> 29, aux = (item >> SLOT_BITS) & AUX_MASK;
    uint32_t slot = item & SLOT_MASK;
    AF_TRACE("it t=%.17g kind=%u aux=%u slot=%u\n", W.now, kind, aux, slot);
    if (kind == I_PUT) {                             // a StorePut event is processed
        InboxS& b = tbl_inbox(W)[aux];
        if (b.pending) { b.pending = 0; nq_push(W, I_GOT, aux, fifo_pop(W, b.head, b.tail)); }
    } else if (kind == I_GOT) {
        { ReqRec r = rq_load(W, slot); node_got(W, aux, slot, r.t0, r.rid, r.pack); }
    } else if (kind == I_CLIENT_LOOP) {
        consumer_get(W, NODE_CLIENT);
    } else if (kind == I_RAM_OK) {                   // the RAM get event is processed: the handler resumes
        ServerS& S = tbl_server(W)[aux];
        ReqRec r = rq_load(W, slot);
        S.ram_in_use += (int32_t)tbl_endpoint(W)[pk_ep(r.pack)].total_ram;
        occ_srv(W, aux, OC_RAM_MB, (int32_t)tbl_endpoint(W)[pk_ep(r.pack)].total_ram);
        run_steps(W, slot, aux, r.rid, r.pack);
    } else if (kind == I_CPU_OK) {                   // the CPU get event is processed
        ServerS& S = tbl_server(W)[aux];
        ReqRec r = rq_load(W, slot);
        if (r.pack & PK_WAIT) { r.pack &= ~PK_WAIT; S.ready_q -= 1; occ_srv(W, aux, OC_CPU_WAIT, -1); }
        run_steps(W, slot, aux, r.rid, r.pack | PK_CORE);
    } else if (kind == I_CPU_PUT) {
        on_cpu_put(W, slot, aux);
    } else {                                         // I_RAM_PUT: waiters first, then forward
        ServerS& S = tbl_server(W)[aux];
        ram_walk(W, S, aux);
        ReqRec r = rq_load(W, slot);
        S.adm_left += 1;
        if (AF_UNLIKELY(r.pack & PK_EXPIRED)) { S.expired += 1; rq_release(W, slot); return; }   // past its deadline: no forward
        edge_send(W, slot, S.out_edge, r.rid, pk_hops(r.pack));
    }
}

// ---------------------------------------------------------------------------------
// timed events
// ---------------------------------------------------------------------------------
// edge.py:110-116: the edge's timeout fired
AF_IN void on_deliver(State& W, uint32_t slot, uint32_t e) {
    EdgeS& E = tbl_edge(W)[e];
    E.conn -= 1;
    occ_add(W, OC_WORDS * AF_L.n_servers + (int32_t)e, -1);
    const uint32_t meta = E.meta;
    ReqRec r = rq_load(W, slot);
    r.pack += 1;                                     // record_hop(edge)
    const uint32_t tk = (meta >> 3) & 3u;
    const uint32_t node = tk == AF_TARGET_CLIENT ? NODE_CLIENT : (tk == AF_TARGET_LB ? NODE_LB : NODE_SERVER0 + (meta >> 5));
    if (can_fuse(W)) {                               // (implies: every inbox empty, every consumer in get())
        node_got(W, node, slot, r.t0, r.rid, r.pack);   // put -> pending get -> resume, nothing in between
        return;                                      // (the consumer stores the record's new pack itself)
    }
    rq_set_pack(W, slot, r.pack);
    InboxS& b = tbl_inbox(W)[node];
    fifo_push(W, b.head, b.tail, slot);              // Store.put: items.append now ...
    nq_push(W, I_PUT, node, slot);                   // ... the put event is processed later
}

// rqs_generator.py:97-119
AF_IN void on_arrival(State& W) {
    const uint32_t rid = ++W.generated;
    uint32_t slot = rq_alloc(W);
    // the generator asks the sampler for the next gap right after transport(): its timeout is
    // scheduled BEFORE the edge's delivery timeout.  The seq is reserved here; the gap itself
    // is drawn at the single arm_generator() site in run_replica().
    W.arm_seq = W.seq++;
    W.need_arrival = 1;
    if (slot == NIL) return;
    ReqRec r; r.t0 = W.now; r.rid = rid; r.pack = 1;  // record_hop(generator)
    rq_store(W, slot, r);
    edge_send(W, slot, (uint32_t)AF_L.gen_edge, rid, 1u);
}

// ---------------------------------------------------------------------------------
// event injection (injection.py:167-226): all marks of this instant, then re-arm
// ---------------------------------------------------------------------------------
AF_FN void on_spike(State& W) {
    AF_SHARED(&W);
    int32_t cur = W.spike_cur;
    double t = tbl_spike(W)[cur].fire;
#pragma unroll 1
    while (cur < AF_L.n_spike && tbl_spike(W)[cur].fire == t) {
        const SpikeS m = tbl_spike(W)[cur];
        tbl_edge(W)[m.edge].spike = tbl_edge(W)[m.edge].spike + m.delta;
        ++cur;
    }
    W.spike_cur = cur;
    if (cur < AF_L.n_spike) push(W, tbl_spike(W)[cur].fire, mk_payload(K_SPIKE, 0, 0));
}
AF_FN void on_outage(State& W) {
    AF_SHARED(&W);
    int32_t cur = W.outage_cur;
    double t = tbl_outage(W)[cur].fire;
    uint32_t* lb = tbl_lb(W);
    int32_t n = W.lb_n;
#pragma unroll 1
    while (cur < AF_L.n_outage && tbl_outage(W)[cur].fire == t) {
        const OutageS m = tbl_outage(W)[cur];
        ++cur;
        if (m.lb_edge < 0) continue;
        int32_t at = -1;
#pragma unroll 1
        for (int32_t i = 0; i < n; ++i) if (lb[i] == (uint32_t)m.lb_edge) { at = i; break; }
        if (at >= 0) {                               // pop (DOWN) or move_to_end (UP)
#pragma unroll 1
            for (int32_t i = at + 1; i < n; ++i) lb[i - 1] = lb[i];
            --n;
        }
        if (!m.down) lb[n++] = (uint32_t)m.lb_edge;
    }
    W.lb_n = n;
    W.outage_cur = cur;
    if (cur < AF_L.n_outage) push(W, tbl_outage(W)[cur].fire, mk_payload(K_OUTAGE, 0, 0));
}

// ---------------------------------------------------------------------------------
// sampled metrics: emit every collector tick ordered before (t, ev_seq) (collector.py:50-66)
// ---------------------------------------------------------------------------------
AF_FN void take_samples(State& W, double t, uint32_t ev_seq) {
    AF_SHARED(&W);
    const int lane = lane_id();
    const int32_t n_series = AF_L.n_series, ns3 = 3 * AF_L.n_servers;
    const bool srv_on = (AF_L.metrics_mask & 7u) == 7u;          // collector.py:60-63
    const bool edge_on = (AF_L.metrics_mask & AF_METRIC_EDGE_CONN) != 0;
    double tick = W.tick_time;
    uint32_t tseq = W.tick_seq, nt = W.n_ticks, seq = W.seq;
    const double horizon = W.horizon;
    const bool traced = W.traced != 0;
    // per-tick bands: from tick band_from on, a series whose value differs from the last one emitted adds the difference
    // (and that of the squares) at this tick's index of the group's difference rows -- the lane engine's contract,
    // evaluated at the ticks instead of at the changes; the first tick emits the full value and joins the count
    // Distribution bands likewise: from band_from on, a selected series whose value differs from the last one emitted
    // moves from bin(prev) to bin(v) at this tick (nothing when the bin stays); the first tick adds bin(v) alone.  Both
    // kinds read the last emitted value before it is updated.
    uint64_t* const band = W.band;
    const uint64_t stride = W.band_stride, sq = (uint64_t)n_series * stride;
    uint32_t* const dist = W.dist;
    const uint32_t last_bin = W.dist_bins - 1u;
#pragma unroll 1
    while ((tick < t || (tick == t && tseq < ev_seq)) && tick < horizon) {
#pragma unroll 1
        for (int32_t j = lane; j < n_series; j += WARP) {
            uint32_t v;
            if (j < ns3) {
                if (!srv_on) continue;
                const ServerS& S = tbl_server(W)[j / 3];
                int m = j % 3;
                v = (uint32_t)(m == 0 ? S.ready_q : (m == 1 ? S.io_q : S.ram_in_use));
            } else {
                if (!edge_on) continue;
                v = tbl_edge(W)[j - ns3].conn;
            }
            tbl_samp_sum(W)[j] += v;
            if (v > tbl_samp_max(W)[j]) tbl_samp_max(W)[j] = v;
            if (traced && (int32_t)nt < AF_L.trace_tick_cap)
                AF_G.trace_series[(W.local * (uint64_t)n_series + (uint32_t)j) * (uint64_t)AF_L.trace_tick_cap + nt] = v;
            if ((band != nullptr || dist != nullptr) && nt >= W.band_from) {
                const uint32_t p = tbl_band_prev(W)[j];
                const int32_t s = dist != nullptr ? W.dist_slot[j] : -1;
                if (s >= 0) {
                    uint32_t* row = dist + (uint64_t)s * W.dist_series_words + (uint64_t)nt * W.dist_bins;
                    uint32_t b1 = afr::gauge_bin(v); b1 = b1 < last_bin ? b1 : last_bin;
                    if (nt == W.band_from) red_add_u32(row + b1, 1u);
                    else {
                        uint32_t b0 = afr::gauge_bin(p); b0 = b0 < last_bin ? b0 : last_bin;
                        if (b0 != b1) { red_add_u32(row + b0, ~0u); red_add_u32(row + b1, 1u); }
                    }
                }
                if (v != p) {
                    if (band != nullptr) {
                        uint64_t* row = band + (uint64_t)(1 + j) * stride + nt;
                        red_add_u64(row, (uint64_t)v - (uint64_t)p);
                        red_add_u64(row + sq, (uint64_t)v * v - (uint64_t)p * p);
                    }
                    tbl_band_prev(W)[j] = v;
                }
            }
        }
        if (band != nullptr && nt == W.band_from && lane == 0) red_add_u64(band + nt, 1u);
        nt += 1;
        tseq = seq++;                                 // the collector re-arms its timeout here
        tick = tick + AF_L.sample_period;
    }
    w_sync();
    W.tick_time = tick; W.tick_seq = tseq; W.n_ticks = nt; W.seq = seq;
}

// a replica that a stop flag ends leaves its group at the tick it stopped at: its last emitted values and its count
// are taken back there (nothing was emitted when it stopped before band_from), and the frozen ticks to the horizon add
// nothing (band = nullptr)
AF_FN void band_stop(State& W) {
    AF_SHARED(&W);
    const int lane = lane_id();
    const uint64_t n = W.n_ticks, stride = W.band_stride, sq = (uint64_t)AF_L.n_series * stride;
    if (n > W.band_from && W.band != nullptr) {
#pragma unroll 1
        for (int32_t j = lane; j < AF_L.n_series; j += WARP) {
            const uint64_t p = tbl_band_prev(W)[j];
            if (p == 0) continue;
            uint64_t* row = W.band + (uint64_t)(1 + j) * stride + n;
            red_add_u64(row, 0 - p);
            red_add_u64(row + sq, 0 - p * p);
        }
        if (lane == 0) red_add_u64(W.band + n, ~0ull);
    }
    if (n > W.band_from && W.dist != nullptr) {       // distribution bands: the last emitted bin, a value of 0 included
        const uint32_t last_bin = W.dist_bins - 1u;
#pragma unroll 1
        for (int32_t j = lane; j < AF_L.n_series; j += WARP) {
            const int32_t s = W.dist_slot[j];
            if (s < 0) continue;
            uint32_t b = afr::gauge_bin(tbl_band_prev(W)[j]);
            b = b < last_bin ? b : last_bin;
            red_add_u32(W.dist + (uint64_t)s * W.dist_series_words + n * W.dist_bins + b, ~0u);
        }
    }
    w_sync();
    W.band = nullptr; W.dist = nullptr;
    w_sync();
}

// ---------------------------------------------------------------------------------
// set-up / write-back (once per replica)
// ---------------------------------------------------------------------------------
AF_IN void bind(State& W, unsigned char* ws, uint64_t warp_slot) {
    (void)ws;
    uint64_t ev_sp = (uint64_t)(AF_L.ev_total - AF_L.ev_smem), rq_sp = (uint64_t)(AF_L.rq_total - AF_L.rq_smem);
    W.sp_ev_time = AF_G.spill_ev_time + warp_slot * ev_sp;
    W.sp_ev_key = AF_G.spill_ev_key + warp_slot * ev_sp;
    W.sp_rq_rec = AF_G.spill_rq_rec + warp_slot * rq_sp;
    W.sp_rq_next = AF_G.spill_rq_next + warp_slot * rq_sp;
}

// a site's rate and burst -> its tau and tolerance L (afr::rl_params; a rate of 0: no limit, tau = 0; a burst below 1
// reads as 1)
AF_IN void rl_finish(double& tau, double& lim) {
    const double rate = tau, burst = lim;
    tau = 0.0; lim = 0.0;
    if (rate > 0.0) afr::rl_params(rate, burst < 1.0 ? 1.0 : burst, tau, lim);
}

// the requests each site of the replica throttled, to its output row `out` ([n_servers + 1], the LB last)
AF_FN void rl_write_back(State& W, uint32_t* out) {
    AF_SHARED(&W);
    for (int32_t i = lane_id(); i < AF_L.n_servers; i += WARP) out[i] = tbl_rate(W)[i].throttled;
    if (lane_id() == 0) out[AF_L.n_servers] = W.lb_rl.throttled;
    w_sync();
}

// `spikes` / `outages`: the replica's mark tables (its timeline row, or the scenario's)
// The caller has set W.lb_rl.tau / .lim to the scenario's LB rate and burst (rl_finish turns them into tau and L).
AF_FN void load_params(State& W, const AfSpikeMark* spikes, const AfOutageMark* outages, double client_timeout) {
    AF_SHARED(&W);
    const int lane = lane_id();
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_edges; i += WARP) {
        const AfEdge a = AF_G.edges[i];
        EdgeS e;
        e.mean = a.mean; e.sigma = a.sigma; e.dropout = a.dropout; e.spike = 0.0;
        e.meta = (uint32_t)a.dist | ((uint32_t)a.target_kind << 3) | ((uint32_t)a.target_index << 5);
        e.conn = 0; e.sent = 0; e.dropped = 0;
        tbl_edge(W)[i] = e;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_servers; i += WARP) {
        const AfServer a = AF_G.servers[i];
        ServerS s;
        s.cpu_free = a.cpu_cores; s.ram_free = a.ram_mb; s.ready_q = 0; s.io_q = 0; s.ram_in_use = 0;
        s.ramq_head = s.ramq_tail = s.cpuq_head = s.cpuq_tail = NIL;
        s.out_edge = (uint32_t)a.out_edge; s.ep_begin = (uint32_t)a.endpoint_begin; s.n_ep = (uint32_t)a.n_endpoints;
        s.ramq_head_need = 0; s.adm_left = a.max_in_service > 0 ? (uint32_t)a.max_in_service : 0xFFFFFFFFu; s.rejected = 0;
        s.expired = 0;
        tbl_deadline(W)[i] = a.deadline > 0.0 ? a.deadline : INF_DEADLINE;
        RateS q; q.tat = 0.0; q.tau = a.rate_limit; q.lim = (double)a.burst; q.throttled = 0; q.pad = 0;   // (rl_finish)
        tbl_rate(W)[i] = q;
        tbl_server(W)[i] = s;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_endpoints; i += WARP) {
        const AfEndpoint a = AF_G.endpoints[i];
        EndpointS e; e.step_begin = (uint32_t)a.step_begin; e.n_steps = (uint32_t)a.n_steps;
        e.total_ram = (uint32_t)a.total_ram; e.pad = 0;
        tbl_endpoint(W)[i] = e;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_steps; i += WARP) {
        const AfStep a = AF_G.steps[i];
        StepS s; s.dur = a.duration; s.kind = (uint32_t)a.kind; s.pad = 0;
        tbl_step(W)[i] = s;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_lb_edges; i += WARP) tbl_lb(W)[i] = (uint32_t)AF_G.lb_edges[i];
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_spike; i += WARP) {
        const AfSpikeMark a = spikes[i];
        SpikeS s; s.fire = a.fire_time; s.delta = a.delta; s.edge = (uint32_t)a.edge; s.pad = 0;
        tbl_spike(W)[i] = s;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_outage; i += WARP) {
        const AfOutageMark a = outages[i];
        OutageS o; o.fire = a.fire_time; o.lb_edge = a.lb_edge; o.down = a.down;
        tbl_outage(W)[i] = o;
    }
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_series; i += WARP) { tbl_samp_sum(W)[i] = 0; tbl_samp_max(W)[i] = 0; }
    if (W.band != nullptr || W.dist != nullptr) for (int32_t i = lane; i < AF_L.n_series; i += WARP) tbl_band_prev(W)[i] = 0;
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_servers + 2; i += WARP) { InboxS b; b.head = b.tail = NIL; b.pending = 1; b.pad = 0; tbl_inbox(W)[i] = b; }
    w_sync();
    W.users_mean = AF_L.users_mean; W.users_sigma = AF_L.users_sigma; W.rate_per_user = AF_L.rate_per_user;
    W.lb_algo = AF_L.lb_algo;
    W.timeout = client_timeout > 0.0 ? client_timeout : INF_DEADLINE; W.late = 0; W.late_pad = 0;
    W.lb_rl.tat = 0.0; W.lb_rl.throttled = 0; W.lb_rl.pad = 0;
    // sweep overrides of this replica (uniform: every lane applies every column)
    const uint64_t replica = AF_G.replica_begin + W.local;     // (W.replica is its stream)
    if (AF_L.n_sweep_cols > 0 && replica >= AF_G.sweep_first && replica - AF_G.sweep_first < AF_G.sweep_rows) {
        const double* row = AF_G.sweep_vals + (replica - AF_G.sweep_first) * (uint64_t)AF_L.n_sweep_cols;
        bool uncovered = false;
#pragma unroll 1
        for (int32_t c = 0; c < AF_L.n_sweep_cols; ++c) {
            const AfSweepColumn col = AF_G.sweep_cols[c];
            double v = row[c];
            switch (col.field) {
            case AF_FIELD_USERS_MEAN: W.users_mean = v; break;
            case AF_FIELD_USERS_SIGMA: W.users_sigma = v; break;
            case AF_FIELD_RATE_PER_USER: W.rate_per_user = v; break;
            case AF_FIELD_EDGE_MEAN: tbl_edge(W)[col.index].mean = v; break;
            case AF_FIELD_EDGE_SIGMA: tbl_edge(W)[col.index].sigma = v; break;
            case AF_FIELD_EDGE_DROPOUT: tbl_edge(W)[col.index].dropout = v; break;
            case AF_FIELD_SERVER_CPU_CORES: tbl_server(W)[col.index].cpu_free = (int32_t)v; break;
            case AF_FIELD_SERVER_RAM_MB: tbl_server(W)[col.index].ram_free = (int32_t)v; break;
            case AF_FIELD_STEP_DURATION: tbl_step(W)[col.index].dur = v; break;
            case AF_FIELD_ENDPOINT_RAM: tbl_endpoint(W)[col.index].total_ram = (uint32_t)v; break;
            case AF_FIELD_SPIKE_DELTA:
                tbl_spike(W)[col.index].delta = tbl_spike(W)[col.index].delta < 0.0 ? -v : v; break;
            case AF_FIELD_LB_COVERED: if (v == 0.0) { tbl_lb(W)[col.index] = NIL; uncovered = true; } break;
            case AF_FIELD_LB_ALGORITHM: W.lb_algo = (int32_t)v; break;
            case AF_FIELD_SERVER_MAX_IN_SERVICE: tbl_server(W)[col.index].adm_left = v > 0.0 ? (uint32_t)v : 0xFFFFFFFFu; break;
            case AF_FIELD_SERVER_DEADLINE: tbl_deadline(W)[col.index] = v > 0.0 ? v : INF_DEADLINE; break;
            case AF_FIELD_CLIENT_TIMEOUT: W.timeout = v > 0.0 ? v : INF_DEADLINE; break;
            case AF_FIELD_SERVER_RATE: tbl_rate(W)[col.index].tau = v; break;       // (rate and burst until rl_finish)
            case AF_FIELD_SERVER_BURST: tbl_rate(W)[col.index].lim = v; break;
            case AF_FIELD_LB_RATE: W.lb_rl.tau = v; break;
            case AF_FIELD_LB_BURST: W.lb_rl.lim = v; break;
            default: break;
            }
        }
        w_sync();
        if (uncovered) {                             // the LB order without the edges the row uncovers (lane 0 alone: in place)
            if (lane == 0) {
                uint32_t* lb = tbl_lb(W);
                int32_t n = 0;
#pragma unroll 1
                for (int32_t i = 0; i < AF_L.n_lb_edges; ++i) if (lb[i] != NIL) lb[n++] = lb[i];
                W.lb_n = n;
            }
            w_sync();
        }
    }
    // rate limits (DESIGN.md §3.14): each site's (rate, burst) of the scenario or the row -> (tau, L)
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_servers; i += WARP) rl_finish(tbl_rate(W)[i].tau, tbl_rate(W)[i].lim);
    if (lane == 0) rl_finish(W.lb_rl.tau, W.lb_rl.lim);
    w_sync();
    if (AF_G.redo_list) {                            // a re-run: the first pass left partial counts in the accumulating outputs
        if (AF_L.collect_hist) for (int32_t b = lane; b < AF_HIST_BINS; b += WARP) AF_G.hist[W.local * AF_HIST_BINS + (uint32_t)b] = 0;
        if (AF_L.collect_thr) for (int32_t b = lane; b < AF_L.horizon_s; b += WARP) AF_G.thr[W.local * (uint64_t)AF_L.horizon_s + (uint32_t)b] = 0;
        w_sync();
    }
}

AF_FN void write_back(State& W) {
    AF_SHARED(&W);
    const int lane = lane_id();
    const uint64_t local = W.local;
#pragma unroll 1
    for (int32_t i = lane; i < AF_L.n_edges; i += WARP) {
        AF_G.edge_sent[local * (uint64_t)AF_L.n_edges + (uint32_t)i] = tbl_edge(W)[i].sent;
        AF_G.edge_dropped[local * (uint64_t)AF_L.n_edges + (uint32_t)i] = tbl_edge(W)[i].dropped;
    }
#pragma unroll 1
    for (int32_t j = lane; j < AF_L.n_series; j += WARP) {
        AF_G.samp_sum[local * (uint64_t)AF_L.n_series + (uint32_t)j] = tbl_samp_sum(W)[j];
        AF_G.samp_max[local * (uint64_t)AF_L.n_series + (uint32_t)j] = tbl_samp_max(W)[j];
    }
    if (lane == 0) {
        AfReplicaStats st;
        st.n_events = W.n_events; st.generated = W.generated; st.completed = W.completed;
        st.flags = W.flags; st.n_ticks = W.n_ticks; st.peak_events = W.peak_ev; st.peak_requests = W.peak_rq;
        st.lat_sum = W.lat_sum; st.lat_sumsq = W.lat_sumsq;
        st.lat_min = W.completed ? W.lat_min : 0.0; st.lat_max = W.lat_max;
        st.p50 = st.p95 = st.p99 = afr::u2d(0x7FF8000000000000ull);
        AF_G.stats[local] = st;
        if (W.traced) { AF_G.trace_counts[local * 2] = W.completed; AF_G.trace_counts[local * 2 + 1] = W.n_ticks; }
    }
    w_sync();
}

// ---------------------------------------------------------------------------------
// the replica
// ---------------------------------------------------------------------------------
AF_IN void run_replica(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl, const StreamArgs& rs) {
    W.local = local_index;
    const uint64_t id = AF_G.replica_begin + local_index;     // the replica's rows; its draws come from its stream
    const uint64_t si = id - rs.first;
    W.replica = si < rs.rows ? rs.stream_of[si] : id;
    W.now = 0.0; W.horizon = (double)AF_L.horizon_s; W.seq = 0;
    W.ev_hw = 0; W.ev_live = 0; W.ev_last_free = -1; W.ev_hole = -1; W.peak_ev = 0;
    W.nq_head = 0; W.nq_tail = 0; W.busy = 0;
    W.rq_free = NIL; W.rq_hw = 0; W.rq_live = 0; W.peak_rq = 0;
    W.g_vnow = 0.0; W.g_window_end = 0.0; W.g_lam = 0.0; W.g_pos = 0; W.generated = 0; W.g_done = 0;
    W.lb_n = AF_L.n_lb_edges;
    W.spike_cur = 0; W.outage_cur = 0;
    W.n_ticks = 0; W.completed = 0; W.flags = 0; W.n_events = 0;
    W.lat_sum = 0.0; W.lat_sumsq = 0.0; W.lat_min = afr::u2d(INF_BITS); W.lat_max = 0.0;
    W.traced = (int64_t)local_index < (int64_t)AF_L.trace_replicas ? 1u : 0u;
    W.band = nullptr; W.band_from = 0; W.band_stride = band.stride; W.band_prev_off = (uint32_t)band.prev_off;
    W.lat = nullptr; W.lat_from = 0; W.lat_window = band.lat_window;
    W.dist = nullptr; W.dist_slot = band.dist_slot; W.dist_series_words = band.dist_series_words; W.dist_bins = band.dist_bins;
    W.occ = nullptr; W.occ_scale = band.occ_scale;
    if (band.occ != nullptr) {                        // a re-run starts over: the first pass's row is overwritten
        const int32_t cols = OC_WORDS * AF_L.n_servers + AF_L.n_edges;
        W.occ = band.occ + local_index * (uint64_t)cols;
        for (int32_t c = lane_id(); c < cols; c += WARP) W.occ[c] = 0;
    }
    if (band.stride || band.lat_window || band.dist_rows) {
        const uint64_t i = id - band.first;
        const uint32_t g = i < band.n ? band.group[i] : band.groups;
        if (band.stride || band.dist_rows)                           // a re-run continues where the lane pass stopped
            W.band_from = AF_G.redo_list ? band.from[local_index] : 0u;
        if (band.stride) W.band = band.rows + (uint64_t)g * band.group_words;
        if (band.dist_rows) W.dist = band.dist_rows + (uint64_t)g * band.dist_group_words;
        if (band.lat_window) {
            W.lat = band.lat_rows + (uint64_t)g * band.lat_windows * afr::LAT_ROW;
            W.lat_from = AF_G.redo_list ? band.lat_from[local_index] : 0u;
        }
    }
    w_sync();
    {
        const uint64_t r = id - tl.first;
        const bool own = r < tl.rows;
        W.lb_rl.tau = band.lb_rate; W.lb_rl.lim = (double)band.lb_burst;
        load_params(W, own ? tl.spikes + r * (uint64_t)AF_L.n_spike : AF_G.spikes, own ? tl.outages + r * (uint64_t)AF_L.n_outage : AF_G.outages,
                    band.client_timeout);
    }

    // start order of the reference (simulation_runner.py:339-342, 301-336):
    // spike timeline, outage timeline, generator, ..., collector
    if (AF_L.n_spike > 0) {
        if (tbl_spike(W)[0].fire == 0.0) on_spike(W); else push(W, tbl_spike(W)[0].fire, mk_payload(K_SPIKE, 0, 0));
    }
    if (AF_L.n_outage > 0) {
        if (tbl_outage(W)[0].fire == 0.0) on_outage(W); else push(W, tbl_outage(W)[0].fire, mk_payload(K_OUTAGE, 0, 0));
    }
    W.arm_seq = W.seq++; W.need_arrival = 1;
    W.tick_seq = W.seq++;
    W.tick_time = 0.0 + AF_L.sample_period;

    uint64_t n_events = 0;
    for (;;) {
        if (W.need_arrival) arm_generator(W);
        const uint32_t busy = W.busy;
        const bool have_item = busy >= 2u;
        if (have_item && !(busy & 1u)) {             // no pool event shares this instant: just drain
            uint32_t item = (uint32_t)tbl_nq(W)[W.nq_head & (NQ_CAP - 1)];
            W.nq_head += 1;
            W.busy = busy - 2u;
            run_item(W, item);
            if (W.flags & STOP_FLAGS) break;
            continue;
        }
        PoolMin m;
        const bool have_ev = pool_scan(W, m);
        if (have_item) {
            const uint64_t front = tbl_nq(W)[W.nq_head & (NQ_CAP - 1)];
            const bool same_t = have_ev && m.tbits == afr::d2u(W.now);
            if (!(same_t && (uint32_t)(m.key >> 32) < (uint32_t)(front >> 32))) {
                W.busy = (same_t ? busy : (busy & ~1u)) - 2u;
                W.nq_head += 1;
                run_item(W, (uint32_t)front);
                if (W.flags & STOP_FLAGS) break;
                continue;
            }
        } else if (!have_ev) break;
        pool_remove(W, m);
        const double t = afr::u2d(m.tbits);
        const uint32_t payload = (uint32_t)m.key, ev_seq = (uint32_t)(m.key >> 32);
        W.busy = (W.busy & ~1u) | (m.more ? 1u : 0u);
        if (!(W.flags & STOP_FLAGS)) {    // (arm_generator's timeout did not fit the pool: stop at the ticks taken so far)
            const double tick = W.tick_time;
            if (tick < t || (tick == t && W.tick_seq < ev_seq)) take_samples(W, t, ev_seq);
        }
        W.now = t;
        ++n_events;
        uint32_t kind = payload >> 29, aux = (payload >> SLOT_BITS) & AUX_MASK, slot = payload & SLOT_MASK;
        AF_TRACE("ev t=%.17g seq=%u kind=%u aux=%u slot=%u rid=%u\n", t, ev_seq, kind, aux, slot,
                 kind == K_DELIVER || kind == K_STEP_END ? rq_load(W, slot).rid : 0u);
        if (kind == K_DELIVER) on_deliver(W, slot, aux);
        else if (kind == K_STEP_END) {
            ReqRec r = rq_load(W, slot);
            run_steps(W, slot, aux, r.rid, r.pack + (1u << 8));   // the timeout fired: next step
        }
        else if (kind == K_ARRIVAL) on_arrival(W);
        else if (kind == K_SPIKE) on_spike(W);
        else on_outage(W);
        if (W.flags & STOP_FLAGS) break;
    }
    W.n_events = n_events;
    if ((W.band != nullptr || W.dist != nullptr) && (W.flags & STOP_FLAGS)) band_stop(W);   // before the frozen ticks to the horizon
    take_samples(W, W.horizon, 0u);                   // ticks strictly before the horizon
    write_back(W);
    if (band.server_rejected != nullptr) {
        for (int32_t i = lane_id(); i < AF_L.n_servers; i += WARP)
            band.server_rejected[local_index * (uint64_t)AF_L.n_servers + (uint32_t)i] = tbl_server(W)[i].rejected;
        w_sync();
    }
    if (band.server_expired != nullptr) {
        for (int32_t i = lane_id(); i < AF_L.n_servers; i += WARP)
            band.server_expired[local_index * (uint64_t)AF_L.n_servers + (uint32_t)i] = tbl_server(W)[i].expired;
        if (lane_id() == 0) band.late[local_index] = W.late;
        w_sync();
    }
    if (band.throttled != nullptr) rl_write_back(W, band.throttled + local_index * ((uint64_t)AF_L.n_servers + 1));
}
AF_IN void run_replica(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl) {
    const StreamArgs none = {};
    run_replica(W, local_index, band, tl, none);
}
AF_IN void run_replica(State& W, uint64_t local_index, const BandArgs& band) {
    const TimelineArgs none = {};
    run_replica(W, local_index, band, none);
}
AF_IN void run_replica(State& W, uint64_t local_index) {
    const BandArgs off = {};
    run_replica(W, local_index, off);
}

}  // namespace afc
