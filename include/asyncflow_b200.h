/* asyncflow_b200 -- C ABI of the H100-native batched discrete-event engine.
 *
 * This is the drop-in boundary for ONE hot path of AsyncFlow (reference
 * /root/reference, v0.1.1): everything `SimulationRunner.run()` executes between
 * "payload validated" and "ResultsAnalyzer built"
 * (reference src/asyncflow/runtime/simulation_runner.py:349-376), i.e. SimPy's
 * Environment.step() loop (simulation_runner.py:369) driving the actors
 *   runtime/actors/rqs_generator.py:97-119   request generator
 *   runtime/actors/edge.py:73-124            network edges
 *   runtime/actors/client.py:43-71           client
 *   runtime/actors/load_balancer.py:60-72    load balancer
 *   runtime/actors/server.py:79-313          server event loop
 *   runtime/events/injection.py:35-226       spikes / outages
 *   metrics/collector.py:50-66               sampled metrics
 * for MANY independent replicas at once (one replica per GPU thread; replicas whose
 * queues outgrow the nominal-load pools are re-run one per warp with large HBM pools).
 *
 * The reference is pure Python and has no FFI; the two seams a maintainer binds
 * are documented in INTEGRATION.md:
 *   IN : SimulationRunner(env=, simulation_input=SimulationPayload)
 *        (simulation_runner.py:52-57)  ->  AfScenario (+ AfSweep)
 *   OUT: ResultsAnalyzer(client=, servers=, edges=, settings=)
 *        (metrics/analyzer.py:51-58)   <-  af_fetch_* below
 *
 * Conventions: every call returns 0 on success or a negative AfStatus; the text
 * of the last error of an engine is af_last_error().  The engine owns all device
 * memory.  Host buffers are caller-owned and only borrowed for the duration of
 * the call.  One engine per device; calls on one engine must be serialised by
 * the caller.  No CPU fallback exists: af_engine_create fails (AF_ERR_CUDA)
 * when no sm_90 device is usable.
 */
#ifndef ASYNCFLOW_B200_H
#define ASYNCFLOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AF_ABI_VERSION 12

typedef enum AfStatus {
    AF_OK = 0,
    AF_ERR_INVALID = -1,   /* bad argument / inconsistent scenario            */
    AF_ERR_CUDA = -2,      /* CUDA runtime error or no usable device          */
    AF_ERR_STATE = -3,     /* call out of order (e.g. run before upload)      */
    AF_ERR_NOMEM = -4      /* device or host allocation failed                */
} AfStatus;

/* Distribution codes: reference config/constants.py:39-51 (Distribution).     */
enum { AF_DIST_POISSON = 0, AF_DIST_NORMAL = 1, AF_DIST_LOG_NORMAL = 2,
       AF_DIST_EXPONENTIAL = 3, AF_DIST_UNIFORM = 4 };
/* Edge targets: which inbox an edge delivers to (simulation_runner.py:219-230) */
enum { AF_TARGET_CLIENT = 0, AF_TARGET_LB = 1, AF_TARGET_SERVER = 2 };
/* Step kinds after flattening.  RAM steps are folded into AfEndpoint.total_ram:
 * the reference reserves their sum up front and skips them in the step loop
 * (runtime/actors/server.py:106-110, 147-149, 197-255).                        */
enum { AF_STEP_CPU = 0, AF_STEP_IO = 1 };
/* Load-balancer algorithms (routing/lb_algorithms.py:39-43); -1 = no LB.       */
enum { AF_LB_NONE = -1, AF_LB_ROUND_ROBIN = 0, AF_LB_LEAST_CONNECTIONS = 1 };
/* enabled_sample_metrics bits (config/constants.py SampledMetricName)          */
enum { AF_METRIC_READY_QUEUE = 1, AF_METRIC_IO_SLEEP = 2, AF_METRIC_RAM_IN_USE = 4,
       AF_METRIC_EDGE_CONN = 8 };

typedef struct AfEdge {          /* schemas/topology/edges.py:25-58 */
    double mean;                 /* latency.mean                                   */
    double sigma;                /* latency.variance, which numpy receives as the  *
                                  * standard deviation (common_helpers.py:31,40)   */
    double dropout;              /* dropout_rate                                   */
    int32_t dist;                /* AF_DIST_*                                      */
    int32_t target_kind;         /* AF_TARGET_*                                    */
    int32_t target_index;        /* server index when target_kind==AF_TARGET_SERVER*/
    int32_t reserved;
} AfEdge;

typedef struct AfServer {        /* schemas/topology/nodes.py:52-104 */
    int32_t cpu_cores;
    int32_t ram_mb;
    int32_t out_edge;            /* the server's single outgoing edge              */
    int32_t endpoint_begin;      /* first AfEndpoint of this server                */
    int32_t n_endpoints;
    int32_t max_in_service;      /* admission limit: requests in service at once   *
                                  * (0 = no limit; see AF_FIELD_SERVER_MAX_IN_SERVICE) */
    double deadline;             /* request deadline in seconds from creation      *
                                  * (0 = none; see AF_FIELD_SERVER_DEADLINE)       */
    double rate_limit;           /* token-bucket rate in requests per second       *
                                  * (0 = none; see AF_FIELD_SERVER_RATE)           */
    int32_t burst;               /* the bucket's size (0 reads as 1)               */
    int32_t reserved;            /* 0                                              */
} AfServer;

typedef struct AfEndpoint {      /* schemas/topology/endpoint.py:92-102 */
    int32_t step_begin;          /* first AfStep (CPU / IO steps only)             */
    int32_t n_steps;
    int32_t total_ram;           /* sum of necessary_ram over the RAM steps        */
    int32_t reserved;
} AfEndpoint;

typedef struct AfStep {
    double duration;             /* cpu_time or io_waiting_time, seconds           */
    int32_t kind;                /* AF_STEP_CPU / AF_STEP_IO                       */
    int32_t reserved;
} AfStep;

/* Event-injection marks, already sorted and with the FIRE TIME the reference's
 * `dt = t - last_t; yield timeout(dt)` chain produces in f64
 * (runtime/events/injection.py:167-226).                                         */
typedef struct AfSpikeMark {
    double fire_time;
    double delta;                /* +spike_s at START, -spike_s at END             */
    int32_t edge;
    int32_t reserved;
} AfSpikeMark;

typedef struct AfOutageMark {
    double fire_time;
    int32_t lb_edge;             /* LB->server edge to remove/re-append; -1 = no-op *
                                  * (server not behind the LB, injection.py:213-215)*/
    int32_t down;                /* 1 = SERVER_DOWN, 0 = SERVER_UP                 */
} AfOutageMark;

typedef struct AfScenario {
    /* generator: schemas/workload/rqs_generator.py:10-27 */
    int32_t users_dist;          /* AF_DIST_POISSON or AF_DIST_NORMAL              */
    int32_t window_s;            /* user_sampling_window                           */
    double users_mean;
    double users_sigma;          /* avg_active_users.variance (used as sigma)      */
    double rate_per_user;        /* avg_request_per_minute_per_user.mean / 60      */
    /* settings: schemas/settings/simulation.py:16-44 */
    int32_t horizon_s;           /* total_simulation_time                          */
    uint32_t metrics_mask;       /* AF_METRIC_* bits                               */
    double sample_period;        /* sample_period_s                                */
    /* topology */
    int32_t n_edges, n_servers, n_endpoints, n_steps;
    int32_t n_lb_edges;          /* 0 when there is no load balancer               */
    int32_t lb_algo;             /* AF_LB_*                                        */
    int32_t gen_edge;            /* generator's out edge                           */
    int32_t client_edge;         /* client's out edge                              */
    int32_t n_spike_marks, n_outage_marks;
    const AfEdge* edges;
    const AfServer* servers;
    const AfEndpoint* endpoints;
    const AfStep* steps;
    const int32_t* lb_edges;     /* initial round-robin order (edge indices)       */
    const AfSpikeMark* spike_marks;
    const AfOutageMark* outage_marks;
    double client_timeout;       /* the client counts a completion later than this  *
                                  * as late (0 = none; AF_FIELD_CLIENT_TIMEOUT)     */
    double lb_rate_limit;        /* the load balancer's token-bucket rate in        *
                                  * requests per second (0 = none; AF_FIELD_LB_RATE) */
    int32_t lb_burst;            /* its bucket's size (0 reads as 1)                */
    int32_t reserved2;           /* 0                                               */
} AfScenario;

/* Per-replica overrides of scenario fields: the Monte-Carlo sweep
 * (BASELINE.json north_star; reference ROADMAP.md:23-27).                          */
enum {
    AF_FIELD_USERS_MEAN = 0, AF_FIELD_USERS_SIGMA = 1, AF_FIELD_RATE_PER_USER = 2,
    AF_FIELD_EDGE_MEAN = 3, AF_FIELD_EDGE_SIGMA = 4, AF_FIELD_EDGE_DROPOUT = 5,
    AF_FIELD_SERVER_CPU_CORES = 6, AF_FIELD_SERVER_RAM_MB = 7,
    AF_FIELD_STEP_DURATION = 8, AF_FIELD_ENDPOINT_RAM = 9,
    AF_FIELD_SPIKE_DELTA = 10,   /* index = spike mark; sign is kept by the engine */
    AF_FIELD_LB_COVERED = 11,    /* index = position in lb_edges; 1 = behind the LB as in the scenario, 0 = not */
    AF_FIELD_LB_ALGORITHM = 12,  /* index 0; an AF_LB_* algorithm (round robin or least connections)           */
    AF_FIELD_SERVER_MAX_IN_SERVICE = 13,  /* index = server; an admission limit, 0 = none (AfServer.max_in_service) */
    AF_FIELD_SERVER_DEADLINE = 14,  /* index = server; a request deadline in seconds, 0 = none (AfServer.deadline) */
    AF_FIELD_CLIENT_TIMEOUT = 15,   /* index 0; the client's timeout in seconds, 0 = none (AfScenario.client_timeout) */
    AF_FIELD_SERVER_RATE = 16,      /* index = server; a rate limit in requests per second, 0 = none (AfServer.rate_limit) */
    AF_FIELD_SERVER_BURST = 17,     /* index = server; its burst, an integer >= 1 (AfServer.burst)                 */
    AF_FIELD_LB_RATE = 18,          /* index 0; the load balancer's rate limit, 0 = none (AfScenario.lb_rate_limit) */
    AF_FIELD_LB_BURST = 19,         /* index 0; its burst, an integer >= 1 (AfScenario.lb_burst)                   */
    AF_FIELD_COUNT = 20
};
/* Load-balancer rows (DESIGN.md §3.11).  A replica whose row sets AF_FIELD_LB_COVERED of position k to 0 runs without
 * the LB edge lb_edges[k]: its round-robin order is lb_edges with the uncovered edges left out; the server and its other
 * edges stay.  AF_FIELD_LB_ALGORITHM picks the replica's algorithm.  Replicas without a row keep the scenario's pool
 * and algorithm.  af_sweep_upload refuses (AF_ERR_INVALID) either field on a scenario without a load balancer, an index
 * out of range, a value other than 0 or 1, and a row that covers no edge (naming the row).  af_run refuses a launch in
 * which a row uncovers an LB edge that the outage marks it runs with (its timeline row, else the scenario's) still name:
 * give such rows timeline rows whose marks for that server have lb_edge = -1. */
/* Admission limits (DESIGN.md §3.12).  A server with a limit L > 0 (AfServer.max_in_service, or the replica's
 * AF_FIELD_SERVER_MAX_IN_SERVICE value) admits a request its dispatcher takes from the inbox only while fewer than L
 * requests are in service there -- from admission until the handler hands them to the server's out-edge, RAM and core
 * waits included.  A request beyond the limit is shed at the door: no hop, no endpoint draw, no handler; it never
 * reaches the client (as an edge dropout), its in-edge still counts it as sent, and af_fetch_server_rejected counts it.
 * No random number is drawn, so replicas sharing a stream see the same traffic whatever their limits.  Replicas without
 * a row keep the scenario's limits.  af_scenario_upload refuses a negative max_in_service; af_sweep_upload refuses an
 * index out of range and a value that is not an integer in [0, 2^31) (naming the row). */
/* Request deadlines (DESIGN.md §3.13).  A request's age is now - t0, t0 the time the generator created it, so a deadline
 * holds end to end across a chain of servers.  A server with a deadline D > 0 (AfServer.deadline, or the replica's
 * AF_FIELD_SERVER_DEADLINE value) checks the age once per CPU step, once the request holds a core and before the step's
 * timeout.  When now - t0 > D the request abandons: it releases its core and RAM as a finished handler does, in the same
 * order, and is not handed to the out-edge; af_fetch_server_expired counts it (and it leaves service for the admission
 * limit).  A request that never runs a CPU step there, or waits for RAM, is not checked until its first CPU step.
 * The client timeout T > 0 (AfScenario.client_timeout or AF_FIELD_CLIENT_TIMEOUT) counts a completion with
 * now - t0 > T in af_fetch_late; the completion counts everywhere else as before.  Neither draws a random number.
 * af_scenario_upload and af_sweep_upload refuse negative, NaN and infinite values (the latter naming the row). */
/* Rate limits (DESIGN.md §3.14).  A site -- a server, or the load balancer -- with a rate r > 0 requests per second
 * (AfServer.rate_limit / AfScenario.lb_rate_limit, or the replica's AF_FIELD_SERVER_RATE / AF_FIELD_LB_RATE value) and
 * a burst B >= 1 runs a GCRA token bucket: one f64 `tat` per site, 0 at the start.  Where the site's process takes a
 * request from its inbox at `now`, with tau = 1/r and L = (B - 1) * tau (each correctly rounded, no FMA):
 *     if (tat - now > L) the request is throttled; else tat = max(tat, now) + tau.
 * A server checks right after its dispatcher takes the request, before the admission limit: a request it throttles is
 * gone as a shed one is (no hop, no endpoint, no handler; its in-edge counts it as sent).  The load balancer checks after
 * it takes the request and records its hop, before the pick: a request it throttles moves no round-robin order and no
 * connection count.  af_fetch_throttled counts them.  No random number is drawn.  A burst of 0 in the scenario reads as
 * 1.  af_scenario_upload refuses a negative, NaN or infinite rate, a negative burst and an LB rate without a load
 * balancer; af_sweep_upload refuses a rate that is not finite and >= 0, a burst that is not an integer in [1, 2^31)
 * (naming the row), an index out of range and the LB fields on a scenario without a load balancer. */
typedef struct AfSweepColumn { int32_t field; int32_t index; } AfSweepColumn;
typedef struct AfSweep {
    int32_t n_columns;
    int32_t reserved;
    uint64_t n_rows;             /* replicas covered                               */
    const AfSweepColumn* columns;
    const double* values;        /* [n_rows][n_columns], row-major                 */
} AfSweep;

typedef struct AfOptions {
    int32_t event_capacity;      /* pending timed events per replica (0 = default) */
    int32_t request_capacity;    /* in-flight requests per replica   (0 = default) */
    int32_t warps_per_block;     /* 1..4 (0 = default 4; larger values are clamped) */
    int32_t blocks_per_sm;       /* 0 = as many as fit                             */
    int32_t collect_histogram;   /* latency histogram per replica (AF_HIST_BINS)   */
    int32_t collect_throughput;  /* completions per 1-s bucket per replica         */
    int32_t trace_replicas;      /* first N replicas of a run keep full traces     */
    int32_t trace_clock_capacity;/* (start,finish) pairs per traced replica        */
} AfOptions;

#define AF_HIST_BINS 4096        /* 128 log-linear bins per octave (<= 0.78 % wide), 2^-20 .. 2^12 s  */
#define AF_HIST_SUB_BITS 7
#define AF_HIST_MIN_EXP (-20)

/* AfReplicaStats.flags */
enum { AF_FLAG_EVENT_OVERFLOW = 1, AF_FLAG_REQUEST_OVERFLOW = 2, AF_FLAG_TRACE_TRUNCATED = 4,
       AF_FLAG_NOWQ_OVERFLOW = 8, /* > 128 zero-delay continuations pending at one instant */
       AF_FLAG_LB_EMPTY = 16      /* a request reached the load balancer while every covered server was down:
                                   * the reference raises here (routing/lb_algorithms.py:22-36 on an empty dict) */ };

typedef struct AfReplicaStats {
    uint64_t n_events;           /* timed events processed                          */
    uint32_t generated;          /* requests created (rqs_generator.py:62-64)       */
    uint32_t completed;          /* RqsClock appends (client.py:64-68)              */
    uint32_t flags;
    uint32_t n_ticks;            /* sampled-metric ticks taken (collector.py:52-53) */
    uint32_t peak_events;        /* high-water mark of pending timed events         */
    uint32_t peak_requests;      /* high-water mark of in-flight requests           */
    double lat_sum;              /* sum of (finish - start), completion order       */
    double lat_sumsq;
    double lat_min;
    double lat_max;
    double p50, p95, p99;        /* from the histogram (NaN when not collected)     */
} AfReplicaStats;

typedef struct af_engine af_engine;

int af_abi_version(void);
int af_engine_create(int device, af_engine** out);
void af_engine_destroy(af_engine* e);
const char* af_last_error(const af_engine* e);   /* e may be NULL: create errors  */

int af_engine_configure(af_engine* e, const AfOptions* opt);
/* Pass structure of af_run.
 * TWO_PASS: every replica runs on the thread-per-replica kernel (one replica per GPU thread), whose per-replica tiers
 *   are sized for nominal load (512 pending events, 2048 requests in flight, more request slots from a shared page
 *   pool); the replicas it flags are re-run by the warp-per-replica kernel with AfOptions' capacities, inside the same
 *   af_run.
 * AUTO (default): TWO_PASS when the launch has replicas for most lanes and the topology leaves the thread-per-replica
 *   kernel a useful occupancy; otherwise the warp-per-replica kernel alone (a thread runs one replica ~10x slower than
 *   a warp does: it pays off in numbers).
 * WARP / LANE pin one kernel (LANE takes AfOptions' capacities as they are and only reports overflows). */
enum { AF_MODE_AUTO = 0, AF_MODE_WARP = 1, AF_MODE_LANE = 2, AF_MODE_TWO_PASS = 3 };
int af_engine_set_mode(af_engine* e, int mode);
int af_scenario_upload(af_engine* e, const AfScenario* host_pod);
/* rows cover replicas [first_replica, first_replica + sweep->n_rows); pass NULL to clear */
int af_sweep_upload(af_engine* e, const AfSweep* sweep, uint64_t first_replica);

/* Per-replica event timelines: row r replaces the scenario's spike and outage mark tables for replica
 * first_replica + r; replicas outside [first_replica, first_replica + n_rows) keep the scenario's, as with sweep rows.
 * A row holds the scenario's number of marks of each kind (n_spike_marks, n_outage_marks), under the contract of
 * AfScenario's tables: sorted by the reference's key, fire times already folded, spike deltas signed.  Only the order,
 * times, amplitudes and targets may differ from row to row (an outage moved across another one reorders the marks).
 * af_timeline_upload refuses (AF_ERR_INVALID, naming the row) a spike mark whose edge is out of range, fire times that
 * decrease within a row, and an outage mark whose lb_edge is neither -1 nor one of the scenario's lb_edges.  NULL (or
 * n_rows = 0) clears the rows; af_scenario_upload clears them too.  af_run refuses (AF_ERR_INVALID) a launch with
 * timeline rows and an AF_FIELD_SPIKE_DELTA sweep column: that column indexes a mark in the scenario's order, which a
 * row may change, so a row carries its amplitudes in its own deltas. */
typedef struct AfTimeline {
    uint64_t n_rows;
    const AfSpikeMark* spikes;   /* [n_rows][n_spike_marks]                                            */
    const AfOutageMark* outages; /* [n_rows][n_outage_marks]                                           */
} AfTimeline;
int af_timeline_upload(af_engine* e, const AfTimeline* timeline, uint64_t first_replica);

/* Random streams (common random numbers): replica first_replica + i, i < n, draws every random number -- users,
 * inter-arrival gaps, edge latencies and dropouts, endpoint choices -- as if its replica id were stream_of[i]; every
 * other replica draws as its own id, the rule sweep and timeline rows follow.  The id still picks the replica's output
 * slot, sweep row, timeline row and band group, so two replicas with one stream see the same traffic whatever their
 * parameters.  Any uint64_t is a stream (both words of the replica half of the Philox counter).  The table costs
 * 8 bytes per replica on the device and is kept, across af_scenario_upload and af_sweep_upload, until the next
 * af_streams_upload; NULL (or n = 0) clears it.  Without a table every output is the one before tables existed, and
 * a table with stream_of[i] = first_replica + i changes no output. */
int af_streams_upload(af_engine* e, const uint64_t* stream_of, uint64_t n, uint64_t first_replica);

/* Simulate replicas [replica_begin, replica_end) start to horizon.  Asynchronous
 * on the engine's stream; af_sync / any af_fetch_* waits for it.                 */
int af_run(af_engine* e, uint64_t seed, uint64_t replica_begin, uint64_t replica_end);
int af_sync(af_engine* e);
/* device time of the last af_run (CUDA events on the engine's stream), ms        */
int af_last_run_ms(af_engine* e, float* ms_total, float* ms_sim_kernel);
/* kernels launched by this engine so far                                          */
uint64_t af_launch_count(const af_engine* e);
/* what the last af_run did */
typedef struct AfRunPasses {
    int32_t lane_pass, warp_pass;        /* which kernels ran                                            */
    int32_t lane_warps_per_sm;           /* occupancy the lane pass chose                                */
    int32_t lane_bytes;                  /* shared memory per replica in flight                          */
    int32_t lane_events_smem, lane_requests_smem;   /* split of the lane's shared-memory pool between heap
                                                       entries and request records, for the launch's
                                                       heaviest replica (each replica is split by its own
                                                       estimated load)                                  */
    uint64_t lane_replicas;              /* replicas the thread-per-replica pass ran                     */
    uint64_t warp_replicas;              /* replicas the warp-per-replica pass ran (AUTO: the flagged)   */
    int32_t lane_pool_elems;             /* 16-byte elements of a lane's pool (heap entries + records)   */
    int32_t lane_lean;                   /* 1: the lane pass ran the lean build of its loop (no spikes,
                                            outages, traces, general edge samplers or endpoint draws)    */
} AfRunPasses;
int af_last_run_passes(af_engine* e, AfRunPasses* out);

/* Results of the last af_run, n = replica_end - replica_begin entries each.       */
int af_fetch_stats(af_engine* e, AfReplicaStats* out, uint64_t n);
int af_fetch_edge_counts(af_engine* e, uint32_t* sent, uint32_t* dropped, uint64_t n); /* [n][n_edges] */
int af_fetch_histograms(af_engine* e, uint32_t* out, uint64_t n);   /* [n][AF_HIST_BINS] */
/* requests each server shed at its admission limit: [n][n_servers] (all 0 when the run had no limit) */
int af_fetch_server_rejected(af_engine* e, uint32_t* out, uint64_t n);
/* requests each server dropped past its deadline: [n][n_servers]; completions later than the client timeout: [n]
 * (all 0 when the run had no deadline and no timeout) */
int af_fetch_server_expired(af_engine* e, uint32_t* out, uint64_t n);
int af_fetch_late(af_engine* e, uint32_t* out, uint64_t n);
/* requests each site throttled at its rate limit: [n][n_servers + 1], column n_servers the load balancer (all 0 when
 * the run had no rate limit) */
int af_fetch_throttled(af_engine* e, uint32_t* out, uint64_t n);
int af_fetch_throughput(af_engine* e, uint32_t* out, uint64_t n);   /* [n][horizon_s]    */
/* sampled-metric aggregates over ticks: per replica, per series j:
 *   j <  3*n_servers : server j/3, metric j%3 in {ready_queue_len, event_loop_io_sleep, ram_in_use}
 *   j >= 3*n_servers : edge j-3*n_servers, edge_concurrent_connection            */
int af_fetch_sampled(af_engine* e, uint64_t* sums, uint32_t* maxima, uint64_t n);
/* sum of the last run's per-replica histograms: out_bins[AF_HIST_BINS] (device reduction) */
int af_reduce_histograms(af_engine* e, uint64_t* out_bins);
/* full trace of one of the first `trace_replicas` replicas of the last run        */
int af_fetch_trace_clocks(af_engine* e, uint64_t local_replica, double* start_finish,
                          uint64_t capacity_pairs, uint64_t* n_pairs);
int af_fetch_trace_series(af_engine* e, uint64_t local_replica, uint32_t* values,
                          uint64_t capacity_ticks, uint64_t* n_ticks); /* [series][capacity_ticks] */

/* Per-tick sampled-metric bands over groups of replicas, accumulated on the device.
 * group_of[i] = group (< n_groups) of replica first_replica + i; NULL clears (bands off).  Every later af_run then
 * sums, for every group g, series j (the order of af_fetch_sampled) and tick k < n_ticks (the ticks a replica that
 * reaches the horizon takes):
 *   count[g][k]     replicas of g that contribute tick k
 *   sum[g][j][k]    sum of their values of series j at tick k (the value a traced replica stores at tick k)
 *   sumsq[g][j][k]  sum of the squares
 * A replica contributes every tick it took before a stop flag ended it; a replica the thread-per-replica pass flags
 * and the warp-per-replica pass re-runs inside the same af_run contributes once, in full.  Replicas without a group
 * entry contribute nothing.  Every other output is the same with bands on or off.  Rejected (AF_ERR_INVALID) when
 * group size x (bound on a gauge)^2 could wrap the u64 sums of squares (the bound is the request capacity or the
 * largest ram_mb, swept values included), when the scenario takes 5e7 ticks or more, or when the band rows,
 * (n_groups + 1) x (1 + 2 n_series) x (n_ticks + 1) x 8 bytes, exceed the device's memory; af_run checks all of it
 * again with the scenario, options and sweep of the run. */
int af_bands_upload(af_engine* e, const uint32_t* group_of, uint64_t n, uint64_t first_replica, uint32_t n_groups);
/* bands of the last af_run: count[g][k], sum[g][j][k], sumsq[g][j][k], k < min(*n_ticks, capacity_ticks), rows of
 * capacity_ticks entries; *n_ticks = the run's tick count.  Any of the three arrays may be NULL (not fetched). */
int af_fetch_bands(af_engine* e, uint32_t* count, uint64_t* sum, uint64_t* sumsq,
                   uint64_t capacity_ticks, uint64_t* n_ticks);

/* Which bands af_run accumulates over the groups of af_bands_upload (defaults: {1, 0}, the per-tick bands alone).
 * latency_window_s = w > 0 adds per-window latency bands: window k < n_windows = ceil(horizon_s / w) holds the
 * completions whose finish time lies in (k w, min((k + 1) w, horizon)] (k = (ceil(finish) - 1) / w in integers, as the
 * throughput buckets), and per group g and window k the device accumulates
 *   hist[g][k][AF_HIST_BINS]   completions per latency bin (the bins of the per-replica histograms)
 *   sum_hi[g][k], sum_lo[g][k] the sum of u = round-to-nearest(latency x 2^32) as sum(u >> 32) and sum(u & 0xFFFFFFFF):
 *                              hi x 2^32 + lo is the exact fixed-point sum while a window has < 2^32 completions
 * A completion counts while its replica has no stop flag; a replica the thread-per-replica pass flags and the
 * warp-per-replica pass re-runs inside the same af_run counts once, in full; host-side re-runs add nothing.  Every
 * other output is the same with latency bands on or off.  Rejected (AF_ERR_INVALID) when w < 0, or when the rows,
 * (n_groups + 1) x n_windows x (AF_HIST_BINS + 2) x 8 bytes, exceed the device's memory; af_bands_upload and af_run
 * check the rows again. */
typedef struct AfBandOptions {
    int32_t sampled;            /* per-tick sampled-metric bands (af_fetch_bands): 1 by default      */
    int32_t latency_window_s;   /* 0: off (default); else per-window latency bands of this width (s)  */
} AfBandOptions;
int af_bands_configure(af_engine* e, const AfBandOptions* opt);
/* latency bands of the last af_run: hist[g][k][AF_HIST_BINS], sum_hi[g][k], sum_lo[g][k] for k < min(*n_windows,
 * capacity_windows), capacity_windows windows per group; *n_windows = the run's window count.  Any array may be NULL. */
int af_fetch_latency_bands(af_engine* e, uint64_t* hist, uint64_t* sum_hi, uint64_t* sum_lo,
                           uint64_t capacity_windows, uint64_t* n_windows);

/* Per-tick distribution bands of selected sampled series over the groups of af_bands_upload, accumulated on the device.
 * series[0 .. n) are af_fetch_sampled indices (n_dist = n of them); NULL or n = 0 turns the distribution bands off
 * (the default).  Every later af_run with groups then counts, for every group g, selected series s, tick k < n_ticks
 * and value bin b < n_bins:
 *   out[g][s][k][b]   replicas of g that contribute tick k with a value of series[s] in bin b
 * Bins: a value v < 64 has bin v; above, 16 log-linear bins per octave, b = 64 + 16 (msb(v) - 6) + ((v >> (msb(v) - 4))
 * & 15) with msb(v) the index of v's highest set bit, so a bin is at most 1/16 of its lower edge wide.  n_bins =
 * bin(bound) + 1 for the bound of af_bands_upload's check (the request capacity or the largest ram_mb, swept values
 * included, of the rows this engine was given); larger values cannot occur and would count in the last bin.  The bin
 * edges do not depend on the launch, only their count does: shards of one sweep may differ in n_bins, and summing
 * them takes padding the narrower ones with empty bins.  A replica contributes every tick it took
 * before a stop flag ended it, with its value at that tick (0 included); a replica the thread-per-replica pass flags and
 * the warp-per-replica pass re-runs inside the same af_run contributes once, in full; host-side re-runs add nothing.
 * The counts are exact: a group holds fewer than 2^32 replicas.  Every other output is the same with distribution
 * bands on or off.  Rejected (AF_ERR_INVALID, with a message) when a series is out of range, not sampled by the
 * scenario or listed twice, when the scenario takes 5e7 ticks or more, or when the rows, (n_groups + 1) x n_dist x
 * (n_ticks + 1) x n_bins x 4 bytes, exceed the device's memory; af_bands_upload and af_run check all of it again.
 * AF_ERR_STATE before af_scenario_upload. */
int af_dist_bands_configure(af_engine* e, const int32_t* series, int32_t n);
/* distribution bands of the last af_run: out[g][s][k][b] for k < min(*n_ticks, capacity_ticks), capacity_ticks tick
 * rows of *n_bins bins per (g, s); *n_ticks = the run's tick count, *n_bins its bins.  out = NULL: the sizes only. */
int af_fetch_dist_bands(af_engine* e, uint32_t* out, uint64_t capacity_ticks, uint64_t* n_ticks, uint32_t* n_bins);

/* Occupancy integrals: per replica, the exact request-seconds spent in each state over [0, horizon), accumulated on the
 * device.  C = 5 n_servers + n_edges u64 columns per replica:
 *   5 s + 0  ram_wait  requests of server s blocked on its RAM (a RAM.get not granted at once)
 *   5 s + 1  cpu_wait  requests in server s's ready queue (the sampled ready_queue_len)
 *   5 s + 2  cpu       requests holding one of server s's cores (cpu_cores - free cores)
 *   5 s + 3  io        requests in server s's I/O wait (the sampled event_loop_io_sleep)
 *   5 s + 4  ram_mb    MB of server s's RAM reserved (the sampled ram_in_use): MB-seconds
 *   5 n_servers + e    requests in transit on edge e (the sampled edge_concurrent_connection)
 * A count n(t) that changes by d_i at times t_i < H (H = horizon_s) adds d_i x round-to-nearest-even((H - t_i) x 2^f)
 * to its column in u64 modular arithmetic: the final value is the integral of n over [0, H) in fixed point with
 * f = frac_bits fraction bits, within (changes / 2) x 2^-f of the exact integral, and the same bits in any summation
 * order.  Every state change counts whatever the scenario samples.  A replica the thread-per-replica pass flags and
 * the warp-per-replica pass re-runs inside the same af_run gets the re-run's row; a replica that stays stopped holds
 * what it accumulated up to the stop.  Every other output is the same with occupancy on or off.
 * on = 1 turns it on for every later af_run until changed.  af_run refuses (AF_ERR_INVALID, with a message) a launch
 * whose bound B (the request capacity or the largest ram_mb, swept values included) does not fit B x H x 2^f <= 2^64 - 1;
 * af_occupancy_configure refuses frac_bits outside [8, 32].  Pick f once for a whole sweep so that its shards share a
 * scale. */
typedef struct AfOccupancyOptions {
    int32_t on;                 /* 0: off (default)                                                          */
    int32_t frac_bits;          /* f, 8..32                                                                  */
} AfOccupancyOptions;
int af_occupancy_configure(af_engine* e, const AfOccupancyOptions* opt);
/* occupancy of the last af_run: out[n][C] (C as above); *frac_bits = its f.  AF_ERR_STATE when it was off. */
int af_fetch_occupancy(af_engine* e, uint64_t* out, uint64_t n, int32_t* frac_bits);

/* AF-RNG known-answer hook: the device's random numbers outside the state machine, n values per call
 * (the streams of oracle/afrng.py; tests/test_gpu_rng.py compares them bit for bit with oracle/afrng_c):
 *   EDGE         request ids 1..n on (replica, hop): a = dropout uniform, b = latency variate of `dist`
 *                (reference runtime/actors/edge.py:78,90 + samplers/common_helpers.py:49-89)
 *   GEN_UNIFORM  positions 0..n-1 of the replica's generator stream: a = u, b = -ln(1 - max(u, 1e-15))
 *                (samplers/poisson_poisson.py:72-74)
 *   GEN_USERS    replicas replica..replica+n-1, first window draw: a = users (`dist` = AF_DIST_POISSON or
 *                AF_DIST_NORMAL), b = stream position after the draw (poisson_poisson.py:58, gaussian_poisson.py:70)
 *   ENDPOINT     request ids 1..n: a = endpoint picked among `dist` endpoints (runtime/actors/server.py:101)
 *   LOG          a = x_i, the double whose bits are bits(mean) + i * (uint64_t)sigma (a grid in bit space, `sigma`
 *                an integer step < 2^53), b = the engine's ln(x_i)
 *   EXP          a = x_i = mean + i * sigma, b = the engine's exp(x_i)                                          */
enum { AF_SELFTEST_EDGE = 0, AF_SELFTEST_GEN_UNIFORM = 1, AF_SELFTEST_GEN_USERS = 2, AF_SELFTEST_ENDPOINT = 3,
       AF_SELFTEST_LOG = 4, AF_SELFTEST_EXP = 5 };
int af_selftest_rng(af_engine* e, uint64_t seed, uint64_t replica, int kind, int dist, double mean, double sigma,
                    uint32_t hop, uint64_t n, double* out_a, double* out_b);

#ifdef __cplusplus
}
#endif
#endif /* ASYNCFLOW_B200_H */
