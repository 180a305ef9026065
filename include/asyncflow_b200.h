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

#define AF_ABI_VERSION 2

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
    int32_t reserved;
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
} AfScenario;

/* Per-replica overrides of scenario fields: the Monte-Carlo sweep
 * (BASELINE.json north_star; reference ROADMAP.md:23-27).                          */
enum {
    AF_FIELD_USERS_MEAN = 0, AF_FIELD_USERS_SIGMA = 1, AF_FIELD_RATE_PER_USER = 2,
    AF_FIELD_EDGE_MEAN = 3, AF_FIELD_EDGE_SIGMA = 4, AF_FIELD_EDGE_DROPOUT = 5,
    AF_FIELD_SERVER_CPU_CORES = 6, AF_FIELD_SERVER_RAM_MB = 7,
    AF_FIELD_STEP_DURATION = 8, AF_FIELD_ENDPOINT_RAM = 9,
    AF_FIELD_SPIKE_DELTA = 10,   /* index = spike mark; sign is kept by the engine */
    AF_FIELD_COUNT = 11
};
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
} AfRunPasses;
int af_last_run_passes(af_engine* e, AfRunPasses* out);

/* Results of the last af_run, n = replica_end - replica_begin entries each.       */
int af_fetch_stats(af_engine* e, AfReplicaStats* out, uint64_t n);
int af_fetch_edge_counts(af_engine* e, uint32_t* sent, uint32_t* dropped, uint64_t n); /* [n][n_edges] */
int af_fetch_histograms(af_engine* e, uint32_t* out, uint64_t n);   /* [n][AF_HIST_BINS] */
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

/* AF-RNG known-answer hook: the device's random numbers outside the state machine, n values per call
 * (the streams of oracle/afrng.py; tests/test_gpu_rng.py compares them bit for bit with oracle/afrng_c):
 *   EDGE         request ids 1..n on (replica, hop): a = dropout uniform, b = latency variate of `dist`
 *                (reference runtime/actors/edge.py:78,90 + samplers/common_helpers.py:49-89)
 *   GEN_UNIFORM  positions 0..n-1 of the replica's generator stream: a = u, b = -ln(1 - max(u, 1e-15))
 *                (samplers/poisson_poisson.py:72-74)
 *   GEN_USERS    replicas replica..replica+n-1, first window draw: a = users (`dist` = AF_DIST_POISSON or
 *                AF_DIST_NORMAL), b = stream position after the draw (poisson_poisson.py:58, gaussian_poisson.py:70)
 *   ENDPOINT     request ids 1..n: a = endpoint picked among `dist` endpoints (runtime/actors/server.py:101)   */
enum { AF_SELFTEST_EDGE = 0, AF_SELFTEST_GEN_UNIFORM = 1, AF_SELFTEST_GEN_USERS = 2, AF_SELFTEST_ENDPOINT = 3 };
int af_selftest_rng(af_engine* e, uint64_t seed, uint64_t replica, int kind, int dist, double mean, double sigma,
                    uint32_t hop, uint64_t n, double* out_a, double* out_b);

#ifdef __cplusplus
}
#endif
#endif /* ASYNCFLOW_B200_H */
