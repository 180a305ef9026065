// af_lane.cuh -- the per-replica next-event engine, ONE REPLICA PER THREAD (round 2).
//
// Same path as af_core.cuh (SimPy's Environment.step() loop, reference
// src/asyncflow/runtime/simulation_runner.py:369, driving the AsyncFlow actors), same event
// semantics, same results bit for bit -- a different mapping onto the SM:
//
//   af_core.cuh (round 1)  one replica per WARP: all 32 lanes run the replica's scalar state machine
//                          redundantly: hundreds of warp-instructions per timed event, issue-slot bound,
//                          much of it 32-way-redundant random-number code.
//   this file              one replica per LANE: every warp instruction advances up to 32 replicas.
//                          The loop body is a fixed sequence of PHASES (lifecycle -> gap -> pick -> ticks ->
//                          decode -> node -> steps -> send -> timer) with a warp rendez-vous between them; a
//                          lane skips the phases its event does not need, so the warp pays each phase at most
//                          once per 32 events (the expensive ones -- the edge's variates, the heap sift --
//                          exist at ONE place in the code and are shared by every event kind that needs
//                          them).
//
// Data layout.  A lane's mutable replica state lives in shared memory, ELEMENT-INTERLEAVED across the
// warp: 128-bit element e of lane l at  base128 + (e * 32 + l) * 16  (a pending event = time | key, a request
// record = t0 | id | pack: one LDS.128 each),  64-bit element e at  base64 + (e * 32 + l) * 8,  32-bit word w at
// base32 + (w * 32 + l) * 4.  Whatever index each lane uses, the lanes of a quarter / half / full warp always hit
// different banks: every access is conflict-free (4 / 2 / 1 wavefronts), no matter how far the replicas have
// drifted apart.  Tables whose size depends on load (pending events, request records, the now-queue) are TIERED:
// the first `*_s` entries in shared memory, the rest in a per-lane region of global memory with the same
// interleave (L2-resident; a branch per access, so that the shared side stays an LDS).  The heap and the request
// records share ONE pool of 128-bit elements, heap from the bottom, records from the top, split per replica by the
// replica's own load (pool_events).  The same region holds the
// cold words (waiter FIFOs, mailboxes, drop counters) and the write-only aggregates (the gauges' sums and
// maxima, the send counters: fire-and-forget REDs).  Read-only scenario tables are NOT replicated per replica:
// they are read through the read-only data path (128-bit __ldg) and a swept field is an index into the lane's
// copy of its sweep row.
//
//   code here           reference being replaced
//   ------------------  ---------------------------------------------------------
//   gen_next_gap        samplers/poisson_poisson.py:52-82, gaussian_poisson.py:64-94
//   phase ARRIVAL       runtime/actors/rqs_generator.py:97-119
//   phase SEND          runtime/actors/edge.py:73-107 (dropout, latency, spike)
//   phase DELIVER       edge.py:110-116 (timeout fired: connection closes, Store.put)
//   phase NODE          client.py:43-71, load_balancer.py:60-72 + routing/lb_algorithms.py:10-36,
//                       server.py:303-313 and 88-149 (endpoint pick, RAM first)
//   phase STEPS         server.py:197-276 (lazy CPU lock, IO queue, release, forward)
//   cpu_walk, ram_walk  simpy Container._trigger_get (FIFO, head-of-line blocking)
//   on_spike/on_outage  runtime/events/injection.py:167-226
//   take_ticks, gauge_touch   metrics/collector.py:50-66 (lazily: settled when a gauge changes)
//   complete            client.py:62-69 + metrics/analyzer.py:83-125
//
// Ordering rule: identical to af_core.cuh (DESIGN.md "tie rule"): timed events pop by (time, seq)
// from a 4-ary min-heap; SimPy's zero-delay events are items of the now-queue, each with its own
// seq; the loop runs the smallest seq among {now-queue front, heap events of the current instant};
// an item pushed as the last action of the running item is applied at once when nothing else
// lives at the instant (can_fuse).
//
// The same source compiles for the host with a "warp" of ONE lane (tests/host_twin: the CPU-only
// tests pin this state machine to the oracle bit for bit; not reachable from the product API).
#pragma once
#include "af_rng.cuh"
#include "../../include/asyncflow_b200.h"

#if defined(__CUDA_ARCH__)
#define AFL_DEVICE 1
#else
#define AFL_DEVICE 0
#endif

#if defined(__CUDACC__)
#define AFL_IN __host__ __device__ __forceinline__
#else
#define AFL_IN static inline
#endif

#define AFL_LIKELY(x) __builtin_expect(!!(x), 1)
#define AFL_UNLIKELY(x) __builtin_expect(!!(x), 0)

#if defined(AF_TRACE_HOST) && !AFL_DEVICE
#include <stdio.h>
#define AFL_TRACE(...) fprintf(stderr, __VA_ARGS__)
#else
#define AFL_TRACE(...) ((void)0)
#endif

namespace afl {

#if AFL_DEVICE
constexpr int LANES = 32;
#else
constexpr int LANES = 1;
#endif
constexpr int STRIDE128 = LANES * 16, STRIDE64 = LANES * 8, STRIDE32 = LANES * 4;

constexpr uint32_t NIL = 0xFFFFFFFFu;
constexpr uint64_t INF_BITS = 0x7FF0000000000000ull;

// ---- event payload: kind[29:32) | aux[20:29) | slot[0:20)  (as af_core.cuh) ------------------
enum : uint32_t { K_ARRIVAL = 0, K_DELIVER = 1, K_STEP_END = 2, K_SPIKE = 3, K_OUTAGE = 4 };
constexpr uint32_t SLOT_BITS = 20, AUX_BITS = 9;
constexpr uint32_t SLOT_MASK = (1u << SLOT_BITS) - 1, AUX_MASK = (1u << AUX_BITS) - 1;
AFL_IN uint32_t mk_payload(uint32_t kind, uint32_t aux, uint32_t slot) { return (kind << 29) | (aux << SLOT_BITS) | slot; }

// ---- request record pack: hops[0:8) step[8:16) ep[16:28) core[28] io[29] wait[30] -------------
constexpr uint32_t PK_CORE = 1u << 28, PK_IO = 1u << 29, PK_WAIT = 1u << 30;
AFL_IN uint32_t pk_hops(uint32_t p) { return p & 0xFFu; }
AFL_IN uint32_t pk_step(uint32_t p) { return (p >> 8) & 0xFFu; }
AFL_IN uint32_t pk_ep(uint32_t p) { return (p >> 16) & 0xFFFu; }

// ---- now-queue items (as af_core.cuh) -------------------------------------------------------
enum : uint32_t { I_PUT = 0, I_GOT = 1, I_CLIENT_LOOP = 2, I_RAM_OK = 3, I_CPU_OK = 4, I_CPU_PUT = 5, I_RAM_PUT = 6 };
constexpr uint32_t NODE_CLIENT = 0, NODE_LB = 1, NODE_SERVER0 = 2;
constexpr int32_t NQ_TOTAL = 128;          // pending zero-delay items per replica (power of two)

// ---- read-only scenario tables (global memory, shared by all replicas; 16-byte multiples so that
//      a record is one or a few 128-bit loads).  `c_*` = index into the lane's sweep-row copy, -1 = not swept.
struct alignas(16) EdgeP { double mean, sigma, dropout; uint32_t meta; int16_t c_mean, c_sigma, c_drop, pad; uint32_t pad2[2]; };   // 48 B; meta: dist[0:3) | target_kind[3:5) | target_index[5:)
struct alignas(16) ServerP { int32_t cpu_cores, ram_mb; uint32_t out_edge, ep_begin, n_ep; int32_t c_cores, c_ram, pad; };           // 32 B
struct alignas(16) EndpointP { uint32_t step_begin, n_steps, total_ram; int32_t c_ram; };                                            // 16 B
struct alignas(16) StepP { double dur; uint32_t kind; int32_t c_dur; };                                                              // 16 B
struct alignas(16) SpikeP { double fire, delta; uint32_t edge; int32_t c_delta; uint32_t pad[2]; };                                  // 32 B
struct alignas(16) OutageP { double fire; int32_t lb_edge, down; };                                                                  // 16 B
struct ColP { int32_t field, index, slot, pad; double base; };     // one sweep column: slot = index into the lane's row copy (-1: consumed at start)

// words of a server's mutable record (32-bit region)
enum : int32_t { SV_CPU_FREE = 0, SV_RAM_FREE, SV_READY_Q, SV_IO_Q, SV_RAM_IN_USE, SV_WORDS };
// ... and of its cold record (global tier): the intrusive FIFOs of the RAM / CPU Containers' waiters
enum : int32_t { SQ_RAMQ_HEAD = 0, SQ_RAMQ_TAIL, SQ_CPUQ_HEAD, SQ_CPUQ_TAIL, SQ_RAMQ_NEED, SQ_WORDS };
enum : int32_t { IB_HEAD = 0, IB_TAIL, IB_PENDING, IB_WORDS };

// Everything the kernel needs to know about one launch; built on the host (af_lane_host.h).
struct Cfg {
    int32_t n_edges, n_servers, n_endpoints, n_steps, n_lb_edges, lb_algo;
    int32_t gen_edge, client_edge, n_spike, n_outage;
    int32_t users_dist, window_s, horizon_s;
    uint32_t metrics_mask;
    double users_mean, users_sigma, rate_per_user, sample_period;
    int32_t n_series, n_sweep_cols, n_row;          // n_row: sweep columns kept per lane (looked up during the run)
    int32_t collect_hist, collect_thr, trace_replicas, trace_clock_cap, trace_tick_cap;
    int32_t redo;                                   // 1: replica indices come from redo_list (re-run of flagged replicas)
    // tiered tables: entries in total; the now-queue's entries in shared memory
    int32_t ev_total, rq_total, nq_s;
    // The lane's POOL of `pool` 128-bit elements holds the first ev_s heap entries (element i) and the first rq_s request
    // records (slot s at element pool - 1 - s), ev_s + rq_s = pool, split per replica by pool_events() from the
    // replica's pending-events estimate row_need[replica - need_first] when the launch has one for the replica; the
    // others take ev_s / rq_s (make_cfg: the split of the scenario's estimate).  ev_lo: the fewest heap entries a
    // replica gets, rq_floor: the fewest records when the events take more.
    int32_t pool, ev_lo, rq_floor, ev_s, rq_s;
    // shared-memory layout of a warp: 128-bit region (the pool), 64-bit region, 32-bit region
    int32_t n128;
    int32_t o64_nq, o64_spike, o64_row, n64;
    int32_t o32_conn, o32_srv, o32_lb, o32_dirty, n_dirty, n32;
    int32_t warp_bytes;                             // n128 * 512 + n64 * 256 + n32 * 128
    // global tier of a warp (same interleave).  Heap entry idx >= ev_s at element idx - ev_s of the 128-bit region,
    // record slot s >= rq_s at element gi_rq + s (= ev_total - ev_s + (s - rq_s): right after the replica's heap entries);
    // gi_* = (offset of the table in its region) - (entries kept in shared memory)
    int32_t gi_rq, gn128;
    int32_t gi_nq, gi_acc, gn64;                    // gi_acc: the gauges' accumulators (write-only during the run: RED)
    int32_t g32_cold, gi_smax, gi_sent, gn32;       // words [0, rq_total): every record's `next` link; then the cold words,
                                                    // the gauges' maxima, the per-edge send counters (RED too)
    int32_t c_srvq, c_inbox, c_drop;                // cold words (offsets from g32_cold): waiter FIFOs, mailboxes, drop counters
    uint64_t gwarp_bytes;                           // gn128 * 512 + gn64 * 256 + gn32 * 128
    // device pointers
    const EdgeP* edges; const ServerP* servers; const EndpointP* endpoints; const StepP* steps;
    const SpikeP* spikes; const OutageP* outages; const int32_t* lb_edges; const ColP* cols;
    const double* sweep_vals; uint64_t sweep_first, sweep_rows;
    const int32_t* row_need; uint64_t need_first, need_rows;   // per-replica pending-events estimates (nullptr: ev_s / rq_s for all)
    unsigned char* gtier;                          // global tiers, one region per resident warp
    AfReplicaStats* stats; uint32_t* edge_sent; uint32_t* edge_dropped;
    uint32_t* hist; uint32_t* thr; uint64_t* samp_sum; uint32_t* samp_max;
    double* trace_clocks; uint32_t* trace_series; uint32_t* trace_counts;
    unsigned long long* work_counter;
    const uint32_t* order;                          // the k-th replica a lane pulls is local index order[k] (af_run)
    const uint32_t* redo_list; const uint32_t* redo_count;
    uint64_t seed, replica_begin, n_replicas;
    // per-tick bands (run_lane<true> only; DESIGN.md §3.4).  Group g's difference rows start at band_rows + g * band_group_words:
    // row 0 counts replicas, rows 1 + j the sum of series j, rows 1 + n_series + j its square; band_stride words per row
    // (ticks, plus one at index n_ticks for changes after the last tick).  A replica without a group entry adds to group
    // band_groups, which is never fetched.
    uint64_t* band_rows; const uint32_t* band_group; uint32_t* band_from;
    uint64_t band_first, band_n, band_group_words;
    int32_t band_groups, band_stride;
    // per-window latency bands (run_lane<*, true> only; DESIGN.md §3.5), over the groups of band_group: window k of
    // group g is the LAT_ROW words at lat_rows + (g * lat_windows + k) * LAT_ROW.  lat_from[local] = the completions a
    // stopped replica added (the warp-per-replica pass adds the rest).
    uint64_t* lat_rows; uint32_t* lat_from;
    int32_t lat_window, lat_windows;
    // per-tick distribution bands (run_lane<*, *, *, true> only; DESIGN.md §3.7), over the groups of band_group: the
    // count of bin b of selected series s at tick row k of group g is the u32 at dist_rows + g * dist_group_words +
    // s * dist_series_words + k * dist_bins + b (difference rows over k until af_dist_scan_kernel).  dist_slot[j] = s
    // for a selected series j, -1 for the others.  band_from is shared with the per-tick bands.
    uint32_t* dist_rows; const int32_t* dist_slot;
    uint64_t dist_group_words, dist_series_words;
    int32_t dist_n, dist_bins;
    // occupancy integrals (run_lane<*, *, *, *, true> only; DESIGN.md §3.8): occ_cols u64 accumulators per replica at
    // elements gi_occ + col of the 64-bit global tier (RED during the run), written to occ[local * occ_cols + col] at
    // write-back; occ_scale = 2^f (afr::occ_fixed)
    uint64_t* occ; double occ_scale;
    int32_t gi_occ, occ_cols;
};


#if defined(__CUDACC__)
__constant__ Cfg c_cfg;
#endif
#if AFL_DEVICE
#define AFL_C c_cfg
#else
static Cfg h_cfg;
#define AFL_C h_cfg
#endif

// ---- read-only loads ----------------------------------------------------------------------------
template <class T> AFL_IN T ro(const T* p) {
#if AFL_DEVICE
    static_assert(sizeof(T) % 16 == 0, "16-byte records");
    T v;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&v);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); ++i) d[i] = __ldg(s + i);
    return v;
#else
    return *p;
#endif
}

// ---- the lane's memory ------------------------------------------------------------------------------
// Shared memory is addressed by absolute 32-bit shared-window addresses through ld.shared / st.shared (one LDS /
// STS, 32-bit address arithmetic).  Going through a pointer into an `extern __shared__` array costs four extra
// instructions per access (S2R SR_CgaCtaId + MOV + LEA + IADD rebuild the window base every time), a generic pointer
// costs 64-bit arithmetic.  A tiered table takes a
// BRANCH on "is it in shared memory", not a select.  All shared accesses are volatile asm: they keep program order.
struct Mem {
    uint32_t s128, s64, s32;                    // shared-memory regions of the warp (window addresses, the lane's column)
    unsigned char* g128; unsigned char* g64; unsigned char* g32;     // global tier of the warp, already offset by the lane
};
#if AFL_DEVICE
AFL_IN uint32_t sm_ld32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
AFL_IN void sm_st32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v)); }
AFL_IN uint64_t sm_ld64(uint32_t a) { uint64_t v; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a)); return v; }
AFL_IN void sm_st64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" :: "r"(a), "l"(v)); }
AFL_IN void sm_ld128(uint32_t a, uint64_t& x, uint64_t& y) { asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "r"(a)); }
AFL_IN void sm_st128(uint32_t a, uint64_t x, uint64_t y) { asm volatile("st.shared.v2.u64 [%0], {%1, %2};" :: "r"(a), "l"(x), "l"(y)); }
AFL_IN void gl_ld128(const unsigned char* p, uint64_t& x, uint64_t& y) { const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p); x = v.x; y = v.y; }
AFL_IN void gl_st128(unsigned char* p, uint64_t x, uint64_t y) { *reinterpret_cast<ulonglong2*>(p) = make_ulonglong2(x, y); }
#else
static unsigned char* afl_smem_host = nullptr;     // the twin's stand-in for the SM's shared memory
AFL_IN uint32_t sm_ld32(uint32_t a) { uint32_t v; memcpy(&v, afl_smem_host + a, 4); return v; }
AFL_IN void sm_st32(uint32_t a, uint32_t v) { memcpy(afl_smem_host + a, &v, 4); }
AFL_IN uint64_t sm_ld64(uint32_t a) { uint64_t v; memcpy(&v, afl_smem_host + a, 8); return v; }
AFL_IN void sm_st64(uint32_t a, uint64_t v) { memcpy(afl_smem_host + a, &v, 8); }
AFL_IN void sm_ld128(uint32_t a, uint64_t& x, uint64_t& y) { memcpy(&x, afl_smem_host + a, 8); memcpy(&y, afl_smem_host + a + 8, 8); }
AFL_IN void sm_st128(uint32_t a, uint64_t x, uint64_t y) { memcpy(afl_smem_host + a, &x, 8); memcpy(afl_smem_host + a + 8, &y, 8); }
AFL_IN void gl_ld128(const unsigned char* p, uint64_t& x, uint64_t& y) { memcpy(&x, p, 8); memcpy(&y, p + 8, 8); }
AFL_IN void gl_st128(unsigned char* p, uint64_t x, uint64_t y) { memcpy(p, &x, 8); memcpy(p + 8, &y, 8); }
#endif
AFL_IN uint32_t a128(const Mem& m, int32_t elem) { return m.s128 + (uint32_t)elem * (uint32_t)STRIDE128; }
AFL_IN uint32_t a64(const Mem& m, int32_t elem) { return m.s64 + (uint32_t)elem * (uint32_t)STRIDE64; }
AFL_IN uint32_t a32(const Mem& m, int32_t word) { return m.s32 + (uint32_t)word * (uint32_t)STRIDE32; }
// global tier: ONE 32-bit element index (table offset folded in on the host), one widening multiply-add onto the
// lane's region pointer
AFL_IN unsigned char* g128p(const Mem& m, int32_t elem) { return m.g128 + (uint64_t)(uint32_t)elem * (uint32_t)STRIDE128; }
AFL_IN uint64_t* g64p(const Mem& m, int32_t elem) { return reinterpret_cast<uint64_t*>(m.g64 + (uint64_t)(uint32_t)elem * (uint32_t)STRIDE64); }
AFL_IN uint32_t* g32p(const Mem& m, int32_t word) { return reinterpret_cast<uint32_t*>(m.g32 + (uint64_t)(uint32_t)word * (uint32_t)STRIDE32); }
// fixed tables in shared memory: connection counts, server levels, LB order, sweep-row copy, spike offsets
AFL_IN uint64_t e64_ld(const Mem& m, int32_t elem) { return sm_ld64(a64(m, elem)); }
AFL_IN void e64_st(const Mem& m, int32_t elem, uint64_t v) { sm_st64(a64(m, elem), v); }
AFL_IN double f64_ld(const Mem& m, int32_t elem) { return afr::u2d(e64_ld(m, elem)); }
AFL_IN void f64_st(const Mem& m, int32_t elem, double v) { e64_st(m, elem, afr::d2u(v)); }
AFL_IN uint32_t w32_ld(const Mem& m, int32_t word) { return sm_ld32(a32(m, word)); }
AFL_IN void w32_st(const Mem& m, int32_t word, uint32_t v) { sm_st32(a32(m, word), v); }
AFL_IN int32_t i32_ld(const Mem& m, int32_t word) { return (int32_t)w32_ld(m, word); }
AFL_IN void i32_st(const Mem& m, int32_t word, int32_t v) { w32_st(m, word, (uint32_t)v); }
// cold words (global tier only): queue links of the Stores and Containers, drop counters -- touched at ties, under
// contention, on a dropped request
AFL_IN uint32_t c32_ld(const Mem& m, int32_t word) { return *g32p(m, AFL_C.g32_cold + word); }
AFL_IN void c32_st(const Mem& m, int32_t word, uint32_t v) { *g32p(m, AFL_C.g32_cold + word) = v; }
// tiered tables: entry idx < split in shared memory (element os + idx), the rest in the global tier (element gi + idx)
AFL_IN void ld_t128(const Mem& m, int32_t os, int32_t gi, int32_t idx, int32_t split, uint64_t& x, uint64_t& y) {
    if (AFL_LIKELY(idx < split)) sm_ld128(a128(m, os + idx), x, y); else gl_ld128(g128p(m, gi + idx), x, y);
}
AFL_IN void st_t128(const Mem& m, int32_t os, int32_t gi, int32_t idx, int32_t split, uint64_t x, uint64_t y) {
    if (AFL_LIKELY(idx < split)) sm_st128(a128(m, os + idx), x, y); else gl_st128(g128p(m, gi + idx), x, y);
}
AFL_IN uint64_t ld_t64(const Mem& m, int32_t os, int32_t gi, int32_t idx, int32_t split) {
    if (AFL_LIKELY(idx < split)) return sm_ld64(a64(m, os + idx));
    return *g64p(m, gi + idx);
}
AFL_IN void st_t64(const Mem& m, int32_t os, int32_t gi, int32_t idx, int32_t split, uint64_t v) {
    if (AFL_LIKELY(idx < split)) sm_st64(a64(m, os + idx), v); else *g64p(m, gi + idx) = v;
}

// the replica's scalar state: registers (nothing here is indexed dynamically)
struct St {
    uint64_t replica, local;
    double now, horizon;
    uint32_t seq; int32_t ev_n; uint32_t peak_ev;
    uint64_t arr_t; uint32_t arr_seq, arr_on;   // the generator's pending timeout: always exactly one, kept out of the heap
    uint32_t nq_head, nq_tail, busy;            // busy = 2 * (items in the now-queue) + (the heap may hold an event of this instant)
    int32_t ev_s, rq_s;                         // this replica's split of the pool: heap entries / record slots in shared memory
    uint32_t rq_mask;                           // free record slots in shared memory (bit s: slot s < rq_s)
    uint32_t rq_free_hi, rq_hw, rq_live, peak_rq;   // slots in the global tier: free list, high-water mark (from rq_s)
    uint32_t n_waiting;                         // requests parked in a RAM / CPU waiter FIFO (0: every such FIFO is empty, no need to look)
    double g_vnow, g_wend, g_lam;               // generator: the sampler's virtual clock (the simulation's is `now`)
    uint32_t g_pos, generated, g_done, need_arrival, arm_seq;
    double gap0, gap1; uint32_t gap_cnt;        // inter-arrival gaps drawn ahead (see the SEND phase)
    double users_mean, users_sigma, rate_per_user;
    int32_t lb_n, spike_cur, outage_cur;
    uint32_t tick_seq, n_ticks; double tick_time;
    uint32_t completed, flags, traced;
    uint64_t n_events;
    double lat_sum, lat_sumsq, lat_min, lat_max;
    uint64_t* band;                             // run_lane<true, *>: the replica's group's difference rows
    uint32_t dist_g;                            // run_lane<*, *, *, true>: the replica's group (distribution bands)
};

// flags that end a replica early (its partial results are written back with the flag set)
constexpr uint32_t STOP_FLAGS = AF_FLAG_EVENT_OVERFLOW | AF_FLAG_REQUEST_OVERFLOW | AF_FLAG_NOWQ_OVERFLOW | AF_FLAG_LB_EMPTY;

// ---- swept parameters ----------------------------------------------------------------------------
AFL_IN double row_val(const Mem& m, int32_t c) { return f64_ld(m, AFL_C.o64_row + c); }
// the generator's parameters a sweep column over `field` sets to `v` when a replica starts; false: not one of them.
// (start_replica, and af_engine.cu's prediction of a replica's work, which must see the same users and rate)
AFL_IN bool gen_field(int32_t field, double v, double& users_mean, double& users_sigma, double& rate_per_user) {
    switch (field) {
    case AF_FIELD_USERS_MEAN: users_mean = v; return true;
    case AF_FIELD_USERS_SIGMA: users_sigma = v; return true;
    case AF_FIELD_RATE_PER_USER: rate_per_user = v; return true;
    default: return false;
    }
}
AFL_IN uint32_t ep_total_ram(const Mem& m, uint32_t ep) {
    const EndpointP p = ro(AFL_C.endpoints + ep);
    return p.c_ram >= 0 ? (uint32_t)row_val(m, p.c_ram) : p.total_ram;
}

// ---- the pool split (af_lane_host.h reports it for the launch's heaviest replica) -------------------------------
// Shared-memory record slots are handed out from a 32-bit mask: at most RQ_BITS of them.
constexpr int32_t RQ_BITS = 32;
// Heap entries a replica with an estimated `need` pending events keeps in shared memory: its need, but no more than
// leaves `rq_floor` record slots and no fewer than `ev_lo` (a heap entry is touched ~20 times per event, a record
// twice: byte for byte the heap is worth more); the records take the rest, at most RQ_BITS and rq_total of them, so
// the heap takes whatever the records cannot.  make_cfg caps the pool at ev_total + min(rq_total, RQ_BITS): the
// records always get exactly pool - ev_s slots.
AFL_IN int32_t pool_events(int32_t pool, int32_t ev_lo, int32_t rq_floor, int32_t ev_total, int32_t rq_total, int32_t need) {
    int32_t ev = need < pool - rq_floor ? need : pool - rq_floor;
    if (ev < ev_lo) ev = ev_lo;
    const int32_t rq_cap = rq_total < RQ_BITS ? rq_total : RQ_BITS;
    if (ev < pool - rq_cap) ev = pool - rq_cap;
    return ev < ev_total ? ev : ev_total;
}
#if AFL_DEVICE
AFL_IN uint32_t lowest_bit(uint32_t x) { return (uint32_t)__ffs((int)x) - 1u; }
#else
AFL_IN uint32_t lowest_bit(uint32_t x) { return (uint32_t)__builtin_ctz(x); }
#endif

// ---- request records (tiered): one 128-bit element  t0 | id : pack.  Slot s < rq_s is element pool - 1 - s of the
//      lane's pool (one LDS.128), the others live in the global tier.  The `next` links (free list of the global slots,
//      waiter FIFOs) are 32-bit words of the global tier for every slot ------------------------------------------------
// (Tried in round 2 and dropped: a third tier of 256-record PAGES from a pool shared by all lanes, so that saturated
//  replicas -- 10^4..10^5 requests parked in a RAM queue -- stay on this engine.  Bit-exact, but the extra tier in every
//  record access grew the loop's instruction footprint and slowed the bench workload, and C2 (10^4 replicas) was still
//  faster one replica per warp.)
AFL_IN uint32_t rq_sm(const Mem& m, uint32_t s) { return a128(m, AFL_C.pool - 1 - (int32_t)s); }
AFL_IN unsigned char* rq_gl(const Mem& m, uint32_t s) { return g128p(m, AFL_C.gi_rq + (int32_t)s); }
AFL_IN void rq_load(const St& W, const Mem& m, uint32_t s, double& t0, uint32_t& rid, uint32_t& pack) {
    uint64_t a, b;
    if (AFL_LIKELY((int32_t)s < W.rq_s)) sm_ld128(rq_sm(m, s), a, b); else gl_ld128(rq_gl(m, s), a, b);
    t0 = afr::u2d(a); rid = (uint32_t)b; pack = (uint32_t)(b >> 32);
}
AFL_IN void rq_store(const St& W, const Mem& m, uint32_t s, double t0, uint32_t rid, uint32_t pack) {
    const uint64_t a = afr::d2u(t0), b = (uint64_t)rid | ((uint64_t)pack << 32);
    if (AFL_LIKELY((int32_t)s < W.rq_s)) sm_st128(rq_sm(m, s), a, b); else gl_st128(rq_gl(m, s), a, b);
}
AFL_IN uint32_t rq_pack(const St& W, const Mem& m, uint32_t s) {
    if (AFL_LIKELY((int32_t)s < W.rq_s)) return sm_ld32(rq_sm(m, s) + 12u);
    return *reinterpret_cast<const uint32_t*>(rq_gl(m, s) + 12);
}
AFL_IN void rq_pack_set(const St& W, const Mem& m, uint32_t s, uint32_t v) {
    if (AFL_LIKELY((int32_t)s < W.rq_s)) sm_st32(rq_sm(m, s) + 12u, v);
    else *reinterpret_cast<uint32_t*>(rq_gl(m, s) + 12) = v;
}
AFL_IN uint32_t rq_next(const Mem& m, uint32_t s) { return *g32p(m, (int32_t)s); }
AFL_IN void rq_next_set(const Mem& m, uint32_t s, uint32_t v) { *g32p(m, (int32_t)s) = v; }

#if AFL_DEVICE
// fire-and-forget reductions (RED.E.ADD / RED.E.MAX: no result, no scoreboard wait) and the loads that read them back
__device__ __forceinline__ void red_add64(uint64_t* p, uint64_t v) { atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); }
__device__ __forceinline__ void red_add32(uint32_t* p, uint32_t v) { atomicAdd(p, v); }
__device__ __forceinline__ void red_max32(uint32_t* p, uint32_t v) { atomicMax(p, v); }
__device__ __forceinline__ uint64_t ld_cg64(const uint64_t* p) { return (uint64_t)__ldcg(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ uint32_t ld_cg32(const uint32_t* p) { return __ldcg(p); }
#else
static inline void red_add64(uint64_t* p, uint64_t v) { *p += v; }
static inline void red_add32(uint32_t* p, uint32_t v) { *p += v; }
static inline void red_max32(uint32_t* p, uint32_t v) { if (v > *p) *p = v; }
static inline uint64_t ld_cg64(const uint64_t* p) { return *p; }
static inline uint32_t ld_cg32(const uint32_t* p) { return *p; }
#endif
// A request takes the LOWEST tier that has a free slot: with one LIFO list the few requests in flight after a burst
// keep cycling through whatever slots were freed last -- often global-tier ones (C1 with 10 shared-memory slots for
// ~3 requests in flight: -9 %).  Shared-memory slots are handed out first (the lowest free bit of the mask), global
// ones after (free list, then fresh ones).
AFL_IN uint32_t rq_alloc(St& W, const Mem& m) {
    uint32_t s;
    if (W.rq_mask != 0u) { s = lowest_bit(W.rq_mask); W.rq_mask &= W.rq_mask - 1u; }
    else if (W.rq_free_hi != NIL) { s = W.rq_free_hi; W.rq_free_hi = rq_next(m, s); }
    else if ((int32_t)W.rq_hw < AFL_C.rq_total) { s = W.rq_hw++; }
    else { W.flags |= AF_FLAG_REQUEST_OVERFLOW; return NIL; }
    const uint32_t live = ++W.rq_live;
    if (live > W.peak_rq) W.peak_rq = live;
    return s;
}
AFL_IN void rq_release(St& W, const Mem& m, uint32_t s) {
    if ((int32_t)s < W.rq_s) W.rq_mask |= 1u << s;
    else { rq_next_set(m, s, W.rq_free_hi); W.rq_free_hi = s; }
    --W.rq_live;
}

// intrusive FIFOs through the `next` links; head / tail are COLD words.  Out of line (Mem by value: a reference across a
// call would force it into local memory): nine call sites, all on paths taken at ties or under contention
#if defined(__CUDACC__)
#define AFL_COLD __host__ __device__ __noinline__
#else
#define AFL_COLD static __attribute__((noinline))
#endif
AFL_COLD void fifo_push(const Mem m, int32_t w_head, int32_t w_tail, uint32_t s) {
    rq_next_set(m, s, NIL);
    const uint32_t tail = c32_ld(m, w_tail);
    if (tail == NIL) c32_st(m, w_head, s); else rq_next_set(m, tail, s);
    c32_st(m, w_tail, s);
}
AFL_COLD uint32_t fifo_pop(const Mem m, int32_t w_head, int32_t w_tail) {
    const uint32_t s = c32_ld(m, w_head);
    const uint32_t h = rq_next(m, s);
    c32_st(m, w_head, h);
    if (h == NIL) c32_st(m, w_tail, NIL);
    return s;
}

// ---- pending timed events: 4-ary min-heap on (time bits, seq), tiered; one 128-bit element per event: entry i < ev_s
//      is element i of the pool.  The root is always in shared memory (pool_events: ev_s >= ev_lo >= 1): the loop reads
//      it with a plain LDS ---------------------------------------------------------------------------------------------
AFL_IN void ev_get(const St& W, const Mem& m, int32_t i, uint64_t& t, uint64_t& k) { ld_t128(m, 0, -W.ev_s, i, W.ev_s, t, k); }
AFL_IN void ev_set(const St& W, const Mem& m, int32_t i, uint64_t t, uint64_t k) { st_t128(m, 0, -W.ev_s, i, W.ev_s, t, k); }
AFL_IN bool ev_less(uint64_t ta, uint64_t ka, uint64_t tb, uint64_t kb) {       // times are non-negative doubles: bit order = value order
    return ta < tb || (ta == tb && (uint32_t)(ka >> 32) < (uint32_t)(kb >> 32));
}
AFL_IN void heap_push(St& W, const Mem& m, uint64_t tb, uint64_t key) {
    int32_t i = W.ev_n;
    const int32_t pending = i + (int32_t)W.arr_on;     // the generator's timeout counts as a pending event
    if (AFL_UNLIKELY(pending >= AFL_C.ev_total)) { W.flags |= AF_FLAG_EVENT_OVERFLOW; return; }
    W.ev_n = i + 1;
    if ((uint32_t)(pending + 1) > W.peak_ev) W.peak_ev = (uint32_t)(pending + 1);
#pragma unroll 1
    while (i > 0) {
        const int32_t p = (i - 1) >> 2;
        uint64_t tp, kp;
        ev_get(W, m, p, tp, kp);
        if (!ev_less(tb, key, tp, kp)) break;
        ev_set(W, m, i, tp, kp);
        i = p;
    }
    ev_set(W, m, i, tb, key);
}
// remove the root (the caller has read it)
// One sift-down level = the four children fetched TOGETHER (indices past the end clamped onto the last child: a
// duplicate never wins a strict comparison), one tier test for the group instead of one per child, the minimum picked
// with selects.  The lanes of a warp sit at different depths with different child counts; this way a level costs every
// lane the same straight-line code and its four loads are in flight at once.
AFL_IN void heap_pop(St& W, const Mem& m) {
    const int32_t n = --W.ev_n;
    if (n == 0) return;
    uint64_t tl, kl;
    ev_get(W, m, n, tl, kl);
    const int32_t last = n - 1;
    int32_t i = 0;
#pragma unroll 1
    for (;;) {
        const int32_t c = 4 * i + 1;
        if (c >= n) break;
        const int32_t c1 = c + 1 < last ? c + 1 : last, c3 = c + 3 < last ? c + 3 : last;
        int32_t c2 = c + 2 < last ? c + 2 : last;
        uint64_t t0, k0, t1, k1, t2, k2, t3, k3;
        if (AFL_LIKELY(c3 < W.ev_s)) {
            sm_ld128(a128(m, c), t0, k0); sm_ld128(a128(m, c1), t1, k1);
            sm_ld128(a128(m, c2), t2, k2); sm_ld128(a128(m, c3), t3, k3);
        } else {
            ev_get(W, m, c, t0, k0); ev_get(W, m, c1, t1, k1); ev_get(W, m, c2, t2, k2); ev_get(W, m, c3, t3, k3);
        }
        int32_t b = c;
        if (ev_less(t1, k1, t0, k0)) { t0 = t1; k0 = k1; b = c1; }
        if (ev_less(t3, k3, t2, k2)) { t2 = t3; k2 = k3; c2 = c3; }
        if (ev_less(t2, k2, t0, k0)) { t0 = t2; k0 = k2; b = c2; }
        if (!ev_less(t0, k0, tl, kl)) break;
        ev_set(W, m, i, t0, k0);
        i = b;
    }
    ev_set(W, m, i, tl, kl);
}

// ---- now-queue (tiered ring of NQ_TOTAL items: seq << 32 | kind:3 aux:9 slot:20) ---------------------
AFL_IN uint64_t nq_ld(const Mem& m, uint32_t pos) {
    return ld_t64(m, AFL_C.o64_nq, AFL_C.gi_nq, (int32_t)(pos & (uint32_t)(NQ_TOTAL - 1)), AFL_C.nq_s);
}
AFL_IN bool can_fuse(const St& W) { return AFL_LIKELY(W.busy == 0); }
AFL_IN void nq_push(St& W, const Mem& m, uint32_t kind, uint32_t aux, uint32_t slot) {
    const uint32_t tail = W.nq_tail;
    if (tail - W.nq_head >= (uint32_t)NQ_TOTAL) { W.flags |= AF_FLAG_NOWQ_OVERFLOW; return; }
    st_t64(m, AFL_C.o64_nq, AFL_C.gi_nq, (int32_t)(tail & (uint32_t)(NQ_TOTAL - 1)), AFL_C.nq_s,
           ((uint64_t)(W.seq++) << 32) | mk_payload(kind, aux, slot));
    W.nq_tail = tail + 1;
    W.busy += 2u;
}
AFL_IN uint32_t nq_take(St& W, const Mem& m) {      // (the caller has adjusted `busy`)
    const uint32_t item = (uint32_t)nq_ld(m, W.nq_head);
    W.nq_head += 1;
    if (W.nq_head == W.nq_tail) { W.nq_head = 0; W.nq_tail = 0; }   // empty: restart at the shared-memory end of the ring
    return item;
}

// ---- generator: samplers/poisson_poisson.py:52-82 / gaussian_poisson.py:64-94 -------------------------------
AFL_IN bool gen_next_gap(St& W, double& gap) {
    const double T = W.horizon;
    double vnow = W.g_vnow, wend = W.g_wend, lam = W.g_lam;
    uint32_t pos = W.g_pos;
    bool ok = false;
#pragma unroll 1
    for (;;) {
        if (!(vnow < T)) break;
        if (vnow >= wend) {
            wend = vnow + (double)AFL_C.window_s;
            afr::GenDraw d = afr::gen_users(AFL_C.seed, W.replica, pos, AFL_C.users_dist, W.users_mean, W.users_sigma);
            pos = d.pos;
            lam = d.value * W.rate_per_user;
        }
        if (lam <= 0.0) { vnow = wend; continue; }
        afr::Src s = afr::make_gen(AFL_C.seed, W.replica, pos);
        double u = s.next53();
        pos = s.pos;
        if (u < 1e-15) u = 1e-15;                   // max(u, 1e-15)
        const double dt = afr::af_div(-afr::af_log(1.0 - u), lam);
        if (vnow + dt > T) break;
        if (vnow + dt >= wend) { vnow = wend; continue; }
        vnow += dt;
        gap = dt;
        ok = true;
        break;
    }
    W.g_vnow = vnow; W.g_wend = wend; W.g_lam = lam; W.g_pos = pos;
    return ok;
}

// ---- sampled metrics (metrics/collector.py:50-66), LAZILY --------------------------------------------------------
// The collector reads every gauge at every tick.  Done literally, that loop (n_series loads, 64-bit adds, maxima) runs
// in every iteration of the warp -- with 32 replicas in a warp some lane always has a tick due.  A gauge only changes
// inside an event, so the tick loop here just counts ticks, and the per-series aggregates are settled when a gauge
// CHANGES:  sum over ticks of v  =  n_ticks * v_final - sum over changes of (delta * ticks taken before the change)
// (u64 modular arithmetic: exact), and the maximum over ticks takes the OLD value at a change iff a tick has seen it
// (one "changed since the last tick" bit per series, cleared by a tick).  Traced replicas also store every reading.
// The accumulator and the maximum are only ever ADDED to / MAXED during the run and read at write-back: they live in
// the lane's global tier and are updated with fire-and-forget reductions (no load, no wait, no shared memory: 12 B
// per series -- on a 32-node topology 1.8 KB per lane, the difference between 2 and 6 warps per SM).
//
// Per-tick bands (kBands) ride on the same moment: a change from v to v + delta with n_ticks ticks taken before it adds
// delta to the series at every tick k >= n_ticks, so the sums over a group's replicas are difference arrays -- one RED
// of delta (and of (v + delta)^2 - v^2) at index n_ticks per change, one prefix scan after the launch (DESIGN.md §3.4).
// Distribution bands (kDist) too, over (tick, value bin): from tick n_ticks on the replica leaves bin(v) for
// bin(v + delta) -- one RED of -1 and one of +1 at row n_ticks of a selected series, none when the bin stays (§3.7).
// The replica's group is W.dist_g (a u32 register; a local of run_lane's would move the SASS of the kernels without).
AFL_IN uint32_t* dist_row(uint32_t dg, int32_t s, uint32_t k) {
    return AFL_C.dist_rows + (uint64_t)dg * AFL_C.dist_group_words + (uint64_t)(uint32_t)s * AFL_C.dist_series_words
           + (uint64_t)k * (uint32_t)AFL_C.dist_bins;
}
AFL_IN uint32_t dist_bin(uint32_t v) {              // (values above the launch's gauge bound cannot occur: clamped anyway)
    const uint32_t b = afr::gauge_bin(v), last = (uint32_t)AFL_C.dist_bins - 1u;
    return b < last ? b : last;
}
AFL_IN int32_t dist_slot(int32_t j) {
#if AFL_DEVICE
    return __ldg(AFL_C.dist_slot + j);
#else
    return AFL_C.dist_slot[j];
#endif
}
template <bool kBands, bool kDist>
AFL_IN void gauge_touch(const St& W, const Mem& m, int32_t j, uint32_t v_old, int32_t delta) {
    red_add64(g64p(m, AFL_C.gi_acc + j), (uint64_t)(int64_t)delta * (uint64_t)W.n_ticks);
    if constexpr (kBands) {
        const uint64_t v1 = (uint64_t)(v_old + (uint32_t)delta), v0 = (uint64_t)v_old;
        uint64_t* row = W.band + (uint64_t)(1 + j) * (uint64_t)AFL_C.band_stride + W.n_ticks;
        red_add64(row, (uint64_t)(int64_t)delta);
        red_add64(row + (uint64_t)AFL_C.n_series * (uint64_t)AFL_C.band_stride, v1 * v1 - v0 * v0);
    }
    if constexpr (kDist) {
        const int32_t s = dist_slot(j);
        if (s >= 0) {
            const uint32_t b0 = dist_bin(v_old), b1 = dist_bin(v_old + (uint32_t)delta);
            if (b0 != b1) {
                uint32_t* row = dist_row(W.dist_g, s, W.n_ticks);
                red_add32(row + b0, ~0u);
                red_add32(row + b1, 1u);
            }
        }
    }
    const int32_t dw = AFL_C.o32_dirty + (j >> 5);
    const uint32_t d = w32_ld(m, dw), bit = 1u << (j & 31);
    if (!(d & bit)) {
        red_max32(g32p(m, AFL_C.gi_smax + j), v_old);
        w32_st(m, dw, d | bit);
    }
}
// Occupancy integrals (kOcc; DESIGN.md §3.8): a count of requests in some state that changes by delta at W.now adds
// delta * fixed(H - now) to its column, whatever the metrics mask samples -- the integral of the count over [0, H)
// (u64 modular arithmetic: exact in any order, the sum below 2^64 by the choice of f).  Columns 5 s + OC_* of server s,
// 5 n_servers + e of edge e.
enum : int32_t { OC_RAM_WAIT = 0, OC_CPU_WAIT, OC_CPU, OC_IO, OC_RAM_MB, OC_WORDS };
template <bool kOcc>
AFL_IN void occ_add(const St& W, const Mem& m, int32_t col, int32_t delta) {
    if constexpr (kOcc) red_add64(g64p(m, AFL_C.gi_occ + col), (uint64_t)(int64_t)delta * afr::occ_fixed(W.horizon - W.now, AFL_C.occ_scale));
}
AFL_IN int32_t occ_col(uint32_t sidx, int32_t state) { return OC_WORDS * (int32_t)sidx + state; }
template <bool kBands, bool kDist, bool kOcc>
AFL_IN void conn_add(const St& W, const Mem& m, uint32_t edge, int32_t delta) {
    const int32_t pw = AFL_C.o32_conn + (int32_t)edge;
    const uint32_t v = w32_ld(m, pw);
    if (AFL_C.metrics_mask & AF_METRIC_EDGE_CONN) gauge_touch<kBands, kDist>(W, m, 3 * AFL_C.n_servers + (int32_t)edge, v, delta);
    occ_add<kOcc>(W, m, OC_WORDS * AFL_C.n_servers + (int32_t)edge, delta);
    w32_st(m, pw, v + (uint32_t)delta);
}
AFL_IN int32_t ib_word(uint32_t node, int32_t f) { return AFL_C.c_inbox + (int32_t)node * IB_WORDS + f; }      // cold
AFL_IN int32_t sq_word(uint32_t sidx, int32_t f) { return AFL_C.c_srvq + (int32_t)sidx * SQ_WORDS + f; }       // cold
AFL_IN int32_t sv_word(uint32_t sidx, int32_t f) { return AFL_C.o32_srv + (int32_t)sidx * SV_WORDS + f; }
// field = SV_READY_Q / SV_IO_Q / SV_RAM_IN_USE (series 3 * sidx + 0 / 1 / 2)
template <bool kBands, bool kDist, bool kOcc>
AFL_IN void srv_gauge_add(const St& W, const Mem& m, uint32_t sidx, int32_t field, int32_t delta) {
    const int32_t pw = sv_word(sidx, field);
    const int32_t v = i32_ld(m, pw);
    if ((AFL_C.metrics_mask & 7u) == 7u) gauge_touch<kBands, kDist>(W, m, 3 * (int32_t)sidx + (field - SV_READY_Q), (uint32_t)v, delta);
    occ_add<kOcc>(W, m, occ_col(sidx, field == SV_READY_Q ? OC_CPU_WAIT : (field == SV_IO_Q ? OC_IO : OC_RAM_MB)), delta);
    i32_st(m, pw, v + delta);
}
AFL_IN uint32_t gauge_value(const Mem& m, int32_t j) {
    const int32_t ns3 = 3 * AFL_C.n_servers;
    if (j < ns3) { const int32_t mt = j % 3; return w32_ld(m, sv_word((uint32_t)(j / 3), mt == 0 ? SV_READY_Q : (mt == 1 ? SV_IO_Q : SV_RAM_IN_USE))); }
    return w32_ld(m, AFL_C.o32_conn + (j - ns3));
}
AFL_IN bool gauge_on(int32_t j) {
    return j < 3 * AFL_C.n_servers ? (AFL_C.metrics_mask & 7u) == 7u          // collector.py:60-63
                                   : (AFL_C.metrics_mask & AF_METRIC_EDGE_CONN) != 0;
}
// every collector tick ordered before (t, ev_seq)
template <bool kLean>
AFL_IN void take_ticks(St& W, const Mem& m, double t, uint32_t ev_seq) {
    double tick = W.tick_time;
    uint32_t tseq = W.tick_seq, nt = W.n_ticks, seq = W.seq;
    const double horizon = W.horizon;
#pragma unroll 1
    while ((tick < t || (tick == t && tseq < ev_seq)) && tick < horizon) {
        if (!kLean && AFL_UNLIKELY(W.traced != 0) && (int32_t)nt < AFL_C.trace_tick_cap) {
#pragma unroll 1
            for (int32_t j = 0; j < AFL_C.n_series; ++j)
                if (gauge_on(j)) AFL_C.trace_series[(W.local * (uint64_t)AFL_C.n_series + (uint32_t)j) * (uint64_t)AFL_C.trace_tick_cap + nt] = gauge_value(m, j);
        }
        nt += 1;
        tseq = seq++;                                 // the collector re-arms its timeout here
        tick = tick + AFL_C.sample_period;
    }
    if (nt != W.n_ticks) {                            // every gauge has now been read at its current value
#pragma unroll 1
        for (int32_t w = 0; w < AFL_C.n_dirty; ++w) w32_st(m, AFL_C.o32_dirty + w, 0u);
    }
    W.tick_time = tick; W.tick_seq = tseq; W.n_ticks = nt; W.seq = seq;
}

// ---- per-tick bands: a replica joins its group's count at tick 0 (every gauge starts at 0), and a replica that a stop
//      flag ends leaves at the tick it stopped at: its current values and its count are taken back there, so the
//      frozen ticks to the horizon add nothing.  Every tick before n_ticks was taken before the event in which the
//      flag was raised: those are exact, and the warp-per-replica pass re-runs the replica from that tick (band_from).
AFL_IN void band_start(St& W) {
    const uint64_t i = W.replica - AFL_C.band_first;
    const uint32_t g = i < AFL_C.band_n ? AFL_C.band_group[i] : (uint32_t)AFL_C.band_groups;
    W.band = AFL_C.band_rows + (uint64_t)g * AFL_C.band_group_words;
    red_add64(W.band, 1u);
}
AFL_IN void band_stop(const St& W, const Mem& m) {
    const uint64_t n = W.n_ticks, stride = (uint64_t)AFL_C.band_stride, sq = (uint64_t)AFL_C.n_series * stride;
#pragma unroll 1
    for (int32_t j = 0; j < AFL_C.n_series; ++j) {
        if (!gauge_on(j)) continue;
        const uint64_t v = gauge_value(m, j);
        if (v == 0) continue;
        uint64_t* row = W.band + (uint64_t)(1 + j) * stride + n;
        red_add64(row, 0 - v);
        red_add64(row + sq, 0 - v * v);
    }
    red_add64(W.band + n, ~0ull);
    AFL_C.band_from[W.local] = (uint32_t)n;
}

// ---- per-window latency bands: a completion adds one to its latency bin and its latency in 32.32 fixed point to the
//      two sum words of its finish window, while no stop flag is set.  A flag raised during an iteration does not stop
//      the rest of it, and what completes after the flag may differ from what the warp-per-replica engine computes;
//      every completion before it is exact.  So the first completion after a flag records how many were added
//      (lat_from) and ends the replica's contribution; a replica stopped without one records them all at the stop.
//      `lat_g` is the replica's group (LAT_OFF: it adds no more), a register of run_lane's, not a member of St: the
//      kernels without latency bands keep the exact code they had before.
constexpr uint32_t LAT_OFF = ~0u;
AFL_IN uint32_t lat_group(const St& W) {
    const uint64_t i = W.replica - AFL_C.band_first;
    return i < AFL_C.band_n ? AFL_C.band_group[i] : (uint32_t)AFL_C.band_groups;
}
AFL_IN void lat_add(const St& W, uint32_t& lat_g, uint32_t done, double lat) {
    if (lat_g == LAT_OFF) return;
    if (AFL_UNLIKELY(W.flags & STOP_FLAGS)) { AFL_C.lat_from[W.local] = done - 1u; lat_g = LAT_OFF; return; }
    int32_t b = (int32_t)ceil(W.now) - 1;            // the throughput bucket, then its window: no division of doubles
    b = b < 0 ? 0 : b;
    if (b >= AFL_C.horizon_s) return;
    const uint64_t k = (uint32_t)b / (uint32_t)AFL_C.lat_window;
    uint64_t* row = AFL_C.lat_rows + ((uint64_t)lat_g * (uint32_t)AFL_C.lat_windows + k) * afr::LAT_ROW;
    red_add64(row + afr::hist_bin(lat), 1u);
    const uint64_t u = afr::lat_fixed32(lat);
    if (u >> 32) red_add64(row + AF_HIST_BINS, u >> 32);
    red_add64(row + AF_HIST_BINS + 1, u & 0xFFFFFFFFull);
}
AFL_IN void lat_stop(const St& W, uint32_t lat_g) {
    if (lat_g != LAT_OFF) AFL_C.lat_from[W.local] = W.completed;
}

// ---- per-tick distribution bands: the join and leave of the per-tick bands, over (tick, value bin) of the selected
//      series.  A replica joins bin(0) = 0 of every selected series at tick 0 and, stopped, leaves the bin of its
//      current value at its stop tick -- a value of 0 included (band_stop skips it: it adds nothing to a sum, but here
//      the replica would stay in the count).  dist_start keeps the replica's group (lat_group's) in W.dist_g for
//      gauge_touch.  One stop tick per replica in band_from, whichever kinds of bands are on.
AFL_IN void dist_start(St& W) {
    W.dist_g = lat_group(W);
#pragma unroll 1
    for (int32_t s = 0; s < AFL_C.dist_n; ++s) red_add32(dist_row(W.dist_g, s, 0u), 1u);
}
AFL_IN void dist_stop(const St& W, const Mem& m) {
    const uint32_t n = W.n_ticks;
#pragma unroll 1
    for (int32_t j = 0; j < AFL_C.n_series; ++j) {
        const int32_t s = dist_slot(j);
        if (s >= 0) red_add32(dist_row(W.dist_g, s, n) + dist_bin(gauge_value(m, j)), ~0u);
    }
    AFL_C.band_from[W.local] = n;
}

// ---- occupancy integrals: a replica starts with zeroed accumulators (a re-run of af_run's second pass starts over in
//      the warp-per-replica engine) and writes them out with its other results
AFL_IN void occ_start(const Mem& m) {
#pragma unroll 1
    for (int32_t c = 0; c < AFL_C.occ_cols; ++c) *g64p(m, AFL_C.gi_occ + c) = 0;
}
AFL_IN void occ_write(const St& W, const Mem& m) {
#pragma unroll 1
    for (int32_t c = 0; c < AFL_C.occ_cols; ++c)
        AFL_C.occ[W.local * (uint64_t)AFL_C.occ_cols + (uint32_t)c] = ld_cg64(g64p(m, AFL_C.gi_occ + c));
}

// ---- Stores (mailboxes), Containers: as af_core.cuh ----------------------------------------------------
// is the waiter FIFO whose head is cold word `head` empty?  (n_waiting == 0: all of them are, without looking)
AFL_IN bool q_empty(const St& W, const Mem& m, int32_t head) { return AFL_LIKELY(W.n_waiting == 0) || c32_ld(m, head) == NIL; }
// `yield box.get()` of the node's consumer process
AFL_IN void consumer_get(St& W, const Mem& m, uint32_t node) {
    if (AFL_UNLIKELY(c32_ld(m, ib_word(node, IB_HEAD)) != NIL)) {
        const uint32_t it = fifo_pop(m, ib_word(node, IB_HEAD), ib_word(node, IB_TAIL));
        nq_push(W, m, I_GOT, node, it);
    } else c32_st(m, ib_word(node, IB_PENDING), 1);
}
// Container._trigger_get over the CPU queue: grant heads while a core is free
// (returns true when `watch` was among the granted: its get is "triggered" at the call)
template <bool kOcc>
AFL_IN bool cpu_walk(St& W, const Mem& m, uint32_t sidx, uint32_t watch) {
    bool hit = false;
#pragma unroll 1
    while (!q_empty(W, m, sq_word(sidx, SQ_CPUQ_HEAD)) && i32_ld(m, sv_word(sidx, SV_CPU_FREE)) > 0) {
        const uint32_t w = fifo_pop(m, sq_word(sidx, SQ_CPUQ_HEAD), sq_word(sidx, SQ_CPUQ_TAIL));
        W.n_waiting -= 1;
        i32_st(m, sv_word(sidx, SV_CPU_FREE), i32_ld(m, sv_word(sidx, SV_CPU_FREE)) - 1);
        occ_add<kOcc>(W, m, occ_col(sidx, OC_CPU), 1);
        hit = hit || w == watch;
        nq_push(W, m, I_CPU_OK, sidx, w);
    }
    return hit;
}
// ... over the RAM queue: grant heads while they fit, stop at the first that does not
template <bool kOcc>
AFL_IN void ram_walk(St& W, const Mem& m, uint32_t sidx) {
#pragma unroll 1
    while (!q_empty(W, m, sq_word(sidx, SQ_RAMQ_HEAD))) {
        const uint32_t need = c32_ld(m, sq_word(sidx, SQ_RAMQ_NEED));
        if ((int32_t)need > i32_ld(m, sv_word(sidx, SV_RAM_FREE))) break;
        const uint32_t w = fifo_pop(m, sq_word(sidx, SQ_RAMQ_HEAD), sq_word(sidx, SQ_RAMQ_TAIL));
        W.n_waiting -= 1;
        occ_add<kOcc>(W, m, occ_col(sidx, OC_RAM_WAIT), -1);
        const uint32_t h = c32_ld(m, sq_word(sidx, SQ_RAMQ_HEAD));
        if (h != NIL) c32_st(m, sq_word(sidx, SQ_RAMQ_NEED), ep_total_ram(m, pk_ep(rq_pack(W, m, h))));
        i32_st(m, sv_word(sidx, SV_RAM_FREE), i32_ld(m, sv_word(sidx, SV_RAM_FREE)) - (int32_t)need);
        nq_push(W, m, I_RAM_OK, sidx, w);
    }
}

// ---- event injection (injection.py:167-226): all marks of this instant; returns true when the timeline re-arms
AFL_IN bool on_spike(St& W, const Mem& m, double& next_fire) {
    int32_t cur = W.spike_cur;
    const double t = ro(AFL_C.spikes + cur).fire;
#pragma unroll 1
    while (cur < AFL_C.n_spike) {
        const SpikeP p = ro(AFL_C.spikes + cur);
        if (p.fire != t) break;
        double delta = p.delta;
        if (p.c_delta >= 0) { const double v = row_val(m, p.c_delta); delta = delta < 0.0 ? -v : v; }
        f64_st(m, AFL_C.o64_spike + (int32_t)p.edge, f64_ld(m, AFL_C.o64_spike + (int32_t)p.edge) + delta);
        ++cur;
    }
    W.spike_cur = cur;
    if (cur < AFL_C.n_spike) { next_fire = ro(AFL_C.spikes + cur).fire; return true; }
    return false;
}
AFL_IN bool on_outage(St& W, const Mem& m, double& next_fire) {
    int32_t cur = W.outage_cur;
    const double t = ro(AFL_C.outages + cur).fire;
    int32_t n = W.lb_n;
    const int32_t lb = AFL_C.o32_lb;
#pragma unroll 1
    while (cur < AFL_C.n_outage) {
        const OutageP p = ro(AFL_C.outages + cur);
        if (p.fire != t) break;
        ++cur;
        if (p.lb_edge < 0) continue;
        int32_t at = -1;
#pragma unroll 1
        for (int32_t i = 0; i < n; ++i) if (w32_ld(m, lb + i) == (uint32_t)p.lb_edge) { at = i; break; }
        if (at >= 0) {                               // pop (DOWN) or move_to_end (UP)
#pragma unroll 1
            for (int32_t i = at + 1; i < n; ++i) w32_st(m, lb + i - 1, w32_ld(m, lb + i));
            --n;
        }
        if (!p.down) { w32_st(m, lb + n, (uint32_t)p.lb_edge); ++n; }
    }
    W.lb_n = n;
    W.outage_cur = cur;
    if (cur < AFL_C.n_outage) { next_fire = ro(AFL_C.outages + cur).fire; return true; }
    return false;
}

#if AFL_DEVICE
__device__ __forceinline__ void red_add(uint32_t* p, uint32_t v) { atomicAdd(p, v); }
#else
static inline void red_add(uint32_t* p, uint32_t v) { *p += v; }
#endif

// client: completion (client.py:62-69 + analyzer.py:83-125)
template <bool kLatency, bool kLean>
AFL_IN void complete(St& W, const Mem& m, uint32_t slot, double t0, uint32_t& lat_g) {
    const double now = W.now;
    const double lat = now - t0;                     // finish - start (analyzer.py:86-89)
    const uint32_t done = ++W.completed;
    W.lat_sum += lat;
    W.lat_sumsq += lat * lat;
    if (lat < W.lat_min) W.lat_min = lat;
    if (lat > W.lat_max) W.lat_max = lat;
    const uint64_t local = W.local;
    if (AFL_C.collect_hist) red_add(&AFL_C.hist[local * AF_HIST_BINS + (uint32_t)afr::hist_bin(lat)], 1u);
    if constexpr (kLatency) lat_add(W, lat_g, done, lat);
    if (AFL_C.collect_thr) {                          // bucket k counts (k, k+1] (analyzer.py:108-125)
        int32_t b = (int32_t)ceil(now) - 1;
        b = b < 0 ? 0 : b;
        if (b < AFL_C.horizon_s) red_add(&AFL_C.thr[local * (uint64_t)AFL_C.horizon_s + (uint32_t)b], 1u);
    }
    if constexpr (!kLean) {              // (`if (!kLean && ...)` here moves the SASS of the full kernel)
        if (AFL_UNLIKELY(W.traced != 0)) {
            if ((int32_t)(done - 1) < AFL_C.trace_clock_cap) {
                double* p = AFL_C.trace_clocks + (local * (uint64_t)AFL_C.trace_clock_cap + (done - 1)) * 2;
                p[0] = t0; p[1] = now;
            } else W.flags |= AF_FLAG_TRACE_TRUNCATED;
        }
    }
    rq_release(W, m, slot);
}

// ---- set-up / write-back (once per replica) -----------------------------------------------------------------
// (kLean: see run_lane -- no spike offsets, no traced replica)
template <bool kLean>
AFL_IN void start_replica(St& W, const Mem& m, uint64_t local_index) {
    const Cfg& C = AFL_C;
    W.local = local_index;
    W.replica = C.replica_begin + local_index;
    W.now = 0.0; W.horizon = (double)C.horizon_s; W.seq = 0;
    W.ev_n = 0; W.peak_ev = 0; W.arr_t = 0; W.arr_seq = 0; W.arr_on = 0;
    W.nq_head = 0; W.nq_tail = 0; W.busy = 0;
    // this replica's split of the pool, from its own pending-events estimate
    const uint64_t nr = W.replica - C.need_first;
    if (C.row_need != nullptr && nr < C.need_rows) {
        W.ev_s = pool_events(C.pool, C.ev_lo, C.rq_floor, C.ev_total, C.rq_total, C.row_need[nr]);
        W.rq_s = C.pool - W.ev_s;
    } else { W.ev_s = C.ev_s; W.rq_s = C.rq_s; }
    W.rq_mask = W.rq_s >= RQ_BITS ? ~0u : (1u << W.rq_s) - 1u;
    W.rq_free_hi = NIL; W.rq_hw = (uint32_t)W.rq_s; W.rq_live = 0; W.peak_rq = 0; W.n_waiting = 0;
    W.g_vnow = 0.0; W.g_wend = 0.0; W.g_lam = 0.0; W.g_pos = 0; W.generated = 0; W.g_done = 0;
    W.gap0 = 0.0; W.gap1 = 0.0; W.gap_cnt = 0;
    W.lb_n = C.n_lb_edges; W.spike_cur = 0; W.outage_cur = 0;
    W.n_ticks = 0; W.completed = 0; W.flags = 0; W.n_events = 0;
    W.lat_sum = 0.0; W.lat_sumsq = 0.0; W.lat_min = afr::u2d(INF_BITS); W.lat_max = 0.0;
    if constexpr (!kLean) W.traced = (int64_t)local_index < (int64_t)C.trace_replicas ? 1u : 0u;
    W.users_mean = C.users_mean; W.users_sigma = C.users_sigma; W.rate_per_user = C.rate_per_user;
#pragma unroll 1
    for (int32_t i = 0; i < C.n_edges; ++i) {
        w32_st(m, C.o32_conn + i, 0); *g32p(m, C.gi_sent + i) = 0; c32_st(m, C.c_drop + i, 0);
        if (!kLean && C.n_spike > 0) f64_st(m, C.o64_spike + i, 0.0);
    }
#pragma unroll 1
    for (int32_t i = 0; i < C.n_servers; ++i) {
        const ServerP p = ro(C.servers + i);
        i32_st(m, sv_word((uint32_t)i, SV_CPU_FREE), p.cpu_cores); i32_st(m, sv_word((uint32_t)i, SV_RAM_FREE), p.ram_mb);
        i32_st(m, sv_word((uint32_t)i, SV_READY_Q), 0); i32_st(m, sv_word((uint32_t)i, SV_IO_Q), 0); i32_st(m, sv_word((uint32_t)i, SV_RAM_IN_USE), 0);
        c32_st(m, sq_word((uint32_t)i, SQ_RAMQ_HEAD), NIL); c32_st(m, sq_word((uint32_t)i, SQ_RAMQ_TAIL), NIL);
        c32_st(m, sq_word((uint32_t)i, SQ_CPUQ_HEAD), NIL); c32_st(m, sq_word((uint32_t)i, SQ_CPUQ_TAIL), NIL);
        c32_st(m, sq_word((uint32_t)i, SQ_RAMQ_NEED), 0);
    }
#pragma unroll 1
    for (int32_t i = 0; i < C.n_servers + 2; ++i) {
        c32_st(m, ib_word((uint32_t)i, IB_HEAD), NIL); c32_st(m, ib_word((uint32_t)i, IB_TAIL), NIL); c32_st(m, ib_word((uint32_t)i, IB_PENDING), 1);
    }
#pragma unroll 1
    for (int32_t i = 0; i < C.n_lb_edges; ++i) w32_st(m, C.o32_lb + i, (uint32_t)C.lb_edges[i]);
#pragma unroll 1
    for (int32_t j = 0; j < C.n_series; ++j) { *g64p(m, C.gi_acc + j) = 0; *g32p(m, C.gi_smax + j) = 0; }
#pragma unroll 1
    for (int32_t w = 0; w < C.n_dirty; ++w) w32_st(m, C.o32_dirty + w, 0xFFFFFFFFu);      // no tick has read anything yet
    // sweep overrides of this replica: fields consumed here, fields looked up during the run (row copy)
    const bool has_row = C.n_sweep_cols > 0 && W.replica >= C.sweep_first && W.replica - C.sweep_first < C.sweep_rows;
    const double* row = C.sweep_vals + (has_row ? (W.replica - C.sweep_first) * (uint64_t)C.n_sweep_cols : 0);
#pragma unroll 1
    for (int32_t c = 0; c < C.n_sweep_cols; ++c) {
        const ColP col = C.cols[c];
        const double v = has_row ? row[c] : col.base;
        if (col.slot >= 0) { f64_st(m, C.o64_row + col.slot, v); continue; }
        if (!has_row || gen_field(col.field, v, W.users_mean, W.users_sigma, W.rate_per_user)) continue;
        switch (col.field) {
        case AF_FIELD_SERVER_CPU_CORES: i32_st(m, sv_word((uint32_t)col.index, SV_CPU_FREE), (int32_t)v); break;
        case AF_FIELD_SERVER_RAM_MB: i32_st(m, sv_word((uint32_t)col.index, SV_RAM_FREE), (int32_t)v); break;
        default: break;
        }
    }
    if (C.redo) {                                     // a re-run: the first pass left partial counts in the accumulating outputs
        if (C.collect_hist) for (int32_t b = 0; b < AF_HIST_BINS; ++b) C.hist[W.local * AF_HIST_BINS + (uint32_t)b] = 0;
        if (C.collect_thr) for (int32_t b = 0; b < C.horizon_s; ++b) C.thr[W.local * (uint64_t)C.horizon_s + (uint32_t)b] = 0;
    }
}

template <bool kLean>
AFL_IN void write_back(St& W, const Mem& m) {
    const Cfg& C = AFL_C;
    const uint64_t local = W.local;
#pragma unroll 1
    for (int32_t i = 0; i < C.n_edges; ++i) {
        C.edge_sent[local * (uint64_t)C.n_edges + (uint32_t)i] = ld_cg32(g32p(m, C.gi_sent + i));
        C.edge_dropped[local * (uint64_t)C.n_edges + (uint32_t)i] = c32_ld(m, C.c_drop + i);
    }
#pragma unroll 1
    for (int32_t j = 0; j < C.n_series; ++j) {       // settle the lazy aggregates (see gauge_touch)
        uint64_t sum = 0; uint32_t mx = 0;
        if (gauge_on(j)) {
            const uint32_t v = gauge_value(m, j);
            sum = (uint64_t)W.n_ticks * (uint64_t)v - ld_cg64(g64p(m, C.gi_acc + j));
            mx = ld_cg32(g32p(m, C.gi_smax + j));
            if (!((w32_ld(m, C.o32_dirty + (j >> 5)) >> (j & 31)) & 1u) && v > mx) mx = v;
        }
        C.samp_sum[local * (uint64_t)C.n_series + (uint32_t)j] = sum;
        C.samp_max[local * (uint64_t)C.n_series + (uint32_t)j] = mx;
    }
    AfReplicaStats st;
    st.n_events = W.n_events; st.generated = W.generated; st.completed = W.completed;
    st.flags = W.flags; st.n_ticks = W.n_ticks; st.peak_events = W.peak_ev; st.peak_requests = W.peak_rq;
    st.lat_sum = W.lat_sum; st.lat_sumsq = W.lat_sumsq;
    st.lat_min = W.completed ? W.lat_min : 0.0; st.lat_max = W.lat_max;
    st.p50 = st.p95 = st.p99 = afr::u2d(0x7FF8000000000000ull);
    C.stats[local] = st;
    if (!kLean && W.traced) { C.trace_counts[local * 2] = W.completed; C.trace_counts[local * 2 + 1] = W.n_ticks; }
}

// what a phase hands to the next one
enum : uint32_t { A_NONE = 0, A_NODE, A_STEPS, A_SEND, A_TIMER };

// Warp-wide rendez-vous between two phases.  Without it the lanes that split on the event kind stay split until
// the top of the loop (the compiler's reconvergence point of a branch inside a loop with early exits is the loop
// header), and a phase most lanes need ran with a few of them active.  Every lane passes every
// AFL_SYNC of an iteration -- no `continue` below.
#if AFL_DEVICE
#define AFL_SYNC() __syncwarp()
#else
#define AFL_SYNC() ((void)0)
#endif

// ---------------------------------------------------------------------------------------------------
// The lane's life: pull a replica, run it to the horizon, write it back, pull the next.  `next_index`
// returns the next local replica index or ~0 when the launch has no more work for this lane.
// `converge` is a warp-wide rendez-vous at the top of every iteration (device: __any_sync).
// The bands to accumulate over the replicas' groups, one flag each: `kSampled` the per-tick bands (Cfg.band_*),
// `kLatency` the per-window latency bands (Cfg.lat_*).  <false, false> compiles to the same code as before bands
// existed, <true, false> to the same code as before latency bands existed (two bools, not one integer mask: with an
// integer parameter the front end emits the same kernel in a different order, and the SASS moves).
// `kLean`: the launch has no spikes, no outages, no traced replica, only normal and exponential edges and one endpoint
// per server (aflh::lean_launch); the code for those features is left out of the loop, which does the same work in
// the same order with fewer instructions to fetch.  <S, L, false> compiles to the same code as before kLean existed.
// `kDist`: the per-tick distribution bands of the selected series (Cfg.dist_*) too; <S, L, Lean, false> compiles to
// the same code as before kDist existed.
// `kOcc`: the occupancy integrals too (Cfg.occ*, occ_add); <S, L, Lean, D, false> compiles to the same code as before
// kOcc existed.
// ---------------------------------------------------------------------------------------------------
template <bool kSampled = false, bool kLatency = false, bool kLean = false, bool kDist = false, bool kOcc = false,
          class NextFn, class ConvFn>
AFL_IN void run_lane(const Mem& m, NextFn next_index, ConvFn converge) {
    const Cfg& C = AFL_C;
    St W;
    uint32_t lat_g = LAT_OFF;
    bool active = false, exhausted = false;
#pragma unroll 1
    for (;;) {
        if (!converge(active || !exhausted)) break;          // all lanes of the warp are done
        // ---- phase: lifecycle -------------------------------------------------------------------
        if (AFL_UNLIKELY(!active && !exhausted)) {
            const uint64_t r = next_index();
            if (r == ~0ull) exhausted = true;
            else {
                start_replica<kLean>(W, m, r);
                if constexpr (kSampled) band_start(W);
                if constexpr (kLatency) lat_g = lat_group(W);
                if constexpr (kDist) dist_start(W);
                if constexpr (kOcc) occ_start(m);
                // start order of the reference (simulation_runner.py:339-342, 301-336):
                // spike timeline, outage timeline, generator, ..., collector
                if (!kLean && C.n_spike > 0) {
                    double f = ro(C.spikes).fire;
                    bool arm = true;
                    if (f == 0.0) arm = on_spike(W, m, f);
                    if (arm && f < W.horizon) { if (f == W.now) W.busy |= 1u; heap_push(W, m, afr::d2u(f), ((uint64_t)(W.seq++) << 32) | mk_payload(K_SPIKE, 0, 0)); }
                }
                if (!kLean && C.n_outage > 0) {
                    double f = ro(C.outages).fire;
                    bool arm = true;
                    if (f == 0.0) arm = on_outage(W, m, f);
                    if (arm && f < W.horizon) { if (f == W.now) W.busy |= 1u; heap_push(W, m, afr::d2u(f), ((uint64_t)(W.seq++) << 32) | mk_payload(K_OUTAGE, 0, 0)); }
                }
                W.arm_seq = W.seq++; W.need_arrival = 1;
                W.tick_seq = W.seq++;
                W.tick_time = 0.0 + C.sample_period;
                active = true;
            }
        }
        AFL_SYNC();
        const bool run = active;                              // a lane without a replica idles through the phases
        const bool dead = run && (W.flags & STOP_FLAGS) != 0; // a pool overflowed in the last iteration: stop the replica here
        // ---- phase: the generator's next timeout (rqs_generator.py:103-104) ------------------------------
        if (run && W.need_arrival && !dead) {
            W.need_arrival = 0;
            double gap = 0.0;
            bool have = false;
            if (W.gap_cnt) { gap = W.gap0; W.gap0 = W.gap1; W.gap_cnt -= 1u; have = true; }      // drawn ahead
            else if (!W.g_done && gen_next_gap(W, gap)) have = true;                          // (rare: see the SEND phase)
            if (have) {
                const double t = W.now + gap;
                if (t < W.horizon) {                         // env.run(until=T): events at >= T never fire
                    if (AFL_UNLIKELY(t == W.now)) W.busy |= 1u;
                    if (AFL_UNLIKELY(W.ev_n >= AFL_C.ev_total)) W.flags |= AF_FLAG_EVENT_OVERFLOW;
                    else {
                        W.arr_t = afr::d2u(t); W.arr_seq = W.arm_seq; W.arr_on = 1u;
                        if ((uint32_t)W.ev_n + 1u > W.peak_ev) W.peak_ev = (uint32_t)W.ev_n + 1u;
                    }
                }
            } else W.g_done = 1;
        }
        AFL_SYNC();
        // ---- phase: pick the next thing to run: a zero-delay item or the earliest timed event ------------
        uint32_t word = 0;                    // item or event payload
        bool is_item = false, finish = false, is_event = false;
        double t_ev = 0.0; uint32_t ev_seq = 0;
        if (run) {
            if (AFL_UNLIKELY(dead)) finish = true;
            else {
                const uint32_t busy = W.busy;
                const bool have_item = busy >= 2u;
                if (have_item && !(busy & 1u)) {         // no heap event shares this instant: just drain
                    W.busy = busy - 2u;
                    word = nq_take(W, m);
                    is_item = true;
                } else {
                    const bool have_heap = W.ev_n > 0, have_ev = have_heap || W.arr_on != 0;
                    uint64_t tb = 0, key = 0;
                    if (have_heap) sm_ld128(m.s128, tb, key);      // the root is always in shared memory (ev_s >= 1)
                    const uint64_t root_t = tb;
                    bool take_arr = false;                // the earliest timed event: the heap's root or the generator's timeout
                    if (W.arr_on) {
                        const uint64_t ak = ((uint64_t)W.arr_seq << 32) | mk_payload(K_ARRIVAL, 0, 0);
                        if (!have_heap || ev_less(W.arr_t, ak, tb, key)) { tb = W.arr_t; key = ak; take_arr = true; }
                    }
                    if (have_item) {
                        const uint64_t front = nq_ld(m, W.nq_head);
                        const bool same_t = have_ev && tb == afr::d2u(W.now);
                        if (!(same_t && (uint32_t)(key >> 32) < (uint32_t)(front >> 32))) {
                            W.busy = (same_t ? busy : (busy & ~1u)) - 2u;
                            word = nq_take(W, m);
                            is_item = true;
                        }
                    } else if (!have_ev) finish = true;
                    if (!is_item && !finish) {
                        bool more;
                        if (take_arr) { W.arr_on = 0u; more = have_heap && root_t == tb; }
                        else { heap_pop(W, m); more = (W.ev_n > 0 && sm_ld64(m.s128) == tb) || (W.arr_on && W.arr_t == tb); }
                        W.busy = (W.busy & ~1u) | (more ? 1u : 0u);
                        t_ev = afr::u2d(tb); ev_seq = (uint32_t)(key >> 32); word = (uint32_t)key;
                        is_event = true;
                    }
                }
            }
            if (finish) { t_ev = W.horizon; ev_seq = 0u; }      // ticks strictly before the horizon
        }
        AFL_SYNC();
        // ---- phase: collector ticks that fall before this event ------------------------------------------------
        if constexpr (kSampled) { if (AFL_UNLIKELY(dead)) band_stop(W, m); }     // before the frozen ticks to the horizon
        if constexpr (kLatency) { if (AFL_UNLIKELY(dead)) lat_stop(W, lat_g); }
        if constexpr (kDist) { if (AFL_UNLIKELY(dead)) dist_stop(W, m); }
        if (run && !is_item) {
            const double tick = W.tick_time;
            if (tick < t_ev || (tick == t_ev && W.tick_seq < ev_seq)) take_ticks<kLean>(W, m, t_ev, ev_seq);
        }
        if (AFL_UNLIKELY(finish)) {
            write_back<kLean>(W, m);
            if constexpr (kOcc) occ_write(W, m);
            active = false;
        }
        AFL_SYNC();
        if (is_event) { W.now = t_ev; W.n_events += 1; }

        // ---- phase: decode -------------------------------------------------------------------------------------
        const uint32_t kind = word >> 29, aux = (word >> SLOT_BITS) & AUX_MASK;
        uint32_t slot = word & SLOT_MASK;
        uint32_t act = A_NONE;
        uint32_t node = 0, sidx = 0, rid = 0, pack = 0, edge = 0;
        bool from_box = true;                  // A_NODE reached through the mailbox (an I_GOT item), not fused with the delivery
        double t0 = 0.0;
        double tm_t = 0.0; uint32_t tm_payload = 0, tm_seq = 0;
        AFL_TRACE("%s t=%.17g seq=%u kind=%u aux=%u slot=%u\n", is_item ? "it" : "ev", W.now, ev_seq, kind, aux, slot);
        // everything that names a request reads its record here, once, for all kinds
        const bool names_request = is_event ? (kind == K_DELIVER || kind == K_STEP_END) : (is_item && kind != I_CLIENT_LOOP && kind != I_PUT);
        if (names_request) rq_load(W, m, slot, t0, rid, pack);
        if (is_event) {
            if (kind == K_DELIVER) {                          // edge.py:110-116: the edge's timeout fired
                conn_add<kSampled, kDist, kOcc>(W, m, aux, -1);
                const uint32_t meta = ro(C.edges + aux).meta;
                pack += 1;                                     // record_hop(edge)
                const uint32_t tk = (meta >> 3) & 3u;
                node = tk == AF_TARGET_CLIENT ? NODE_CLIENT : (tk == AF_TARGET_LB ? NODE_LB : NODE_SERVER0 + (meta >> 5));
                if (can_fuse(W)) { act = A_NODE; from_box = false; }   // put -> pending get -> resume, nothing in between
                else {                                         // (fused implies: every inbox empty, every consumer in get())
                    rq_pack_set(W, m, slot, pack);
                    fifo_push(m, ib_word(node, IB_HEAD), ib_word(node, IB_TAIL), slot);   // Store.put: items.append now ...
                    nq_push(W, m, I_PUT, node, slot);                                       // ... the put event is processed later
                }
            } else if (kind == K_STEP_END) {
                sidx = aux;
                pack += (1u << 8);                             // the timeout fired: next step
                act = A_STEPS;
            } else if (kLean || kind == K_ARRIVAL) {          // rqs_generator.py:97-119 (lean: the only kind left)
                rid = ++W.generated;
                slot = rq_alloc(W, m);
                // the generator asks the sampler for the next gap right after transport(): its timeout is
                // scheduled BEFORE the edge's delivery timeout.  The seq is reserved here.
                W.arm_seq = W.seq++;
                W.need_arrival = 1;
                if (slot != NIL) {
                    pack = 1u; edge = (uint32_t)C.gen_edge;        // record_hop(generator)
                    rq_store(W, m, slot, W.now, rid, pack);
                    act = A_SEND;
                }
            } else if (kind == K_SPIKE) {
                double f;
                if (on_spike(W, m, f)) { tm_t = f; tm_payload = mk_payload(K_SPIKE, 0, 0); tm_seq = W.seq++; act = A_TIMER; }
            } else {
                double f;
                if (on_outage(W, m, f)) { tm_t = f; tm_payload = mk_payload(K_OUTAGE, 0, 0); tm_seq = W.seq++; act = A_TIMER; }
            }
        } else if (is_item) {
            if (kind == I_GOT) {
                node = aux;
                act = A_NODE;
            } else if (kind == I_PUT) {                        // a StorePut event is processed
                if (c32_ld(m, ib_word(aux, IB_PENDING))) {
                    c32_st(m, ib_word(aux, IB_PENDING), 0);
                    nq_push(W, m, I_GOT, aux, fifo_pop(m, ib_word(aux, IB_HEAD), ib_word(aux, IB_TAIL)));
                }
            } else if (kind == I_CLIENT_LOOP) {
                consumer_get(W, m, NODE_CLIENT);
            } else if (kind == I_RAM_OK) {                     // the RAM get event is processed: the handler resumes
                sidx = aux;
                srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_RAM_IN_USE, (int32_t)ep_total_ram(m, pk_ep(pack)));
                act = A_STEPS;
            } else if (kind == I_CPU_OK) {                     // the CPU get event is processed
                sidx = aux;
                if (pack & PK_WAIT) { pack &= ~PK_WAIT; srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_READY_Q, -1); }
                pack |= PK_CORE;
                act = A_STEPS;
            } else if (kind == I_CPU_PUT) {                    // waiters are re-examined, then the request goes on
                sidx = aux;
                cpu_walk<kOcc>(W, m, sidx, NIL);
                pack &= ~PK_CORE;                              // core_locked = False; same step again
                act = A_STEPS;
            } else {                                           // I_RAM_PUT: waiters first, then forward
                sidx = aux;
                ram_walk<kOcc>(W, m, sidx);
                edge = ro(C.servers + sidx).out_edge;
                act = A_SEND;
            }
        }
        AFL_SYNC();

        // ---- phase: a node's consumer process resumes with `slot` (the StoreGet event is processed) ---------------
        if (act == A_NODE) {
            act = A_NONE;
            if (node >= NODE_SERVER0) {                       // server.py:303-313, then the head of _handle_request (:88-149)
                sidx = node - NODE_SERVER0;
                if (from_box) consumer_get(W, m, node);        // the dispatcher loops back to get() first (fused: the box is empty and
                                                               // the consumer already marked as waiting -- nothing to do)
                const ServerP sp = ro(C.servers + sidx);
                pack += 1;                                     // record_hop(SERVER)
                uint32_t epi = 0;
                if (!kLean && sp.n_ep > 1) {
                    afr::Src src = afr::make_request(C.seed, W.replica, afr::P_SERVER, rid, pk_hops(pack));
                    src.load(0);
                    epi = (uint32_t)(((uint64_t)src.w.x * sp.n_ep) >> 32);
                }
                const uint32_t ep_global = sp.ep_begin + epi;
                pack = (pack & 0xFFu) | (ep_global << 16);     // step 0, flags clear
                const uint32_t total_ram = ep_total_ram(m, ep_global);
                bool go = true;
                if (total_ram) {                               // yield RAM.get(total_ram)
                    if (!(can_fuse(W) && (int32_t)total_ram <= i32_ld(m, sv_word(sidx, SV_RAM_FREE)) && q_empty(W, m, sq_word(sidx, SQ_RAMQ_HEAD)))) {
                        // cannot be served at once: join the queue, walk it
                        rq_pack_set(W, m, slot, pack);
                        if (q_empty(W, m, sq_word(sidx, SQ_RAMQ_HEAD))) c32_st(m, sq_word(sidx, SQ_RAMQ_NEED), total_ram);
                        fifo_push(m, sq_word(sidx, SQ_RAMQ_HEAD), sq_word(sidx, SQ_RAMQ_TAIL), slot);
                        W.n_waiting += 1;
                        occ_add<kOcc>(W, m, occ_col(sidx, OC_RAM_WAIT), 1);
                        ram_walk<kOcc>(W, m, sidx);
                        go = false;
                    } else {
                        i32_st(m, sv_word(sidx, SV_RAM_FREE), i32_ld(m, sv_word(sidx, SV_RAM_FREE)) - (int32_t)total_ram);   // granted, and its get event would run next
                        srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_RAM_IN_USE, (int32_t)total_ram);
                    }
                }
                if (go) act = A_STEPS;
            } else {
                pack += 1;                                     // record_hop(client / LB)
                if (node == NODE_CLIENT) {
                    if (pk_hops(pack) > 3) {                   // client.py:62: back from the servers
                        complete<kLatency, kLean>(W, m, slot, t0, lat_g);
                        if (can_fuse(W)) { if (from_box) consumer_get(W, m, NODE_CLIENT); }
                        else nq_push(W, m, I_CLIENT_LOOP, 0, 0);   // yield completed_box.put(state)
                    } else {
                        if (from_box) consumer_get(W, m, NODE_CLIENT);
                        edge = (uint32_t)C.client_edge;
                        act = A_SEND;
                    }
                } else {
                    const int32_t lb = C.o32_lb, n = W.lb_n;
                    // every covered server is down: the reference dies here (StopIteration inside round_robin);
                    // the replica stops and says so (flatten() rejects timelines that can reach this state)
                    if (AFL_UNLIKELY(n <= 0)) { rq_pack_set(W, m, slot, pack); W.flags |= AF_FLAG_LB_EMPTY; }
                    else {
                        uint32_t pick = w32_ld(m, lb);
                        if (C.lb_algo == AF_LB_ROUND_ROBIN) {      // lb_algorithms.py:22-36
#pragma unroll 1
                            for (int32_t i = 1; i < n; ++i) w32_st(m, lb + i - 1, w32_ld(m, lb + i));
                            w32_st(m, lb + n - 1, pick);
                        } else {                                   // least_connections, :10-20 (first min wins)
                            uint32_t best = w32_ld(m, C.o32_conn + (int32_t)pick);
#pragma unroll 1
                            for (int32_t i = 1; i < n; ++i) {
                                const uint32_t e2 = w32_ld(m, lb + i), c2 = w32_ld(m, C.o32_conn + (int32_t)e2);
                                if (c2 < best) { best = c2; pick = e2; }
                            }
                        }
                        if (from_box) consumer_get(W, m, NODE_LB);
                        edge = pick;
                        act = A_SEND;
                    }
                }
            }
        }
        AFL_SYNC();

        // ---- phase: the `for step in endpoint.steps` loop (server.py:197-255) up to the request's next yield,
        //      and the tail of the handler (server.py:257-276) ---------------------------------------------------------
        if (act == A_STEPS) {
            act = A_NONE;
            const EndpointP ep = ro(C.endpoints + pk_ep(pack));
#pragma unroll 1
            for (;;) {
                const uint32_t st = pk_step(pack);
                if (st < ep.n_steps) {
                    const StepP sp = ro(C.steps + ep.step_begin + st);
                    if (sp.kind == AF_STEP_CPU) {
                        if (pack & PK_IO) { pack &= ~PK_IO; srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_IO_Q, -1); }
                        if (!(pack & PK_CORE)) {             // cpu_req = CPU.get(1); yield cpu_req
                            if (can_fuse(W) && i32_ld(m, sv_word(sidx, SV_CPU_FREE)) > 0 && q_empty(W, m, sq_word(sidx, SQ_CPUQ_HEAD))) {
                                i32_st(m, sv_word(sidx, SV_CPU_FREE), i32_ld(m, sv_word(sidx, SV_CPU_FREE)) - 1);     // granted, and its get event would run next
                                occ_add<kOcc>(W, m, occ_col(sidx, OC_CPU), 1);
                                pack |= PK_CORE;
                            } else {
                                fifo_push(m, sq_word(sidx, SQ_CPUQ_HEAD), sq_word(sidx, SQ_CPUQ_TAIL), slot);
                                W.n_waiting += 1;
                                if (!cpu_walk<kOcc>(W, m, sidx, slot)) { pack |= PK_WAIT; srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_READY_Q, 1); }   // not cpu_req.triggered
                                break;
                            }
                        }
                    } else {
                        if (pack & PK_CORE) {                // yield CPU.put(1): level rises NOW
                            i32_st(m, sv_word(sidx, SV_CPU_FREE), i32_ld(m, sv_word(sidx, SV_CPU_FREE)) + 1);
                            occ_add<kOcc>(W, m, occ_col(sidx, OC_CPU), -1);
                            if (can_fuse(W)) {
                                if (AFL_UNLIKELY(!q_empty(W, m, sq_word(sidx, SQ_CPUQ_HEAD)))) cpu_walk<kOcc>(W, m, sidx, NIL);
                                pack &= ~PK_CORE;
                                continue;
                            }
                            nq_push(W, m, I_CPU_PUT, sidx, slot);
                            break;
                        }
                        if (!(pack & PK_IO)) { pack |= PK_IO; srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_IO_Q, 1); }
                    }
                    const double dur = sp.c_dur >= 0 ? row_val(m, sp.c_dur) : sp.dur;
                    tm_t = W.now + dur; tm_payload = mk_payload(K_STEP_END, sidx, slot); tm_seq = W.seq++;
                    act = A_TIMER;
                    break;
                }
                // end of the endpoint (server.py:257-276)
                if (pack & PK_CORE) {                        // yield CPU.put(1)
                    i32_st(m, sv_word(sidx, SV_CPU_FREE), i32_ld(m, sv_word(sidx, SV_CPU_FREE)) + 1);
                    occ_add<kOcc>(W, m, occ_col(sidx, OC_CPU), -1);
                    if (can_fuse(W)) {
                        if (AFL_UNLIKELY(!q_empty(W, m, sq_word(sidx, SQ_CPUQ_HEAD)))) cpu_walk<kOcc>(W, m, sidx, NIL);
                        pack &= ~PK_CORE;
                        continue;
                    }
                    nq_push(W, m, I_CPU_PUT, sidx, slot);
                    break;
                }
                if (pack & PK_IO) { pack &= ~PK_IO; srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_IO_Q, -1); }
                const uint32_t total_ram = ep.c_ram >= 0 ? (uint32_t)row_val(m, ep.c_ram) : ep.total_ram;
                if (total_ram) {                             // yield RAM.put(total_ram): level rises NOW
                    srv_gauge_add<kSampled, kDist, kOcc>(W, m, sidx, SV_RAM_IN_USE, -(int32_t)total_ram);
                    i32_st(m, sv_word(sidx, SV_RAM_FREE), i32_ld(m, sv_word(sidx, SV_RAM_FREE)) + (int32_t)total_ram);
                    if (!can_fuse(W)) { nq_push(W, m, I_RAM_PUT, sidx, slot); break; }
                    if (AFL_UNLIKELY(!q_empty(W, m, sq_word(sidx, SQ_RAMQ_HEAD)))) ram_walk<kOcc>(W, m, sidx);   // the put event would run next: waiters, then forward
                }
                edge = ro(C.servers + sidx).out_edge;
                act = A_SEND;
                break;
            }
            if (act != A_SEND) rq_pack_set(W, m, slot, pack);   // the request yields here: its record goes back (SEND stores its own)
        }
        AFL_SYNC();

        // ---- phase: EdgeRuntime.transport -> _deliver up to its timeout (edge.py:73-107) ---------------------------
        // The edge's variates are the most expensive thing an event does (Philox, a logarithm, a division), and the
        // lanes that do not send in this iteration would sit them out.  They ride along instead: a lane whose
        // generator has room in its two-deep gap buffer draws its NEXT inter-arrival gap here -- same Philox, same
        // logarithm, same division, other operands.  AF-RNG is counter-based and the generator's stream is a function
        // of its own virtual clock alone, so WHEN a gap is drawn cannot change it.  Only the plain case is taken (one
        // uniform, inside the current window); anything else is left to gen_next_gap at the arrival.
        {
            const bool send = act == A_SEND;
            uint32_t s = 0; double dropout = 0.0, mean = 0.0, sigma = 0.0; int dist = 0;
            if (send) {
                act = A_NONE;
                const EdgeP E = ro(C.edges + edge);
                s = W.seq++;                                 // the timeout's place in SimPy's eid order
                dropout = E.c_drop >= 0 ? row_val(m, E.c_drop) : E.dropout;
                mean = E.c_mean >= 0 ? row_val(m, E.c_mean) : E.mean;
                sigma = E.c_sigma >= 0 ? row_val(m, E.c_sigma) : E.sigma;
                dist = (int)(E.meta & 7u);
            }
            const bool fast = kLean ? send : send && (dist == 1 /*NORMAL*/ || dist == 3 /*EXPONENTIAL*/);
            const bool ride = !send && (is_event || is_item) && !finish && W.gap_cnt < 2u && !W.g_done
                              && W.g_vnow < W.horizon && W.g_vnow < W.g_wend && W.g_lam > 0.0;
            double u = 0.0, transit = 0.0;
            if (!kLean && send && !fast) {                   // the other distributions: the general sampler, out of line
                const afr::EdgeDraw d = afr::edge_draw(C.seed, W.replica, rid, pk_hops(pack), dist, mean, sigma, dropout);
                u = d.u; transit = d.transit;
            }
            // (a rendez-vous of its own: without it the compiler specialises the block below for senders and for riders
            //  -- `send` is known on either path -- and the two copies run one after the other)
            AFL_SYNC();
            if (fast || ride) {
                const uint32_t k0 = (uint32_t)C.seed, k1 = (uint32_t)(C.seed >> 32);
                const uint32_t tag = (afr::P_EDGE << 24) | ((pk_hops(pack) & 0xFFFFu) << 8);
                afr::U4 c;
                c.x = send ? rid : (W.g_pos >> 1); c.y = send ? tag : (afr::P_GEN << 24);
                c.z = (uint32_t)W.replica; c.w = (uint32_t)(W.replica >> 32);
                afr::U4 w = afr::philox4x32_10(c, k0, k1);
                double arg = 1.0, v1 = 0.0, q = 1.0;
                bool need = true;
                if (send) {
                    u = afr::u53(w.x, w.y);                  // rng.uniform() < dropout_rate (edge.py:78)
                    if (u < dropout) need = false;
                    else if (dist == 3) arg = 1.0 - afr::u53(w.z, w.w);
                    else {                                   // polar method: first pair from this block, more from the next ones
                        v1 = afr::s32(w.z); const double v2 = afr::s32(w.w);
                        q = v1 * v1 + v2 * v2;
                        uint32_t blk = 0; bool second = true;
#pragma unroll 1
                        while (!(q > 0.0 && q < 1.0)) {
                            if (second) { ++blk; c.y = tag | afr::block_bits(blk); w = afr::philox4x32_10(c, k0, k1); v1 = afr::s32(w.x); const double b = afr::s32(w.y); q = v1 * v1 + b * b; }
                            else { v1 = afr::s32(w.z); const double b = afr::s32(w.w); q = v1 * v1 + b * b; }
                            second = !second;
                        }
                        arg = q;
                    }
                } else {
                    double ug = (W.g_pos & 1u) ? afr::u53(w.z, w.w) : afr::u53(w.x, w.y);
                    if (ug < 1e-15) ug = 1e-15;             // max(u, 1e-15)
                    arg = 1.0 - ug;
                }
                double L = 0.0;
                if (need) L = afr::af_log(arg);
                const bool divide = need && !(send && dist == 3);
                double D = 0.0;
                if (divide) D = send ? afr::af_div(-2.0 * L, q) : afr::af_div(-L, W.g_lam);
                if (send) {
                    if (need) {
                        if (dist == 3) transit = mean * -L;
                        else { const double v = mean + sigma * (v1 * afr::af_sqrt(D)); transit = v > 0.0 ? v : 0.0; }
                    }
                } else if (!(W.g_vnow + D > W.horizon) && !(W.g_vnow + D >= W.g_wend)) {       // the plain case of gen_next_gap
                    W.g_vnow += D; W.g_pos += 1u;
                    if (W.gap_cnt == 0u) W.gap0 = D; else W.gap1 = D;
                    W.gap_cnt += 1u;
                }
            }
            if (send) {
                red_add32(g32p(m, C.gi_sent + (int32_t)edge), 1u);
                if (u < dropout) {                          // the request vanishes (edge.py:79-86)
                    c32_st(m, C.c_drop + (int32_t)edge, c32_ld(m, C.c_drop + (int32_t)edge) + 1);
                    rq_release(W, m, slot);
                } else {
                    rq_pack_set(W, m, slot, pack);              // (the one store of the record on the request's way out of a node)
                    conn_add<kSampled, kDist, kOcc>(W, m, edge, 1);
                    double effective = transit;
                    if (!kLean && C.n_spike > 0) effective = transit + f64_ld(m, C.o64_spike + (int32_t)edge);   // spike read at SEND time (edge.py:94-106)
                    else effective = transit + 0.0;         // (-0.0 + 0.0 = +0.0, as with a spike table of zeros)
                    tm_t = W.now + effective; tm_payload = mk_payload(K_DELIVER, edge, slot); tm_seq = s;
                    act = A_TIMER;
                }
            }
        }
        AFL_SYNC();

        // ---- phase: schedule the timeout ------------------------------------------------------------------------------
        if (act == A_TIMER) {
            if (tm_t < W.horizon) {                          // env.run(until=T): events at >= T never fire
                if (AFL_UNLIKELY(tm_t == W.now)) W.busy |= 1u;   // a zero-delay timeout: it competes with the now-queue
                heap_push(W, m, afr::d2u(tm_t), ((uint64_t)tm_seq << 32) | tm_payload);
            }
        }
    }
}

}  // namespace afl
