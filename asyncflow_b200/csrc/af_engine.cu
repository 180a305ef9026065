// af_engine.cu -- sm_90a kernels and the C ABI of include/asyncflow_b200.h.
//
// Kernels:
//   af_lane_kernel        one replica per THREAD (af_lane.cuh).  One persistent CTA of up to 12 warps per SM; a
//                         lane's mutable state is element-interleaved in shared memory (conflict-free however far
//                         the 32 replicas of a warp drift apart), deep tiers and write-only aggregates in global
//                         memory; lanes pull replica indices from a global counter through the pull order
//                         (af_order_key_kernel + radix sorts: heaviest first).  af_run uses it when the launch
//                         has replicas for most lanes (AF_MODE_AUTO: n >= 3 x SMs x 32) and the topology leaves it
//                         at least 4 warps per SM.
//   af_flagged_kernel     compacts the replicas that overflowed the lane kernel's tiers (sized for nominal load)
//                         into a list ...
//   af_sim_kernel         ... which the warp-per-replica engine (af_core.cuh, large HBM tiers) re-runs; also the
//                         whole run for small launches and very wide topologies.  One replica per warp,
//                         persistent CTAs pulling replica indices from a global counter; per-warp workspace in
//                         shared memory with spill tiers in HBM.
//   af_band_scan_kernel   per-tick bands (af_bands_upload): the groups' difference rows -> per-tick sums, in place
//                         (per-window latency bands need no pass after the kernels: their rows are the sums)
//   af_percentile_kernel  HBM-bound pass over the per-replica latency histograms:
//                         one warp per replica, coalesced 128-byte row reads, warp
//                         prefix sums, numpy-"linear" p50/p95/p99.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false
// (-fmad=false is part of the parity contract: see af_rng.cuh).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "af_host_common.h"
#include "af_lane_host.h"

// Per-event cost of a replica in units of one event it keeps pending: an event costs AF_ORDER_EVENT_COST + need.
// Least-squares fit of lane time per event against the row's estimate on the bench workload (H100, DESIGN.md §6).
#ifndef AF_ORDER_EVENT_COST
#define AF_ORDER_EVENT_COST 44.0
#endif

// thread-per-replica pass: most warps per SM when the caller does not say (AfOptions.warps_per_block); af_run lowers it
// to whole waves and to what the topology's fixed tables leave room for (12: see af_lane_kernel)
#ifndef AF_LANE_DEFAULT_WARPS
#define AF_LANE_DEFAULT_WARPS 12
#endif

// occupancy knob: registers are capped (64/thread, a few bytes of spills) so that 8 128-thread CTAs fit per SM.
#ifndef AF_MIN_BLOCKS
#define AF_MIN_BLOCKS 8
#endif
#if AF_MIN_BLOCKS > 0
#define AF_LAUNCH_BOUNDS __launch_bounds__(128, AF_MIN_BLOCKS)
#else
#define AF_LAUNCH_BOUNDS
#endif

// ---------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------
__global__ void AF_LAUNCH_BOUNDS af_sim_kernel(const afc::BandArgs band) {
    extern __shared__ __align__(16) unsigned char af_smem[];
    const int warp = (int)(threadIdx.x >> 5);
    const int lane = (int)(threadIdx.x & 31u);
    unsigned char* ws = af_smem + (size_t)warp * (size_t)afc::c_L.warp_bytes;
    const uint64_t warp_slot = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (uint64_t)warp;
    afc::State& W = *reinterpret_cast<afc::State*>(ws);
    afc::bind(W, ws, warp_slot);
    __syncwarp();
    for (;;) {
        unsigned long long r = 0;
        if (lane == 0) r = atomicAdd(afc::c_G.work_counter, 1ull);
        r = __shfl_sync(0xFFFFFFFFu, r, 0);
        if (afc::c_G.redo_list) {                      // second pass: only the replicas the first pass flagged
            if (r >= (unsigned long long)*afc::c_G.redo_count) break;
            r = afc::c_G.redo_list[r];
        } else if (r >= afc::c_G.n_replicas) break;
        else r = afc::c_G.order[r];
        afc::run_replica(W, (uint64_t)r, band);
        __syncwarp();
    }
}

// One replica per thread.  Compiled for one CTA of up to 384 threads per SM (the shared-memory budget of a
// lane decides the CTA size at launch).  More warps shrink each lane's share of shared memory (more of the heap lives
// in L2), so the register budget is spent at 12 warps: 158 registers on sm_90a, no spills.  kSampled / kLatency: the
// same kernel also accumulating the per-tick / per-window latency bands of the uploaded groups (af_run picks the one
// the band options ask for); <false, false> is the kernel without them.  kLean: the loop without spikes, outages,
// traces, the general edge sampler and the endpoint draw (af_run picks it when aflh::lean_launch says the launch can
// reach none of them).  kDist: the per-tick distribution bands of the selected series too (af_dist_bands_configure).
// kOcc: the occupancy integrals too (af_occupancy_configure).
#ifndef AF_LANE_MAX_THREADS
#define AF_LANE_MAX_THREADS 384
#endif
template <bool kSampled = false, bool kLatency = false, bool kLean = false, bool kDist = false, bool kOcc = false>
__global__ void __launch_bounds__(AF_LANE_MAX_THREADS, 1) af_lane_kernel() {
    const afl::Cfg& C = afl::c_cfg;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t ws = warp * (uint32_t)C.warp_bytes;
    unsigned char* gs = C.gtier + ((uint64_t)blockIdx.x * (blockDim.x >> 5) + warp) * C.gwarp_bytes;
    afl::Mem m;
    m.s128 = ws + lane * 16u;
    m.s64 = ws + (uint32_t)C.n128 * (uint32_t)afl::STRIDE128 + lane * 8u;
    m.s32 = ws + (uint32_t)C.n128 * (uint32_t)afl::STRIDE128 + (uint32_t)C.n64 * (uint32_t)afl::STRIDE64 + lane * 4u;
    m.g128 = gs + lane * 16u;
    m.g64 = gs + (size_t)C.gn128 * afl::STRIDE128 + lane * 8u;
    m.g32 = gs + (size_t)C.gn128 * afl::STRIDE128 + (size_t)C.gn64 * afl::STRIDE64 + lane * 4u;
    afl::run_lane<kSampled, kLatency, kLean, kDist, kOcc>(m,
        [&]() -> uint64_t {
            const unsigned long long k = atomicAdd(C.work_counter, 1ull);
            return k < C.n_replicas ? (uint64_t)C.order[k] : ~0ull;
        },
        [](bool alive) -> bool { return __any_sync(0xFFFFFFFFu, alive) != 0; });
}

// per-tick bands: the difference rows -> per-tick values, in place.  One warp per row: 32 ticks at a time, a warp prefix
// sum plus the carry of the ticks before (u64 modular arithmetic: exact, whatever order the lanes added in)
__global__ void af_band_scan_kernel(uint64_t* __restrict__ rows, uint64_t n_rows, uint64_t stride, uint64_t n_ticks) {
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (row >= n_rows) return;
    uint64_t* r = rows + row * stride;
    uint64_t carry = 0;
    for (uint64_t base = 0; base < n_ticks; base += 32) {
        const uint64_t k = base + lane;
        uint64_t x = k < n_ticks ? r[k] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t up = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if ((int)lane >= d) x += up;
        }
        x += carry;
        if (k < n_ticks) r[k] = x;
        carry = __shfl_sync(0xFFFFFFFFu, x, 31);
    }
}

// per-tick distribution bands: the difference rows -> per-tick bin counts, in place.  One thread per (group, series, bin)
// of the n_rows = groups x series rows, a running u32 carry down the ticks; the threads of a warp read consecutive bins
// of one tick row (coalesced).  u32 modular arithmetic: exact whatever order the REDs landed in, as a bin count stays
// below 2^32 (a group holds fewer replicas than that).
__global__ void af_dist_scan_kernel(uint32_t* __restrict__ rows, uint64_t n_rows, uint32_t n_bins, uint64_t series_words,
                                    uint64_t n_ticks) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rows * n_bins) return;
    uint32_t* r = rows + (i / n_bins) * series_words + (i % n_bins);
    uint32_t carry = 0;
    for (uint64_t k = 0; k < n_ticks; ++k) {
        carry += r[k * n_bins];
        r[k * n_bins] = carry;
    }
}

// replicas whose pools overflowed in the thread-per-replica pass -> list for the warp-per-replica pass
__global__ void af_flagged_kernel(const AfReplicaStats* __restrict__ stats, uint64_t n, uint32_t mask,
                                  uint32_t* __restrict__ list, uint32_t* __restrict__ count) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (stats[i].flags & mask)) list[atomicAdd(count, 1u)] = (uint32_t)i;
}

// ---- pull order ------------------------------------------------------------------------------------------------
// A lane runs replicas back to back, and the launch ends when its last lane does.  Pulled in id order, the heaviest
// replicas of a sweep tend to come last and the launch ends on a few busy lanes; the simulation kernels therefore pull
// local indices through an order: heaviest first by each replica's predicted work (DESIGN.md §3.3).  Which lane runs a
// replica, and when, changes no result: its random numbers are keyed by its replica id, its outputs by its local index.
struct OrderArgs {
    const AfSweepColumn* cols; const double* vals; int32_t n_cols; uint64_t sweep_first, sweep_rows;
    const int32_t* row_need; int32_t need;     // per-row pending-events estimates (nullptr: `need` for every replica)
    uint64_t seed, begin, n;
    int32_t users_dist; double users_mean, users_sigma, rate_per_user, span;   // span: the first window, at most the horizon
};

// the replica's pending-events estimate: its row's, else the scenario's
__device__ __forceinline__ int32_t order_need(const OrderArgs& a, uint64_t i) {
    const uint64_t r = a.begin + i - a.sweep_first;
    return a.row_need != nullptr && r < a.sweep_rows ? a.row_need[r] : a.need;
}

// Predicted work of a replica: the requests of its first window -- the users it draws at t = 0 (the same draw its
// generator makes) x rate x window -- times the per-event cost of its load, which grows with the events it keeps
// pending (measured: DESIGN.md §3.3).  Non-negative floats: the bits sort as the values.
__global__ void af_order_key_kernel(const OrderArgs a, uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const uint64_t replica = a.begin + i, r = replica - a.sweep_first;
    double um = a.users_mean, us = a.users_sigma, rate = a.rate_per_user;
    if (r < a.sweep_rows)
        for (int32_t c = 0; c < a.n_cols; ++c) afl::gen_field(a.cols[c].field, a.vals[r * (uint64_t)a.n_cols + (uint64_t)c], um, us, rate);
    const double users = afr::gen_users(a.seed, replica, 0u, a.users_dist, um, us).value;
    const double cost = users * rate * a.span * (AF_ORDER_EVENT_COST + (double)order_need(a, i));
    key[i] = cost > 0.0 ? __float_as_uint((float)cost) : 0u;
    idx[i] = (uint32_t)i;
}

// The first wave (the heaviest `lanes` replicas) again, grouped by estimate, then by work: the 32 lanes of a warp start
// replicas with the same split of the pool and similar loads.  key64 = estimate : work.
__global__ void af_order_group_kernel(const OrderArgs a, const uint32_t* __restrict__ key, const uint32_t* __restrict__ order,
                                      uint64_t lanes, uint64_t* __restrict__ key64, uint32_t* __restrict__ idx) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= lanes) return;
    const uint32_t i = order[j];
    key64[j] = ((uint64_t)(uint32_t)order_need(a, i) << 32) | key[j];
    idx[j] = i;
}

// AF-RNG on the device, outside the state machine: what tests/test_gpu_rng.py compares with oracle/afrng_c
// (kind: see af_selftest_rng in the header)
__global__ void af_selftest_rng_kernel(uint64_t seed, uint64_t replica, int kind, int dist, double mean, double sigma,
                                       uint32_t hop, uint64_t n, double* __restrict__ a, double* __restrict__ b) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (kind == AF_SELFTEST_EDGE) {
        const afr::EdgeDraw d = afr::edge_draw(seed, replica, (uint32_t)i + 1u, hop, dist, mean, sigma, 0.0);
        a[i] = d.u; b[i] = d.transit;
    } else if (kind == AF_SELFTEST_GEN_UNIFORM) {
        afr::Src s = afr::make_gen(seed, replica, (uint32_t)i);
        double u = s.next53();
        a[i] = u;
        if (u < 1e-15) u = 1e-15;
        b[i] = -afr::af_log(1.0 - u);
    } else if (kind == AF_SELFTEST_GEN_USERS) {
        const afr::GenDraw g = afr::gen_users(seed, replica + i, 0u, dist, mean, sigma);
        a[i] = g.value; b[i] = (double)g.pos;
    } else if (kind == AF_SELFTEST_ENDPOINT) {
        afr::Src src = afr::make_request(seed, replica, afr::P_SERVER, (uint32_t)i + 1u, hop);
        src.load(0);
        a[i] = (double)(uint32_t)(((uint64_t)src.w.x * (uint32_t)dist) >> 32); b[i] = 0.0;
    } else if (kind == AF_SELFTEST_LOG) {
        const double x = afr::u2d(afr::d2u(mean) + i * (uint64_t)sigma);
        a[i] = x; b[i] = afr::af_log(x);
    } else {
        const double x = mean + (double)i * sigma;
        a[i] = x; b[i] = afr::af_exp(x);
    }
}

// value of order statistic `rank` given the bin that holds it.  The two end bins also hold every latency the histogram
// clamps into them, so they reach out to the replica's exact extremes (afh::hist_order_stat).
__device__ __forceinline__ double af_bin_value(int bin, uint64_t rank, uint64_t cum_before, uint32_t cnt,
                                               double lat_min, double lat_max) {
    const long long base = (long long)((1023 + AF_HIST_MIN_EXP) << AF_HIST_SUB_BITS);
    double lo = __longlong_as_double(((long long)bin + base) << (52 - AF_HIST_SUB_BITS));
    double hi = __longlong_as_double(((long long)bin + 1 + base) << (52 - AF_HIST_SUB_BITS));
    if (bin == 0 && lat_min < lo) lo = lat_min;
    if (bin == AF_HIST_BINS - 1 && lat_max > hi) hi = lat_max;
    double frac = ((double)(rank - cum_before) + 0.5) / (double)cnt;
    return lo + frac * (hi - lo);
}

__global__ void af_percentile_kernel(const uint32_t* __restrict__ hist, AfReplicaStats* __restrict__ stats,
                                     uint64_t n_replicas) {
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = (int)(threadIdx.x & 31u);
    if (warp >= n_replicas) return;
    const uint32_t* row = hist + warp * AF_HIST_BINS;
    const uint64_t n = stats[warp].completed;
    const double lat_min = stats[warp].lat_min, lat_max = stats[warp].lat_max;
    // target order statistics (numpy linear interpolation between two neighbours)
    const double qs[3] = {50.0, 95.0, 99.0};
    uint64_t rank[6]; double frac[3]; double val[6];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        double pos = n ? qs[i] / 100.0 * (double)(n - 1) : 0.0;
        uint64_t lo = (uint64_t)floor(pos);
        frac[i] = pos - (double)lo;
        rank[2 * i] = lo;
        rank[2 * i + 1] = (lo + 1 < n) ? lo + 1 : lo;
        val[2 * i] = val[2 * i + 1] = 0.0;
    }
    uint64_t carry = 0;
    for (int base = 0; base < AF_HIST_BINS; base += 32) {
        uint32_t c = row[base + lane];                 // one coalesced 128-byte read per warp
        uint32_t incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += up;
        }
        uint64_t before = carry + (incl - c);
#pragma unroll
        for (int i = 0; i < 6; ++i)
            if (c && rank[i] >= before && rank[i] < before + c) val[i] = af_bin_value(base + lane, rank[i], before, c, lat_min, lat_max);
        carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    // each target was found by exactly one lane: sum-reduce to share it
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double v = val[i];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
        val[i] = v;
    }
    if (lane == 0) {
        const double nan = __longlong_as_double(0x7FF8000000000000ll);
        double p[3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
            p[i] = n ? ((frac[i] == 0.0 || rank[2 * i + 1] == rank[2 * i]) ? val[2 * i]
                                                                            : val[2 * i] + frac[i] * (val[2 * i + 1] - val[2 * i]))
                     : nan;
        stats[warp].p50 = p[0]; stats[warp].p95 = p[1]; stats[warp].p99 = p[2];
    }
}


// Sum the per-replica latency histograms into one [AF_HIST_BINS] u64 histogram (the summary
// block a rank contributes to the end-of-sweep NCCL all-gather).  HBM-bound: each block walks
// a strip of replicas, a thread owns bins t, t+256, ... so every row read is coalesced.
__global__ void af_hist_reduce_kernel(const uint32_t* __restrict__ hist, unsigned long long* __restrict__ total,
                                      uint64_t n_replicas, uint64_t rows_per_block) {
    uint64_t r0 = (uint64_t)blockIdx.x * rows_per_block;
    uint64_t r1 = r0 + rows_per_block < n_replicas ? r0 + rows_per_block : n_replicas;
    unsigned long long acc[AF_HIST_BINS / 256];
#pragma unroll
    for (int j = 0; j < AF_HIST_BINS / 256; ++j) acc[j] = 0;
    for (uint64_t r = r0; r < r1; ++r) {
        const uint32_t* row = hist + r * AF_HIST_BINS;
#pragma unroll
        for (int j = 0; j < AF_HIST_BINS / 256; ++j) acc[j] += row[j * 256 + threadIdx.x];
    }
#pragma unroll
    for (int j = 0; j < AF_HIST_BINS / 256; ++j)
        if (acc[j]) atomicAdd(&total[j * 256 + threadIdx.x], acc[j]);
}

// ---------------------------------------------------------------------------------
// engine
// ---------------------------------------------------------------------------------
namespace {

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

thread_local std::string g_create_error;

// The launch parameters live in __constant__ memory, which is per device, not per engine: a
// second engine on the same device must not overwrite them while the first one's kernel runs.
constexpr int kMaxDevices = 64;
std::mutex g_const_mutex;
af_engine* g_const_owner[kMaxDevices] = {};

}  // namespace

struct af_engine {
    int device = 0;
    int sm_count = 0;
    int max_smem_optin = 0;
    uint64_t mem_total = 0;     // device memory: the bound on what the band rows may ask for
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_begin = nullptr, ev_sim = nullptr, ev_end = nullptr;
    std::string err;
    AfOptions opt{};
    bool have_scenario = false;
    AfScenario sc{};            // host copy; pointers repointed at the vectors below
    std::vector<AfEdge> h_edges; std::vector<AfServer> h_servers; std::vector<AfEndpoint> h_eps;
    std::vector<AfStep> h_steps; std::vector<int32_t> h_lb; std::vector<AfSpikeMark> h_spikes;
    std::vector<AfOutageMark> h_outages;
    DevBuf d_edges, d_servers, d_eps, d_steps, d_lb, d_spikes, d_outages;
    // sweep
    int32_t sweep_cols = 0; uint64_t sweep_rows = 0, sweep_first = 0;
    std::vector<AfSweepColumn> h_sweep_cols;
    std::vector<int32_t> h_sweep_alias;            // aflh::column_aliases of the uploaded values
    int32_t ev_need = 0;                           // aflh::pending_events_estimate of the scenario (replicas without a row)
    std::vector<int32_t> h_row_need;               // aflh::row_events_estimates of the sweep's rows ...
    int32_t row_need_max = 0;                      // ... and the largest of them
    DevBuf d_sweep_cols, d_sweep_vals, d_row_need;
    // thread-per-replica pass: read-only tables (af_lane_host.h), global tiers, the list of flagged replicas
    int mode = AF_MODE_AUTO;
    aflh::Tables lt;
    DevBuf d_l_edges, d_l_servers, d_l_eps, d_l_steps, d_l_spikes, d_l_outages, d_l_lb, d_l_cols, d_gtier, d_redo_list, d_redo_count, d_counter2;
    afl::Cfg C_host{};
    int32_t last_ev_s = 0, last_rq_s = 0;          // the pool split of the launch's heaviest replica (AfRunPasses)
    bool last_lane = false, last_warp = false, last_lean = false; int last_lane_warps = 0;
    // spill + outputs
    DevBuf d_sp_evt, d_sp_evk, d_sp_rq, d_sp_nx;
    DevBuf d_okey, d_oidx, d_order, d_okey64, d_sort_tmp;     // pull order (af_order_*_kernel + radix sorts)
    DevBuf d_stats, d_sent, d_dropped, d_hist, d_thr, d_ssum, d_smax, d_tclk, d_tser, d_tcnt, d_counter, d_htot;
    // last run
    uint64_t last_n = 0; bool ran = false;
    afc::Layout L{};
    afc::Globals G_host{};
    uint64_t launches = 0;
    float ms_total = 0.f, ms_sim = 0.f; bool timing_valid = false;
    // per-tick bands (af_bands_upload): group of replica band_first + i, n_groups groups (0: bands off); the difference
    // rows of n_groups + 1 groups (the last: replicas without a group entry), the tick each flagged replica stopped at
    std::vector<uint32_t> h_band_group; uint64_t band_first = 0; uint32_t band_groups = 0;
    DevBuf d_band_group, d_band, d_band_from;
    uint64_t band_swept_ram = 0; int32_t band_swept_server = -1;     // afh::swept_ram_max of the uploaded sweep
    bool last_bands = false; uint32_t last_band_groups = 0, last_band_ticks = 0; uint64_t last_band_stride = 0;
    // af_bands_configure: per-tick bands on (default) / off; per-window latency bands of lat_window seconds (0: off) --
    // their rows, the completions each flagged replica added in the thread-per-replica pass
    int32_t band_sampled = 1, lat_window = 0;
    DevBuf d_lat, d_lat_from;
    bool last_lat = false; uint32_t last_lat_groups = 0; uint64_t last_lat_windows = 0;
    // af_dist_bands_configure: the selected series (empty: per-tick distribution bands off), af_run's table of each
    // series' slot (-1: not selected) and the rows over the groups of af_bands_upload
    std::vector<int32_t> h_dist_series, h_dist_slot;
    DevBuf d_dist_slot, d_dist;
    bool last_dist = false; uint32_t last_dist_groups = 0, last_dist_ticks = 0, last_dist_bins = 0, last_dist_n = 0;
    uint64_t last_dist_series_words = 0;
    // af_occupancy_configure: on / off and f; the [n][occ_cols] rows of the last run
    AfOccupancyOptions occ_opt{0, 32};
    DevBuf d_occ;
    bool last_occ = false; int32_t last_occ_bits = 0, last_occ_cols = 0;

    int fail(int code, const std::string& m) { err = m; return code; }
    int cuda_fail(cudaError_t e, const char* what) {
        err = std::string(what) + ": " + cudaGetErrorString(e);
        return AF_ERR_CUDA;
    }
};

#define AF_CUDA(e_, call, what) do { cudaError_t _c = (call); if (_c != cudaSuccess) return (e_)->cuda_fail(_c, what); } while (0)

template <class T>
static int upload_vec(af_engine* e, DevBuf& d, const std::vector<T>& h, const char* what) {
    AF_CUDA(e, d.ensure(h.size() * sizeof(T)), what);
    if (!h.empty()) AF_CUDA(e, cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, e->stream), what);
    return AF_OK;
}

// the instantiation of af_lane_kernel for a launch's bands, build and occupancy
template <bool S, bool L, bool Lean, bool D>
static void (*lane_kernel_for(bool occ))() { return occ ? af_lane_kernel<S, L, Lean, D, true> : af_lane_kernel<S, L, Lean, D, false>; }
template <bool S, bool L>
static void (*lane_kernel_for(bool lean, bool dist, bool occ))() {
    return lean ? (dist ? lane_kernel_for<S, L, true, true>(occ) : lane_kernel_for<S, L, true, false>(occ))
                : (dist ? lane_kernel_for<S, L, false, true>(occ) : lane_kernel_for<S, L, false, false>(occ));
}

extern "C" {

int af_abi_version(void) { return AF_ABI_VERSION; }

const char* af_last_error(const af_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int af_engine_create(int device, af_engine** out) {
    if (!out) { g_create_error = "out is NULL"; return AF_ERR_INVALID; }
    *out = nullptr;
    int n = 0;
    cudaError_t ce = cudaGetDeviceCount(&n);
    if (ce != cudaSuccess || n == 0) {
        g_create_error = std::string("no CUDA device: ") + (ce != cudaSuccess ? cudaGetErrorString(ce) : "count is 0")
                         + " (asyncflow_b200 has no CPU fallback)";
        return AF_ERR_CUDA;
    }
    if (device < 0 || device >= n) { g_create_error = "device index out of range"; return AF_ERR_INVALID; }
    cudaDeviceProp prop;
    if ((ce = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) { g_create_error = cudaGetErrorString(ce); return AF_ERR_CUDA; }
    if (prop.major != 9 || prop.minor != 0) {
        char b[160]; snprintf(b, sizeof b, "device %d is sm_%d%d; this library carries sm_90a code only", device, prop.major, prop.minor);
        g_create_error = b; return AF_ERR_CUDA;
    }
    af_engine* e = new (std::nothrow) af_engine();
    if (!e) { g_create_error = "host allocation failed"; return AF_ERR_NOMEM; }
    e->device = device; e->sm_count = prop.multiProcessorCount; e->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    e->mem_total = (uint64_t)prop.totalGlobalMem;
    if ((ce = cudaSetDevice(device)) != cudaSuccess || (ce = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess
        || (ce = cudaEventCreate(&e->ev_begin)) != cudaSuccess || (ce = cudaEventCreate(&e->ev_sim)) != cudaSuccess
        || (ce = cudaEventCreate(&e->ev_end)) != cudaSuccess) {
        g_create_error = cudaGetErrorString(ce); delete e; return AF_ERR_CUDA;
    }
    e->opt.collect_histogram = 1; e->opt.collect_throughput = 1;
    if (const char* m = getenv("ASYNCFLOW_B200_ENGINE")) {      // kernel experiments: pin the pass structure
        if (!strcmp(m, "warp")) e->mode = AF_MODE_WARP; else if (!strcmp(m, "lane")) e->mode = AF_MODE_LANE;
        else if (!strcmp(m, "two_pass")) e->mode = AF_MODE_TWO_PASS;
    }
    *out = e;
    return AF_OK;
}

void af_engine_destroy(af_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    {
        std::lock_guard<std::mutex> lock(g_const_mutex);
        if (g_const_owner[e->device % kMaxDevices] == e) g_const_owner[e->device % kMaxDevices] = nullptr;
    }
    DevBuf* bufs[] = {&e->d_l_edges, &e->d_l_servers, &e->d_l_eps, &e->d_l_steps, &e->d_l_spikes, &e->d_l_outages, &e->d_l_lb, &e->d_l_cols,
                      &e->d_gtier, &e->d_redo_list, &e->d_redo_count, &e->d_counter2,
                      &e->d_edges, &e->d_servers, &e->d_eps, &e->d_steps, &e->d_lb, &e->d_spikes, &e->d_outages,
                      &e->d_sweep_cols, &e->d_sweep_vals, &e->d_row_need, &e->d_sp_evt, &e->d_sp_evk, &e->d_sp_rq, &e->d_sp_nx,
                      &e->d_stats, &e->d_sent, &e->d_dropped, &e->d_hist, &e->d_thr, &e->d_ssum, &e->d_smax,
                      &e->d_tclk, &e->d_tser, &e->d_tcnt, &e->d_counter, &e->d_htot,
                      &e->d_okey, &e->d_oidx, &e->d_order, &e->d_okey64, &e->d_sort_tmp,
                      &e->d_band_group, &e->d_band, &e->d_band_from, &e->d_lat, &e->d_lat_from,
                      &e->d_dist_slot, &e->d_dist, &e->d_occ};
    for (DevBuf* b : bufs) b->release();
    cudaEventDestroy(e->ev_begin); cudaEventDestroy(e->ev_sim); cudaEventDestroy(e->ev_end);
    cudaStreamDestroy(e->stream);
    delete e;
}

int af_engine_configure(af_engine* e, const AfOptions* opt) {
    if (!e || !opt) return AF_ERR_INVALID;
    if (opt->event_capacity < 0 || opt->request_capacity < 0 || opt->warps_per_block < 0 || opt->warps_per_block > 32 || opt->blocks_per_sm < 0
        || opt->trace_replicas < 0 || opt->trace_clock_capacity < 0)
        return e->fail(AF_ERR_INVALID, "AfOptions: negative or out-of-range field");
    e->opt = *opt;
    return AF_OK;
}

int af_scenario_upload(af_engine* e, const AfScenario* s) {
    if (!e || !s) return AF_ERR_INVALID;
    std::string why;
    if (!afh::validate(*s, why)) return e->fail(AF_ERR_INVALID, "scenario: " + why);
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    // wait for any run still reading the old tables
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "sync before upload");
    e->sc = *s;
    e->h_edges.assign(s->edges, s->edges + s->n_edges);
    e->h_servers.assign(s->servers, s->servers + s->n_servers);
    e->h_eps.assign(s->endpoints, s->endpoints + s->n_endpoints);
    e->h_steps.assign(s->steps, s->steps + s->n_steps);
    e->h_lb.assign(s->lb_edges, s->lb_edges + s->n_lb_edges);
    e->h_spikes.assign(s->spike_marks, s->spike_marks + s->n_spike_marks);
    e->h_outages.assign(s->outage_marks, s->outage_marks + s->n_outage_marks);
    int rc;
    if ((rc = upload_vec(e, e->d_edges, e->h_edges, "edges"))) return rc;
    if ((rc = upload_vec(e, e->d_servers, e->h_servers, "servers"))) return rc;
    if ((rc = upload_vec(e, e->d_eps, e->h_eps, "endpoints"))) return rc;
    if ((rc = upload_vec(e, e->d_steps, e->h_steps, "steps"))) return rc;
    if ((rc = upload_vec(e, e->d_lb, e->h_lb, "lb_edges"))) return rc;
    if ((rc = upload_vec(e, e->d_spikes, e->h_spikes, "spike_marks"))) return rc;
    if ((rc = upload_vec(e, e->d_outages, e->h_outages, "outage_marks"))) return rc;
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "scenario upload");
    e->sc.edges = e->h_edges.data(); e->sc.servers = e->h_servers.data(); e->sc.endpoints = e->h_eps.data();
    e->sc.steps = e->h_steps.data(); e->sc.lb_edges = e->h_lb.data(); e->sc.spike_marks = e->h_spikes.data();
    e->sc.outage_marks = e->h_outages.data();
    e->have_scenario = true;
    e->sweep_cols = 0; e->sweep_rows = 0; e->h_sweep_cols.clear();     // a sweep belongs to the scenario it was built for
    e->ev_need = aflh::pending_events_estimate(e->sc, nullptr); e->row_need_max = 0;
    e->band_swept_ram = 0; e->band_swept_server = -1;
    e->ran = false;
    return AF_OK;
}

int af_sweep_upload(af_engine* e, const AfSweep* sw, uint64_t first_replica) {
    if (!e) return AF_ERR_INVALID;
    if (!e->have_scenario) return e->fail(AF_ERR_STATE, "af_sweep_upload before af_scenario_upload");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "sync before sweep upload");
    if (!sw || sw->n_columns == 0 || sw->n_rows == 0) {
        e->sweep_cols = 0; e->sweep_rows = 0; e->h_sweep_cols.clear(); e->row_need_max = 0; e->band_swept_ram = 0; e->band_swept_server = -1;
        return AF_OK;
    }
    if (!sw->columns || !sw->values) return e->fail(AF_ERR_INVALID, "sweep: null columns/values");
    const AfScenario& s = e->sc;
    for (int c = 0; c < sw->n_columns; ++c) {
        int f = sw->columns[c].field, i = sw->columns[c].index, lim = 1;
        switch (f) {
        case AF_FIELD_USERS_MEAN: case AF_FIELD_USERS_SIGMA: case AF_FIELD_RATE_PER_USER: lim = 1; break;
        case AF_FIELD_EDGE_MEAN: case AF_FIELD_EDGE_SIGMA: case AF_FIELD_EDGE_DROPOUT: lim = s.n_edges; break;
        case AF_FIELD_SERVER_CPU_CORES: case AF_FIELD_SERVER_RAM_MB: lim = s.n_servers; break;
        case AF_FIELD_STEP_DURATION: lim = s.n_steps; break;
        case AF_FIELD_ENDPOINT_RAM: lim = s.n_endpoints; break;
        case AF_FIELD_SPIKE_DELTA: lim = s.n_spike_marks; break;
        default: return e->fail(AF_ERR_INVALID, "sweep: unknown field id");
        }
        if (i < 0 || i >= lim) return e->fail(AF_ERR_INVALID, "sweep: column index out of range");
    }
    // the values get the checks afh::validate applies to the base scenario (a swept cpu_cores of 0 would queue forever)
    for (uint64_t r = 0; r < sw->n_rows; ++r)
        for (int c = 0; c < sw->n_columns; ++c) {
            const double v = sw->values[r * (uint64_t)sw->n_columns + (uint64_t)c];
            bool ok = v == v && v - v == 0.0;                     // finite
            switch (sw->columns[c].field) {
            case AF_FIELD_EDGE_DROPOUT: ok = ok && v >= 0.0 && v <= 1.0; break;
            case AF_FIELD_SERVER_CPU_CORES: case AF_FIELD_SERVER_RAM_MB: ok = ok && v >= 1.0 && v <= 2147483647.0; break;
            case AF_FIELD_ENDPOINT_RAM: ok = ok && v >= 0.0 && v <= 2147483647.0; break;
            case AF_FIELD_EDGE_MEAN: {
                const int d = s.edges[sw->columns[c].index].dist;
                ok = ok && (v >= 0.0 || d == AF_DIST_LOG_NORMAL || d == AF_DIST_NORMAL);
                if (ok && d == AF_DIST_POISSON && v > afr::EDGE_POISSON_MEAN_MAX) {
                    char b[200]; snprintf(b, sizeof b, "sweep: row %llu column %d: edge %d's Poisson mean %g above %g, the "
                                          "largest a request's random-number blocks cover", (unsigned long long)r, c,
                                          sw->columns[c].index, v, afr::EDGE_POISSON_MEAN_MAX);
                    return e->fail(AF_ERR_INVALID, b);
                }
                break;
            }
            case AF_FIELD_USERS_SIGMA: ok = ok && v >= 0.0 && s.users_dist == AF_DIST_NORMAL; break;
            default: ok = ok && v >= 0.0; break;            // users, rates, sigmas, durations, spike amplitudes
            }
            if (!ok) {
                char b[200]; snprintf(b, sizeof b, "sweep: row %llu column %d (field %d, index %d): value %g out of range",
                                      (unsigned long long)r, c, sw->columns[c].field, sw->columns[c].index, v);
                return e->fail(AF_ERR_INVALID, b);
            }
        }
    e->h_sweep_cols.assign(sw->columns, sw->columns + sw->n_columns);
    e->h_sweep_alias = aflh::column_aliases(sw->values, sw->n_rows, sw->n_columns);
    // each row's own pending-events estimate: the lane kernel splits the replica's shared-memory pool by it.  On the
    // host, here: one pass over the values (as the checks above), and the kernel's start of a replica stays one load
    e->row_need_max = aflh::row_events_estimates(e->sc, *sw, e->h_row_need);
    e->band_swept_ram = afh::swept_ram_max(sw->columns, sw->n_columns, sw->values, sw->n_rows, e->band_swept_server);
    size_t cb = (size_t)sw->n_columns * sizeof(AfSweepColumn), vb = (size_t)sw->n_columns * sw->n_rows * sizeof(double);
    AF_CUDA(e, e->d_sweep_cols.ensure(cb), "sweep columns");
    AF_CUDA(e, e->d_sweep_vals.ensure(vb), "sweep values");
    AF_CUDA(e, e->d_row_need.ensure(sw->n_rows * sizeof(int32_t)), "sweep row estimates");
    AF_CUDA(e, cudaMemcpyAsync(e->d_sweep_cols.p, sw->columns, cb, cudaMemcpyHostToDevice, e->stream), "sweep columns H2D");
    AF_CUDA(e, cudaMemcpyAsync(e->d_sweep_vals.p, sw->values, vb, cudaMemcpyHostToDevice, e->stream), "sweep values H2D");
    AF_CUDA(e, cudaMemcpyAsync(e->d_row_need.p, e->h_row_need.data(), sw->n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream),
            "sweep row estimates H2D");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "sweep upload");
    e->sweep_cols = sw->n_columns; e->sweep_rows = sw->n_rows; e->sweep_first = first_replica;
    return AF_OK;
}

// sumsq of the per-tick bands is a u64 sum of squares: refuse a group size and gauge bound that could wrap it
static int band_check(af_engine* e, uint64_t group) {
    std::string what;
    const uint64_t bound = afh::band_gauge_bound(e->sc, e->opt, e->band_swept_ram, e->band_swept_server, what);
    if (afh::band_sumsq_fits(group, bound)) return AF_OK;
    char b[320];
    snprintf(b, sizeof b, "bands: a group of %llu replicas x (%llu, the bound on a gauge: %s)^2 could wrap the u64 sum of squares; "
             "use smaller groups", (unsigned long long)group, (unsigned long long)bound, what.c_str());
    return e->fail(AF_ERR_INVALID, b);
}

// The band rows of `n_groups` groups for the current scenario: every tick a replica can take needs its word (the kernels
// index the rows by the tick count, unchecked), and the rows must fit the device.  ticks = the scenario's tick count.
static int band_shape_check(af_engine* e, uint64_t n_groups, uint32_t& ticks) {
    std::string why;
    if (!afh::band_ticks_fit(e->sc, ticks, why)) return e->fail(AF_ERR_INVALID, why);
    const unsigned __int128 bytes = afh::band_row_bytes(n_groups, 3 * e->sc.n_servers + e->sc.n_edges, ticks);
    if (bytes > (unsigned __int128)e->mem_total) {
        char b[240];
        snprintf(b, sizeof b, "bands: %llu groups x %u ticks need %.3g GB of band rows, more than the device's %.3g GB",
                 (unsigned long long)n_groups, ticks, (double)bytes / 1e9, (double)e->mem_total / 1e9);
        return e->fail(AF_ERR_INVALID, b);
    }
    return AF_OK;
}

// the most replicas one group holds among group_of[0 .. n)
static uint64_t largest_group(const uint32_t* group_of, uint64_t n) {
    std::vector<uint32_t> g(group_of, group_of + n);
    std::sort(g.begin(), g.end());
    uint64_t best = 0;
    for (uint64_t i = 0, j; i < n; i = j) {
        for (j = i + 1; j < n && g[j] == g[i]; ++j) {}
        best = j - i > best ? j - i : best;
    }
    return best;
}

// the latency bands' window and rows for `n_groups` groups of the current scenario (afh::lat_bands_fit)
static int lat_check(af_engine* e, uint64_t n_groups) {
    std::string why;
    if (!afh::lat_bands_fit(e->lat_window, e->sc.horizon_s, n_groups, e->mem_total, why)) return e->fail(AF_ERR_INVALID, why);
    return AF_OK;
}

// the distribution bands' series and rows for `n_groups` groups of the current scenario, options and sweep
// (afh::dist_series_check, afh::dist_bands_fit); sets the tick count and bins per tick row
static int dist_check(af_engine* e, uint64_t n_groups, uint32_t& ticks, uint32_t& bins) {
    std::string why;
    if (!afh::dist_series_check(e->sc, e->h_dist_series.data(), (int32_t)e->h_dist_series.size(), why)
        || !afh::dist_bands_fit(e->sc, e->opt, e->band_swept_ram, e->band_swept_server, n_groups, e->h_dist_series.size(),
                                e->mem_total, ticks, bins, why))
        return e->fail(AF_ERR_INVALID, why);
    return AF_OK;
}

int af_dist_bands_configure(af_engine* e, const int32_t* series, int32_t n) {
    if (!e) return AF_ERR_INVALID;
    if (n < 0) return e->fail(AF_ERR_INVALID, "distribution bands: negative series count");
    if (!series || n == 0) { e->h_dist_series.clear(); return AF_OK; }
    if (!e->have_scenario) return e->fail(AF_ERR_STATE, "af_dist_bands_configure before af_scenario_upload");
    std::vector<int32_t> old;
    old.swap(e->h_dist_series);
    e->h_dist_series.assign(series, series + n);
    uint32_t ticks = 0, bins = 0;
    std::string why;
    int rc = AF_OK;
    if (!afh::dist_series_check(e->sc, series, n, why)) rc = e->fail(AF_ERR_INVALID, why);
    else if (e->band_groups > 0) rc = dist_check(e, e->band_groups, ticks, bins);     // the uploaded groups
    if (rc) e->h_dist_series.swap(old);
    return rc;
}

int af_occupancy_configure(af_engine* e, const AfOccupancyOptions* opt) {
    if (!e || !opt) return AF_ERR_INVALID;
    if (opt->on && (opt->frac_bits < 8 || opt->frac_bits > 32)) {
        char b[160]; snprintf(b, sizeof b, "occupancy: %d fraction bits; 8 to 32 are supported", opt->frac_bits);
        return e->fail(AF_ERR_INVALID, b);
    }
    e->occ_opt = *opt;
    e->occ_opt.on = opt->on != 0;
    return AF_OK;
}

int af_bands_configure(af_engine* e, const AfBandOptions* opt) {
    if (!e || !opt) return AF_ERR_INVALID;
    if (opt->latency_window_s != 0) {
        std::string why;
        if (!afh::lat_bands_fit(opt->latency_window_s, 0, 0, e->mem_total, why)) return e->fail(AF_ERR_INVALID, why);
    }
    const int32_t sampled = e->band_sampled, window = e->lat_window;
    e->band_sampled = opt->sampled != 0; e->lat_window = opt->latency_window_s;
    int rc = AF_OK;
    if (e->have_scenario && e->band_groups > 0) {        // the uploaded groups, under the new options
        uint32_t ticks = 0;
        if (e->band_sampled && !(rc = band_shape_check(e, e->band_groups, ticks)))
            rc = band_check(e, largest_group(e->h_band_group.data(), e->h_band_group.size()));
        if (!rc && e->lat_window) rc = lat_check(e, e->band_groups);
    }
    if (rc) { e->band_sampled = sampled; e->lat_window = window; }
    return rc;
}

int af_bands_upload(af_engine* e, const uint32_t* group_of, uint64_t n, uint64_t first_replica, uint32_t n_groups) {
    if (!e) return AF_ERR_INVALID;
    if (!e->have_scenario) return e->fail(AF_ERR_STATE, "af_bands_upload before af_scenario_upload");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "sync before bands upload");
    if (!group_of) { e->band_groups = 0; e->h_band_group.clear(); return AF_OK; }
    if (n == 0 || n_groups == 0) return e->fail(AF_ERR_INVALID, "bands: empty group table or n_groups == 0");
    for (uint64_t i = 0; i < n; ++i)
        if (group_of[i] >= n_groups) {
            char b[160]; snprintf(b, sizeof b, "bands: group_of[%llu] = %u is not < n_groups = %u", (unsigned long long)i, group_of[i], n_groups);
            return e->fail(AF_ERR_INVALID, b);
        }
    uint32_t ticks = 0;
    int rc;
    if (e->band_sampled) {
        if ((rc = band_shape_check(e, n_groups, ticks))) return rc;
        if ((rc = band_check(e, largest_group(group_of, n)))) return rc;
    }
    if (e->lat_window && (rc = lat_check(e, n_groups))) return rc;
    uint32_t bins = 0;
    if (!e->h_dist_series.empty() && (rc = dist_check(e, n_groups, ticks, bins))) return rc;
    e->h_band_group.assign(group_of, group_of + n);
    if ((rc = upload_vec(e, e->d_band_group, e->h_band_group, "band groups"))) return rc;
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "band groups H2D");
    e->band_first = first_replica; e->band_groups = n_groups;
    return AF_OK;
}

// shared-memory budget of one lane when the CTA has `warps` warps (one CTA per SM)
static int32_t lane_budget(const af_engine* e, int warps) {
    int32_t b = (int32_t)((e->max_smem_optin / (warps * 32)) & ~3);
    if (const char* cap = getenv("ASYNCFLOW_B200_LANE_BYTES")) { const int32_t c = atoi(cap) & ~3; if (c > 0 && c < b) b = c; }   // experiments: leave more of the SM's 256 KB to L1
    return b;
}

int af_run(af_engine* e, uint64_t seed, uint64_t begin, uint64_t end) {
    if (!e) return AF_ERR_INVALID;
    if (!e->have_scenario) return e->fail(AF_ERR_STATE, "af_run before af_scenario_upload");
    if (end <= begin) return e->fail(AF_ERR_INVALID, "af_run: empty replica range");
    if (end - begin > 0xFFFFFFFFull) return e->fail(AF_ERR_INVALID, "af_run: more than 2^32 replicas in one call");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    const uint64_t n = end - begin;
    int rc;

    // ---- pass structure ---------------------------------------------------------------------------------
    // AUTO: every replica runs on the thread-per-replica engine with tiers sized for nominal load; the ones
    // it flags (pool overflow) are re-run by the warp-per-replica engine with the caller's capacities.
    bool lane = e->mode != AF_MODE_WARP;
    afl::Cfg& C = e->C_host;
    int lane_warps = 0;
    if (lane) {
        std::string why;
        // columns that repeat an earlier column share its slot -- only when every replica of this run has a sweep row
        // (a replica outside the sweep takes each column's own base value)
        const bool all_rows = e->sweep_cols > 0 && begin >= e->sweep_first && end - e->sweep_first <= e->sweep_rows;
        if (!aflh::build_tables(e->sc, e->h_sweep_cols.data(), e->sweep_cols, all_rows ? e->h_sweep_alias.data() : nullptr, e->lt, why)) {
            if (e->mode == AF_MODE_LANE) return e->fail(AF_ERR_INVALID, why);
            lane = false;
        }
    }
    AfOptions o = e->opt;
    if (lane) {
        if (e->mode == AF_MODE_AUTO || e->mode == AF_MODE_TWO_PASS) {   // nominal-load tiers per lane; anything larger escalates
            if (o.event_capacity <= 0 || o.event_capacity > aflh::LANE_EVENT_CAPACITY) o.event_capacity = aflh::LANE_EVENT_CAPACITY;
            if (o.request_capacity <= 0 || o.request_capacity > aflh::LANE_REQUEST_CAPACITY) o.request_capacity = aflh::LANE_REQUEST_CAPACITY;
        }
        lane_warps = e->opt.warps_per_block > 0 ? e->opt.warps_per_block : AF_LANE_DEFAULT_WARPS;
        if (lane_warps > AF_LANE_MAX_THREADS / 32) lane_warps = AF_LANE_MAX_THREADS / 32;
        // fewer warps per SM when the topology's fixed tables need a larger share of shared memory (dependent L2 round
        // trips to tables in the global tier cost more than the occupancy buys)
        while (lane_warps > 1 && lane_budget(e, lane_warps) < aflh::min_lane_bytes(e->sc, e->lt) + 128)
            lane_warps -= lane_warps > 8 ? 4 : (lane_warps > 4 ? 2 : 1);
        // (a topology that leaves fewer than 4 warps per SM is faster on the warp-per-replica engine)
        if (e->mode == AF_MODE_AUTO && lane_warps < 4) lane = false;
        // A lane runs ONE replica about ten times slower than a warp does (it shares every instruction with 31 other
        // replicas): the thread-per-replica engine pays off when there are replicas for most lanes.
        if (e->mode == AF_MODE_AUTO && n < 3ull * (uint64_t)e->sm_count * 32ull) lane = false;
        if (lane && e->opt.warps_per_block <= 0) {
            // whole waves: with W warps per SM the launch takes ceil(n / lanes(W)) waves; the smallest W with that many
            // waves leaves each lane more shared memory and each warp more issue slots (100 000 replicas on 148 SMs: 11, not 12)
            const uint64_t per_warp = (uint64_t)e->sm_count * 32ull;
            const uint64_t waves = (n + per_warp * (uint64_t)lane_warps - 1) / (per_warp * (uint64_t)lane_warps);
            int w = (int)((n + waves * per_warp - 1) / (waves * per_warp));
            if (w < 4) w = 4;
            if (w < lane_warps) lane_warps = w;
        }
    }
    if (lane) {
        memset(&C, 0, sizeof C);
        // experiment knobs: every replica on the even split; the record slots the heap leaves
        const bool even = getenv("ASYNCFLOW_B200_EVEN_SPLIT") != nullptr;
        if (!aflh::make_cfg(e->sc, o, e->lt, lane_budget(e, lane_warps), afh::trace_tick_capacity(e->sc), 32, C, even ? 0 : e->ev_need,
                            getenv("ASYNCFLOW_B200_RQ_MIN") ? atoi(getenv("ASYNCFLOW_B200_RQ_MIN")) : 2)) {
            if (e->mode == AF_MODE_LANE) return e->fail(AF_ERR_INVALID, "scenario tables do not fit a lane's shared memory (thread-per-replica engine)");
            lane = false;
        } else {
            // the replicas with a sweep row split their pool by the row's estimate, the others by the scenario's
            const bool rows = !even && e->sweep_cols > 0;
            const bool all_rows = rows && begin >= e->sweep_first && end - e->sweep_first <= e->sweep_rows;
            int32_t heaviest = even ? 0 : (rows ? e->row_need_max : e->ev_need);
            if (rows && !all_rows && e->ev_need > heaviest) heaviest = e->ev_need;
            aflh::pool_split(C, heaviest, e->last_ev_s, e->last_rq_s);
            if (rows) { C.need_first = e->sweep_first; C.need_rows = e->sweep_rows; }
        }
    }
    const bool warp = e->mode != AF_MODE_LANE;
    const bool redo = lane && warp;

    afc::Layout& L = e->L;
    memset(&L, 0, sizeof L);
    afh::make_layout(e->sc, e->opt, e->sweep_cols, L);

    // ---- per-tick bands: difference rows of (groups + 1) x (1 + 2 n_series) x (ticks + 1) words -----------------------
    const bool bands = e->band_groups > 0 && e->band_sampled;
    uint32_t ticks32 = 0;
    if (bands) {      // (the scenario, options and sweep may have changed since af_bands_upload)
        if ((rc = band_shape_check(e, e->band_groups, ticks32))) return rc;
        const uint64_t lo = begin > e->band_first ? begin : e->band_first;          // this run's replicas with a group
        const uint64_t hi = end < e->band_first + e->h_band_group.size() ? end : e->band_first + e->h_band_group.size();
        if ((rc = band_check(e, lo < hi ? largest_group(e->h_band_group.data() + (lo - e->band_first), hi - lo) : 0))) return rc;
    }
    const uint64_t band_ticks = ticks32, band_stride = band_ticks + 1;
    const uint64_t band_group_words = (1 + 2 * (uint64_t)L.n_series) * band_stride;
    const uint64_t band_words = bands ? ((uint64_t)e->band_groups + 1) * band_group_words : 0;
    // ---- per-tick distribution bands: (groups + 1) x n_dist x (ticks + 1) x bins u32 -----------------------------------
    const bool dist = e->band_groups > 0 && !e->h_dist_series.empty();
    uint32_t dist_ticks = 0, dist_bins = 0;
    if (dist && (rc = dist_check(e, e->band_groups, dist_ticks, dist_bins))) return rc;
    const uint64_t dist_n = dist ? e->h_dist_series.size() : 0;
    const uint64_t dist_series_words = ((uint64_t)dist_ticks + 1) * dist_bins, dist_group_words = dist_n * dist_series_words;
    const uint64_t dist_words = dist ? ((uint64_t)e->band_groups + 1) * dist_group_words : 0;
    if (dist) {
        e->h_dist_slot.assign((size_t)L.n_series, -1);
        for (uint64_t s = 0; s < dist_n; ++s) e->h_dist_slot[(size_t)e->h_dist_series[s]] = (int32_t)s;
    }
    afc::BandArgs band = {};
    if (bands || dist) {
        band.prev_off = L.warp_bytes;                       // the warp engine: each series' last emitted value, behind its tables
        L.warp_bytes += afc::align_up(4 * L.n_series, 16);
    }
    // ---- per-window latency bands: (groups + 1) x windows x afr::LAT_ROW words ---------------------------------------------
    const bool lat = e->band_groups > 0 && e->lat_window > 0;
    if (lat && (rc = lat_check(e, e->band_groups))) return rc;
    const uint64_t lat_windows = lat ? afh::lat_windows(L.horizon_s, e->lat_window) : 0;
    const uint64_t lat_words = lat ? ((uint64_t)e->band_groups + 1) * lat_windows * afr::LAT_ROW : 0;
    // ---- occupancy integrals: n x occ_cols u64 ----------------------------------------------------------------------
    const bool occ = e->occ_opt.on != 0;
    const int32_t occ_cols = afh::occ_cols(e->sc);
    if (occ) {
        std::string why;
        if (!afh::occ_fits(e->sc, e->opt, e->band_swept_ram, e->band_swept_server, e->occ_opt.frac_bits, why))
            return e->fail(AF_ERR_INVALID, why);
    }

    // ---- launch shapes -------------------------------------------------------------------------------------
    // warp-per-replica: persistent CTAs of <= 4 warps (__launch_bounds__(128, AF_MIN_BLOCKS)), as many per SM as fit
    int wpb = 4; size_t smem = 0; uint64_t grid = 0, warp_slots = 0;
    if (warp) {
        if (!lane && e->opt.warps_per_block > 0 && e->opt.warps_per_block < 4) wpb = e->opt.warps_per_block;
        smem = (size_t)wpb * (size_t)L.warp_bytes;
        while (wpb > 1 && smem > (size_t)e->max_smem_optin) { --wpb; smem = (size_t)wpb * (size_t)L.warp_bytes; }
        if (smem > (size_t)e->max_smem_optin)
            return e->fail(AF_ERR_INVALID, "scenario tables do not fit in shared memory (one warp needs more than the 227 KB opt-in limit)");
        AF_CUDA(e, cudaFuncSetAttribute(af_sim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "smem attribute");
        int bps = 0;
        AF_CUDA(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, af_sim_kernel, wpb * 32, smem), "occupancy");
        if (bps < 1) return e->fail(AF_ERR_CUDA, "kernel cannot be resident (occupancy 0)");
        if (e->opt.blocks_per_sm > 0 && e->opt.blocks_per_sm < bps) bps = e->opt.blocks_per_sm;
        grid = (uint64_t)e->sm_count * (uint64_t)bps;
        const uint64_t need_blocks = (n + wpb - 1) / wpb;
        if (grid > need_blocks) grid = need_blocks;
        warp_slots = grid * wpb;
    }
    // thread-per-replica: one persistent CTA per SM
    uint64_t lgrid = 0; size_t lsmem = 0;
    // the lean build of the loop when the launch cannot reach what it leaves out; ASYNCFLOW_B200_LANE_FULL (A/B
    // experiments) keeps the full one
    const bool lean = lane && aflh::lean_launch(e->sc, o.trace_replicas) && getenv("ASYNCFLOW_B200_LANE_FULL") == nullptr;
    void (*const lane_kernel)() = bands ? (lat ? lane_kernel_for<true, true>(lean, dist, occ) : lane_kernel_for<true, false>(lean, dist, occ))
                                        : (lat ? lane_kernel_for<false, true>(lean, dist, occ) : lane_kernel_for<false, false>(lean, dist, occ));
    if (lane) {
        lsmem = (size_t)lane_warps * (size_t)C.warp_bytes;
        AF_CUDA(e, cudaFuncSetAttribute(lane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lsmem), "smem attribute");
        lgrid = (uint64_t)e->sm_count;
        const uint64_t need = (n + (uint64_t)lane_warps * 32 - 1) / ((uint64_t)lane_warps * 32);
        if (lgrid > need) lgrid = need;
    }

    // ---- device memory (grow-only) -----------------------------------------------------------------------------
    if (warp) {
        const uint64_t ev_sp = (uint64_t)(L.ev_total - L.ev_smem), rq_sp = (uint64_t)(L.rq_total - L.rq_smem);
        AF_CUDA(e, e->d_sp_evt.ensure(warp_slots * ev_sp * 8 + 8), "spill events");
        AF_CUDA(e, e->d_sp_evk.ensure(warp_slots * ev_sp * 8 + 8), "spill events");
        AF_CUDA(e, e->d_sp_rq.ensure(warp_slots * rq_sp * 16 + 16), "spill requests");
        AF_CUDA(e, e->d_sp_nx.ensure(warp_slots * rq_sp * 4 + 4), "spill requests");
    }
    if (lane && occ) aflh::add_occupancy(C, 32, occ_cols, e->occ_opt.frac_bits);
    if (lane) {
        AF_CUDA(e, e->d_gtier.ensure(lgrid * (uint64_t)lane_warps * C.gwarp_bytes + 256), "lane global tiers");
        if ((rc = upload_vec(e, e->d_l_edges, e->lt.edges, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_servers, e->lt.servers, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_eps, e->lt.endpoints, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_steps, e->lt.steps, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_spikes, e->lt.spikes, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_outages, e->lt.outages, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_lb, e->lt.lb, "lane tables"))) return rc;
        if ((rc = upload_vec(e, e->d_l_cols, e->lt.cols, "lane tables"))) return rc;
        AF_CUDA(e, e->d_counter2.ensure(8), "work counter");
        AF_CUDA(e, e->d_redo_list.ensure(n * 4), "flagged-replica list");
        AF_CUDA(e, e->d_redo_count.ensure(4), "flagged-replica count");
    }
    const uint64_t ntr = (uint64_t)(L.trace_replicas < 0 ? 0 : L.trace_replicas) < n ? (uint64_t)L.trace_replicas : n;
    L.trace_replicas = (int32_t)ntr; C.trace_replicas = (int32_t)ntr;
    AF_CUDA(e, e->d_stats.ensure(n * sizeof(AfReplicaStats)), "stats");
    AF_CUDA(e, e->d_sent.ensure(n * L.n_edges * 4), "edge counts");
    AF_CUDA(e, e->d_dropped.ensure(n * L.n_edges * 4), "edge counts");
    AF_CUDA(e, e->d_ssum.ensure(n * L.n_series * 8), "sampled sums");
    AF_CUDA(e, e->d_smax.ensure(n * L.n_series * 4), "sampled maxima");
    AF_CUDA(e, e->d_counter.ensure(8), "work counter");
    if (L.collect_hist) AF_CUDA(e, e->d_hist.ensure(n * AF_HIST_BINS * 4), "histograms");
    if (L.collect_thr) AF_CUDA(e, e->d_thr.ensure(n * (uint64_t)L.horizon_s * 4), "throughput");
    if (ntr) {
        AF_CUDA(e, e->d_tclk.ensure(ntr * (uint64_t)L.trace_clock_cap * 16 + 16), "trace clocks");
        AF_CUDA(e, e->d_tser.ensure(ntr * (uint64_t)L.n_series * (uint64_t)L.trace_tick_cap * 4 + 4), "trace series");
    }
    AF_CUDA(e, e->d_tcnt.ensure((ntr ? ntr : 1) * 8), "trace counts");
    if (bands) AF_CUDA(e, e->d_band.ensure(band_words * 8), "band rows");
    if (bands || dist) AF_CUDA(e, e->d_band_from.ensure(n * 4), "band stop ticks");
    if (dist) {
        AF_CUDA(e, e->d_dist.ensure(dist_words * 4), "distribution band rows");
        if ((rc = upload_vec(e, e->d_dist_slot, e->h_dist_slot, "distribution band series"))) return rc;
    }
    if (lat) {
        AF_CUDA(e, e->d_lat.ensure(lat_words * 8), "latency band rows");
        AF_CUDA(e, e->d_lat_from.ensure(n * 4), "latency band completions");
    }
    if (occ) AF_CUDA(e, e->d_occ.ensure(n * (uint64_t)occ_cols * 8), "occupancy rows");
    // pull order: the first pass runs `workers` replicas at once (lanes, or warps without the thread-per-replica pass)
    const uint64_t workers = lane ? lgrid * (uint64_t)lane_warps * 32ull : warp_slots;
    const uint64_t wave = workers < n ? workers : n;
    size_t sort_bytes = 0, sort2_bytes = 0;
    AF_CUDA(e, cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                         (const uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t)n, 0, 32, e->stream), "order sort size");
    AF_CUDA(e, cub::DeviceRadixSort::SortPairsDescending(nullptr, sort2_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                         (const uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t)wave, 0, 64, e->stream), "order sort size");
    AF_CUDA(e, e->d_okey.ensure(n * 8), "pull order keys");
    AF_CUDA(e, e->d_oidx.ensure(n * 4), "pull order");
    AF_CUDA(e, e->d_order.ensure(n * 4), "pull order");
    AF_CUDA(e, e->d_okey64.ensure(wave * 16), "pull order keys");
    AF_CUDA(e, e->d_sort_tmp.ensure(sort_bytes > sort2_bytes ? sort_bytes : sort2_bytes), "pull order sort");
    OrderArgs oa;
    memset(&oa, 0, sizeof oa);
    oa.cols = (const AfSweepColumn*)e->d_sweep_cols.p; oa.vals = (const double*)e->d_sweep_vals.p; oa.n_cols = e->sweep_cols;
    oa.sweep_first = e->sweep_first; oa.sweep_rows = e->sweep_cols ? e->sweep_rows : 0;
    oa.row_need = e->sweep_cols ? (const int32_t*)e->d_row_need.p : nullptr; oa.need = e->ev_need;
    oa.seed = seed; oa.begin = begin; oa.n = n;
    oa.users_dist = e->sc.users_dist; oa.users_mean = e->sc.users_mean; oa.users_sigma = e->sc.users_sigma;
    oa.rate_per_user = e->sc.rate_per_user;
    oa.span = (double)(e->sc.window_s < e->sc.horizon_s ? e->sc.window_s : e->sc.horizon_s);   // only the first window is predicted

    afc::Globals G;
    memset(&G, 0, sizeof G);
    G.edges = (const AfEdge*)e->d_edges.p; G.servers = (const AfServer*)e->d_servers.p;
    G.endpoints = (const AfEndpoint*)e->d_eps.p; G.steps = (const AfStep*)e->d_steps.p;
    G.lb_edges = (const int32_t*)e->d_lb.p; G.spikes = (const AfSpikeMark*)e->d_spikes.p;
    G.outages = (const AfOutageMark*)e->d_outages.p;
    G.sweep_cols = (const AfSweepColumn*)e->d_sweep_cols.p; G.sweep_vals = (const double*)e->d_sweep_vals.p;
    G.sweep_first = e->sweep_first; G.sweep_rows = e->sweep_cols ? e->sweep_rows : 0;
    G.spill_ev_time = (double*)e->d_sp_evt.p; G.spill_ev_key = (uint64_t*)e->d_sp_evk.p;
    G.spill_rq_rec = (afc::ReqRec*)e->d_sp_rq.p; G.spill_rq_next = (uint32_t*)e->d_sp_nx.p;
    G.stats = (AfReplicaStats*)e->d_stats.p; G.edge_sent = (uint32_t*)e->d_sent.p; G.edge_dropped = (uint32_t*)e->d_dropped.p;
    G.hist = (uint32_t*)e->d_hist.p; G.thr = (uint32_t*)e->d_thr.p;
    G.samp_sum = (uint64_t*)e->d_ssum.p; G.samp_max = (uint32_t*)e->d_smax.p;
    G.trace_clocks = (double*)e->d_tclk.p; G.trace_series = (uint32_t*)e->d_tser.p; G.trace_counts = (uint32_t*)e->d_tcnt.p;
    G.work_counter = (unsigned long long*)e->d_counter.p;
    G.order = (const uint32_t*)e->d_order.p;
    G.redo_list = redo ? (const uint32_t*)e->d_redo_list.p : nullptr;
    G.redo_count = redo ? (const uint32_t*)e->d_redo_count.p : nullptr;
    G.seed = seed; G.replica_begin = begin; G.n_replicas = n;
    if (occ) { band.occ = (uint64_t*)e->d_occ.p; band.occ_scale = ldexp(1.0, e->occ_opt.frac_bits); }
    if (bands || lat || dist) { band.group = (const uint32_t*)e->d_band_group.p; band.first = e->band_first; band.n = e->h_band_group.size(); band.groups = e->band_groups; }
    if (dist) {
        band.from = (const uint32_t*)e->d_band_from.p;
        band.dist_rows = (uint32_t*)e->d_dist.p; band.dist_slot = (const int32_t*)e->d_dist_slot.p;
        band.dist_group_words = dist_group_words; band.dist_series_words = dist_series_words; band.dist_bins = dist_bins;
    }
    if (bands) {
        band.rows = (uint64_t*)e->d_band.p; band.from = (const uint32_t*)e->d_band_from.p;
        band.group_words = band_group_words; band.stride = (uint32_t)band_stride;
    }
    if (lat) {
        band.lat_rows = (uint64_t*)e->d_lat.p; band.lat_from = (const uint32_t*)e->d_lat_from.p;
        band.lat_window = (uint32_t)e->lat_window; band.lat_windows = (uint32_t)lat_windows;
    }
    if (lane) {
        C.edges = (const afl::EdgeP*)e->d_l_edges.p; C.servers = (const afl::ServerP*)e->d_l_servers.p;
        C.endpoints = (const afl::EndpointP*)e->d_l_eps.p; C.steps = (const afl::StepP*)e->d_l_steps.p;
        C.spikes = (const afl::SpikeP*)e->d_l_spikes.p; C.outages = (const afl::OutageP*)e->d_l_outages.p;
        C.lb_edges = (const int32_t*)e->d_l_lb.p; C.cols = (const afl::ColP*)e->d_l_cols.p;
        C.sweep_vals = G.sweep_vals; C.sweep_first = G.sweep_first; C.sweep_rows = G.sweep_rows;
        C.row_need = C.need_rows ? (const int32_t*)e->d_row_need.p : nullptr;
        C.gtier = (unsigned char*)e->d_gtier.p;
        C.stats = G.stats; C.edge_sent = G.edge_sent; C.edge_dropped = G.edge_dropped; C.hist = G.hist; C.thr = G.thr;
        C.samp_sum = G.samp_sum; C.samp_max = G.samp_max; C.trace_clocks = G.trace_clocks; C.trace_series = G.trace_series;
        C.trace_counts = G.trace_counts;
        C.work_counter = (unsigned long long*)e->d_counter2.p;
        C.order = G.order;
        C.seed = seed; C.replica_begin = begin; C.n_replicas = n;
        if (bands || lat || dist) { C.band_group = band.group; C.band_first = band.first; C.band_n = band.n; C.band_groups = (int32_t)e->band_groups; }
        if (dist) {
            C.band_from = (uint32_t*)e->d_band_from.p;
            C.dist_rows = band.dist_rows; C.dist_slot = band.dist_slot;
            C.dist_group_words = dist_group_words; C.dist_series_words = dist_series_words;
            C.dist_n = (int32_t)dist_n; C.dist_bins = (int32_t)dist_bins;
        }
        if (bands) {
            C.band_rows = band.rows; C.band_from = (uint32_t*)e->d_band_from.p;
            C.band_group_words = band_group_words; C.band_stride = (int32_t)band_stride;
        }
        if (lat) {
            C.lat_rows = band.lat_rows; C.lat_from = (uint32_t*)e->d_lat_from.p;
            C.lat_window = e->lat_window; C.lat_windows = (int32_t)lat_windows;
        }
        C.occ = band.occ;
    }

    // ---- enqueue ---------------------------------------------------------------------------------------------------
    // The launch parameters live in __constant__ memory, which is per device: hold the lock until this engine's
    // copies and launches are in its stream, and wait for the device's previous engine before overwriting them.
    std::lock_guard<std::mutex> lock(g_const_mutex);
    {
        af_engine*& owner = g_const_owner[e->device % kMaxDevices];
        if (owner && owner != e) AF_CUDA(e, cudaStreamSynchronize(owner->stream), "waiting for the device's previous engine");
        owner = e;
    }
    AF_CUDA(e, cudaEventRecord(e->ev_begin, e->stream), "event");
    AF_CUDA(e, cudaMemsetAsync(e->d_counter.p, 0, 8, e->stream), "memset");
    if (L.collect_hist) AF_CUDA(e, cudaMemsetAsync(e->d_hist.p, 0, n * AF_HIST_BINS * 4, e->stream), "memset hist");
    if (L.collect_thr) AF_CUDA(e, cudaMemsetAsync(e->d_thr.p, 0, n * (uint64_t)L.horizon_s * 4, e->stream), "memset thr");
    if (bands) AF_CUDA(e, cudaMemsetAsync(e->d_band.p, 0, band_words * 8, e->stream), "memset band rows");
    if (lat) AF_CUDA(e, cudaMemsetAsync(e->d_lat.p, 0, lat_words * 8, e->stream), "memset latency band rows");
    if (dist) AF_CUDA(e, cudaMemsetAsync(e->d_dist.p, 0, dist_words * 4, e->stream), "memset distribution band rows");
    {   // the pull order: (work, local index) heaviest first; then the first wave grouped by estimate
        uint32_t* key = (uint32_t*)e->d_okey.p; uint32_t* idx = (uint32_t*)e->d_oidx.p; uint32_t* order = (uint32_t*)e->d_order.p;
        uint64_t* key64 = (uint64_t*)e->d_okey64.p;
        af_order_key_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(oa, key, idx);
        AF_CUDA(e, cudaGetLastError(), "af_order_key_kernel launch");
        AF_CUDA(e, cub::DeviceRadixSort::SortPairsDescending(e->d_sort_tmp.p, sort_bytes, key, key + n, idx, order, (uint32_t)n, 0, 32,
                                                             e->stream), "order sort");
        af_order_group_kernel<<<(unsigned)((wave + 255) / 256), 256, 0, e->stream>>>(oa, key + n, order, wave, key64, idx);
        AF_CUDA(e, cudaGetLastError(), "af_order_group_kernel launch");
        AF_CUDA(e, cub::DeviceRadixSort::SortPairsDescending(e->d_sort_tmp.p, sort2_bytes, key64, key64 + wave, idx, order, (uint32_t)wave,
                                                             0, 64, e->stream), "order sort");
        e->launches += 4;
    }
    if (lane) {
        AF_CUDA(e, cudaMemsetAsync(e->d_counter2.p, 0, 8, e->stream), "memset");
        AF_CUDA(e, cudaMemsetAsync(e->d_redo_count.p, 0, 4, e->stream), "memset");
        AF_CUDA(e, cudaMemcpyToSymbolAsync(afl::c_cfg, &C, sizeof C, 0, cudaMemcpyHostToDevice, e->stream), "lane config -> constant memory");
        lane_kernel<<<(unsigned)lgrid, lane_warps * 32, lsmem, e->stream>>>();
        AF_CUDA(e, cudaGetLastError(), "af_lane_kernel launch");
        e->launches += 1;
        if (redo) {
            af_flagged_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>((const AfReplicaStats*)e->d_stats.p, n,
                AF_FLAG_EVENT_OVERFLOW | AF_FLAG_REQUEST_OVERFLOW | AF_FLAG_NOWQ_OVERFLOW, (uint32_t*)e->d_redo_list.p, (uint32_t*)e->d_redo_count.p);
            AF_CUDA(e, cudaGetLastError(), "af_flagged_kernel launch");
            e->launches += 1;
        }
    }
    if (warp) {
        AF_CUDA(e, cudaMemcpyToSymbolAsync(afc::c_L, &L, sizeof L, 0, cudaMemcpyHostToDevice, e->stream), "layout -> constant memory");
        e->G_host = G;   // keep the source alive until the async copy has been issued from pageable memory
        AF_CUDA(e, cudaMemcpyToSymbolAsync(afc::c_G, &e->G_host, sizeof G, 0, cudaMemcpyHostToDevice, e->stream), "globals -> constant memory");
        af_sim_kernel<<<(unsigned)grid, wpb * 32, smem, e->stream>>>(band);
        AF_CUDA(e, cudaGetLastError(), "af_sim_kernel launch");
        e->launches += 1;
    }
    AF_CUDA(e, cudaEventRecord(e->ev_sim, e->stream), "event");
    if (bands) {      // the fetched groups' difference rows -> per-tick values (the last group collects replicas without one)
        const uint64_t rows = (uint64_t)e->band_groups * (1 + 2 * (uint64_t)L.n_series);
        af_band_scan_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, e->stream>>>((uint64_t*)e->d_band.p, rows, band_stride, band_ticks);
        AF_CUDA(e, cudaGetLastError(), "af_band_scan_kernel launch");
        e->launches += 1;
    }
    if (dist) {       // the fetched groups' rows -> per-tick bin counts
        const uint64_t rows = (uint64_t)e->band_groups * dist_n, threads = rows * dist_bins;
        af_dist_scan_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, e->stream>>>((uint32_t*)e->d_dist.p, rows, dist_bins,
                                                                                     dist_series_words, dist_ticks);
        AF_CUDA(e, cudaGetLastError(), "af_dist_scan_kernel launch");
        e->launches += 1;
    }
    if (L.collect_hist) {
        unsigned blocks = (unsigned)((n * 32 + 255) / 256);
        af_percentile_kernel<<<blocks, 256, 0, e->stream>>>((const uint32_t*)e->d_hist.p, (AfReplicaStats*)e->d_stats.p, n);
        AF_CUDA(e, cudaGetLastError(), "af_percentile_kernel launch");
        e->launches += 1;
    }
    AF_CUDA(e, cudaEventRecord(e->ev_end, e->stream), "event");
    e->last_n = n; e->ran = true; e->timing_valid = false;
    e->last_lane = lane; e->last_warp = warp; e->last_lean = lean; e->last_lane_warps = lane_warps;
    e->last_bands = bands; e->last_band_groups = e->band_groups; e->last_band_ticks = (uint32_t)band_ticks;
    e->last_band_stride = band_stride;
    e->last_lat = lat; e->last_lat_groups = e->band_groups; e->last_lat_windows = lat_windows;
    e->last_dist = dist; e->last_dist_groups = e->band_groups; e->last_dist_ticks = dist_ticks; e->last_dist_bins = dist_bins;
    e->last_dist_n = (uint32_t)dist_n; e->last_dist_series_words = dist_series_words;
    e->last_occ = occ; e->last_occ_bits = e->occ_opt.frac_bits; e->last_occ_cols = occ_cols;
    return AF_OK;
}

int af_selftest_rng(af_engine* e, uint64_t seed, uint64_t replica, int kind, int dist, double mean, double sigma,
                    uint32_t hop, uint64_t n, double* out_a, double* out_b) {
    if (!e || !out_a || !out_b || n == 0) return AF_ERR_INVALID;
    if (kind < AF_SELFTEST_EDGE || kind > AF_SELFTEST_EXP) return e->fail(AF_ERR_INVALID, "af_selftest_rng: unknown kind");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    DevBuf da, db;
    cudaError_t ce;
    if ((ce = da.ensure(n * 8)) != cudaSuccess || (ce = db.ensure(n * 8)) != cudaSuccess) { da.release(); db.release(); return e->cuda_fail(ce, "selftest buffers"); }
    af_selftest_rng_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(seed, replica, kind, dist, mean, sigma, hop, n, (double*)da.p, (double*)db.p);
    e->launches += 1;
    ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(out_a, da.p, n * 8, cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(out_b, db.p, n * 8, cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    da.release(); db.release();
    if (ce != cudaSuccess) return e->cuda_fail(ce, "af_selftest_rng");
    return AF_OK;
}

int af_engine_set_mode(af_engine* e, int mode) {
    if (!e) return AF_ERR_INVALID;
    if (mode != AF_MODE_AUTO && mode != AF_MODE_WARP && mode != AF_MODE_LANE && mode != AF_MODE_TWO_PASS) return e->fail(AF_ERR_INVALID, "af_engine_set_mode: unknown mode");
    e->mode = mode;
    return AF_OK;
}

int af_last_run_passes(af_engine* e, AfRunPasses* out) {
    if (!e || !out) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "no run yet");
    int rc = af_sync(e);
    if (rc) return rc;
    memset(out, 0, sizeof *out);
    out->lane_pass = e->last_lane ? 1 : 0; out->warp_pass = e->last_warp ? 1 : 0;
    out->lane_warps_per_sm = e->last_lane_warps;
    out->lane_bytes = e->last_lane ? e->C_host.warp_bytes / 32 : 0;
    out->lane_events_smem = e->last_lane ? e->last_ev_s : 0; out->lane_requests_smem = e->last_lane ? e->last_rq_s : 0;
    out->lane_pool_elems = e->last_lane ? e->C_host.pool : 0;
    out->lane_lean = e->last_lean ? 1 : 0;
    out->lane_replicas = e->last_lane ? e->last_n : 0;
    out->warp_replicas = e->last_warp ? e->last_n : 0;
    if (e->last_lane && e->last_warp) {
        uint32_t c = 0;
        AF_CUDA(e, cudaMemcpyAsync(&c, e->d_redo_count.p, 4, cudaMemcpyDeviceToHost, e->stream), "flagged count D2H");
        AF_CUDA(e, cudaStreamSynchronize(e->stream), "flagged count D2H");
        out->warp_replicas = c;
    }
    return AF_OK;
}

int af_sync(af_engine* e) {
    if (!e) return AF_ERR_INVALID;
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "af_sync");
    if (e->ran && !e->timing_valid) {
        float a = 0.f, b = 0.f;
        // begin -> end spans memsets + both kernels; begin -> sim spans memsets + the simulation kernel
        if (cudaEventElapsedTime(&a, e->ev_begin, e->ev_end) == cudaSuccess
            && cudaEventElapsedTime(&b, e->ev_begin, e->ev_sim) == cudaSuccess) {
            e->ms_total = a; e->ms_sim = b; e->timing_valid = true;
        }
    }
    return AF_OK;
}

int af_last_run_ms(af_engine* e, float* ms_total, float* ms_sim) {
    if (!e) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "no run yet");
    int rc = af_sync(e);
    if (rc) return rc;
    if (ms_total) *ms_total = e->ms_total;
    if (ms_sim) *ms_sim = e->ms_sim;
    return AF_OK;
}

uint64_t af_launch_count(const af_engine* e) { return e ? e->launches : 0; }

static int fetch(af_engine* e, void* dst, const DevBuf& src, size_t bytes, uint64_t n, const char* what) {
    if (!e || !dst) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (n != e->last_n) return e->fail(AF_ERR_INVALID, "fetch: n differs from the last run's replica count");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    AF_CUDA(e, cudaMemcpyAsync(dst, src.p, bytes, cudaMemcpyDeviceToHost, e->stream), what);
    return af_sync(e);
}

int af_fetch_stats(af_engine* e, AfReplicaStats* out, uint64_t n) {
    return fetch(e, out, e->d_stats, n * sizeof(AfReplicaStats), n, "stats D2H");
}
int af_fetch_edge_counts(af_engine* e, uint32_t* sent, uint32_t* dropped, uint64_t n) {
    int rc = fetch(e, sent, e->d_sent, n * e->L.n_edges * 4, n, "edge sent D2H");
    if (rc) return rc;
    return fetch(e, dropped, e->d_dropped, n * e->L.n_edges * 4, n, "edge dropped D2H");
}
int af_fetch_histograms(af_engine* e, uint32_t* out, uint64_t n) {
    if (e && e->ran && !e->L.collect_hist) return e->fail(AF_ERR_STATE, "histograms were not collected");
    return fetch(e, out, e->d_hist, n * AF_HIST_BINS * 4, n, "hist D2H");
}
int af_fetch_throughput(af_engine* e, uint32_t* out, uint64_t n) {
    if (e && e->ran && !e->L.collect_thr) return e->fail(AF_ERR_STATE, "throughput was not collected");
    return fetch(e, out, e->d_thr, n * (uint64_t)e->L.horizon_s * 4, n, "throughput D2H");
}
int af_fetch_sampled(af_engine* e, uint64_t* sums, uint32_t* maxima, uint64_t n) {
    int rc = fetch(e, sums, e->d_ssum, n * e->L.n_series * 8, n, "sampled sums D2H");
    if (rc) return rc;
    return fetch(e, maxima, e->d_smax, n * e->L.n_series * 4, n, "sampled maxima D2H");
}

int af_reduce_histograms(af_engine* e, uint64_t* out_bins) {
    if (!e || !out_bins) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "reduce before af_run");
    if (!e->L.collect_hist) return e->fail(AF_ERR_STATE, "histograms were not collected");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    AF_CUDA(e, e->d_htot.ensure(AF_HIST_BINS * 8), "histogram total");
    AF_CUDA(e, cudaMemsetAsync(e->d_htot.p, 0, AF_HIST_BINS * 8, e->stream), "memset");
    const uint64_t n = e->last_n;
    uint64_t blocks = (uint64_t)e->sm_count * 8;
    if (blocks > n) blocks = n;
    uint64_t rows = (n + blocks - 1) / blocks;
    blocks = (n + rows - 1) / rows;
    af_hist_reduce_kernel<<<(unsigned)blocks, 256, 0, e->stream>>>((const uint32_t*)e->d_hist.p,
                                                                  (unsigned long long*)e->d_htot.p, n, rows);
    AF_CUDA(e, cudaGetLastError(), "af_hist_reduce_kernel launch");
    e->launches += 1;
    AF_CUDA(e, cudaMemcpyAsync(out_bins, e->d_htot.p, AF_HIST_BINS * 8, cudaMemcpyDeviceToHost, e->stream), "hist total D2H");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "af_reduce_histograms");
    return AF_OK;
}

int af_fetch_trace_clocks(af_engine* e, uint64_t local, double* out, uint64_t cap_pairs, uint64_t* n_pairs) {
    if (!e || !out || !n_pairs) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (local >= (uint64_t)e->L.trace_replicas) return e->fail(AF_ERR_INVALID, "replica was not traced");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    uint32_t cnt[2];
    AF_CUDA(e, cudaMemcpyAsync(cnt, (uint32_t*)e->d_tcnt.p + local * 2, 8, cudaMemcpyDeviceToHost, e->stream), "trace counts");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "trace counts");
    uint64_t n = cnt[0];
    if (n > (uint64_t)e->L.trace_clock_cap) n = (uint64_t)e->L.trace_clock_cap;
    if (n > cap_pairs) n = cap_pairs;
    *n_pairs = n;
    if (n) AF_CUDA(e, cudaMemcpyAsync(out, (double*)e->d_tclk.p + local * (uint64_t)e->L.trace_clock_cap * 2, n * 16,
                                      cudaMemcpyDeviceToHost, e->stream), "trace clocks");
    return af_sync(e);
}

int af_fetch_bands(af_engine* e, uint32_t* count, uint64_t* sum, uint64_t* sumsq, uint64_t cap_ticks, uint64_t* n_ticks) {
    if (!e || !n_ticks) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (!e->last_bands) return e->fail(AF_ERR_STATE, "the last run collected no bands (af_bands_upload)");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    const uint64_t T = e->last_band_ticks, G = e->last_band_groups, S = (uint64_t)e->L.n_series, stride = e->last_band_stride;
    const uint64_t k = T < cap_ticks ? T : cap_ticks;
    *n_ticks = T;
    const uint64_t* base = (const uint64_t*)e->d_band.p;
    const uint64_t group_words = (1 + 2 * S) * stride;
    std::vector<uint64_t> c64(count && k ? G * k : 0);
    for (uint64_t g = 0; g < G && k; ++g) {
        const uint64_t* gb = base + g * group_words;
        if (count) AF_CUDA(e, cudaMemcpyAsync(c64.data() + g * k, gb, k * 8, cudaMemcpyDeviceToHost, e->stream), "band counts D2H");
        if (sum) AF_CUDA(e, cudaMemcpy2DAsync(sum + g * S * cap_ticks, cap_ticks * 8, gb + stride, stride * 8, k * 8, S,
                                              cudaMemcpyDeviceToHost, e->stream), "band sums D2H");
        if (sumsq) AF_CUDA(e, cudaMemcpy2DAsync(sumsq + g * S * cap_ticks, cap_ticks * 8, gb + (1 + S) * stride, stride * 8, k * 8, S,
                                                cudaMemcpyDeviceToHost, e->stream), "band sums of squares D2H");
    }
    int rc = af_sync(e);
    if (rc) return rc;
    if (count)
        for (uint64_t g = 0; g < G; ++g)
            for (uint64_t t = 0; t < k; ++t) count[g * cap_ticks + t] = (uint32_t)c64[g * k + t];
    return AF_OK;
}

int af_fetch_latency_bands(af_engine* e, uint64_t* hist, uint64_t* sum_hi, uint64_t* sum_lo, uint64_t cap_windows,
                           uint64_t* n_windows) {
    if (!e || !n_windows) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (!e->last_lat) return e->fail(AF_ERR_STATE, "the last run collected no latency bands (af_bands_configure, af_bands_upload)");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    const uint64_t W = e->last_lat_windows, G = e->last_lat_groups, R = afr::LAT_ROW, B = AF_HIST_BINS;
    const uint64_t k = W < cap_windows ? W : cap_windows;
    *n_windows = W;
    const uint64_t* base = (const uint64_t*)e->d_lat.p;
    for (uint64_t g = 0; g < G && k; ++g) {                // window j of group g: row g * W + j
        const uint64_t* gb = base + g * W * R;
        if (hist) AF_CUDA(e, cudaMemcpy2DAsync(hist + g * cap_windows * B, B * 8, gb, R * 8, B * 8, k, cudaMemcpyDeviceToHost, e->stream),
                          "latency band histograms D2H");
        if (sum_hi) AF_CUDA(e, cudaMemcpy2DAsync(sum_hi + g * cap_windows, 8, gb + B, R * 8, 8, k, cudaMemcpyDeviceToHost, e->stream),
                            "latency band sums D2H");
        if (sum_lo) AF_CUDA(e, cudaMemcpy2DAsync(sum_lo + g * cap_windows, 8, gb + B + 1, R * 8, 8, k, cudaMemcpyDeviceToHost, e->stream),
                            "latency band sums D2H");
    }
    return af_sync(e);
}

int af_fetch_dist_bands(af_engine* e, uint32_t* out, uint64_t cap_ticks, uint64_t* n_ticks, uint32_t* n_bins) {
    if (!e || !n_ticks || !n_bins) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (!e->last_dist) return e->fail(AF_ERR_STATE, "the last run collected no distribution bands (af_dist_bands_configure, af_bands_upload)");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    const uint64_t T = e->last_dist_ticks, B = e->last_dist_bins, rows = (uint64_t)e->last_dist_groups * e->last_dist_n;
    const uint64_t k = T < cap_ticks ? T : cap_ticks;
    *n_ticks = T; *n_bins = (uint32_t)B;
    if (!out || !k) return AF_OK;
    // row (g, s) of the device is (T + 1) tick rows of B bins; the caller's holds cap_ticks of them
    AF_CUDA(e, cudaMemcpy2DAsync(out, cap_ticks * B * 4, e->d_dist.p, e->last_dist_series_words * 4, k * B * 4, rows,
                                 cudaMemcpyDeviceToHost, e->stream), "distribution bands D2H");
    return af_sync(e);
}

int af_fetch_occupancy(af_engine* e, uint64_t* out, uint64_t n, int32_t* frac_bits) {
    if (!e) return AF_ERR_INVALID;
    if (e->ran && !e->last_occ) return e->fail(AF_ERR_STATE, "the last run collected no occupancy (af_occupancy_configure)");
    if (frac_bits) *frac_bits = e->last_occ_bits;
    return fetch(e, out, e->d_occ, n * (uint64_t)e->last_occ_cols * 8, n, "occupancy D2H");
}

int af_fetch_trace_series(af_engine* e, uint64_t local, uint32_t* out, uint64_t cap_ticks, uint64_t* n_ticks) {
    if (!e || !out || !n_ticks) return AF_ERR_INVALID;
    if (!e->ran) return e->fail(AF_ERR_STATE, "fetch before af_run");
    if (local >= (uint64_t)e->L.trace_replicas) return e->fail(AF_ERR_INVALID, "replica was not traced");
    AF_CUDA(e, cudaSetDevice(e->device), "cudaSetDevice");
    uint32_t cnt[2];
    AF_CUDA(e, cudaMemcpyAsync(cnt, (uint32_t*)e->d_tcnt.p + local * 2, 8, cudaMemcpyDeviceToHost, e->stream), "trace counts");
    AF_CUDA(e, cudaStreamSynchronize(e->stream), "trace counts");
    uint64_t n = cnt[1];
    if (n > (uint64_t)e->L.trace_tick_cap) n = (uint64_t)e->L.trace_tick_cap;
    if (n > cap_ticks) n = cap_ticks;
    *n_ticks = n;
    const uint32_t* base = (const uint32_t*)e->d_tser.p + local * (uint64_t)e->L.n_series * (uint64_t)e->L.trace_tick_cap;
    if (n) AF_CUDA(e, cudaMemcpy2DAsync(out, cap_ticks * 4, base, (size_t)e->L.trace_tick_cap * 4, n * 4, (size_t)e->L.n_series,
                                        cudaMemcpyDeviceToHost, e->stream), "trace series");
    return af_sync(e);
}

}  // extern "C"
