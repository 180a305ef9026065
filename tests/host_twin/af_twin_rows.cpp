// The CPU twin (af_twin.cpp) with per-replica timeline rows -- TEST INFRASTRUCTURE ONLY.
//
// af_timeline_upload's rows reach the kernels as afl::Cfg's tl_* fields (thread per replica) and as af_sim_kernel's
// afc::TimelineArgs (warp per replica).  This file compiles af_twin.cpp unchanged and routes its two calls into the state
// machines -- afl::run_lane and afc::run_replica -- through hooks that hand them the rows set by af_twin_rows_set, the
// way af_run does; every other line of a launch is af_twin.cpp's.  With no rows set the hooks pass none, and the library
// behaves as libaf_twin.so.  Built into tests/host_twin/_build/ and loaded by tests/twin_rows.py only.
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

namespace twin_rows {
AfTimeline rows = {};                      // n_rows == 0: none
uint64_t first = 0;                        // the replica row 0 describes
std::vector<afl::SpikeP> lane_spikes;      // the spike rows in the lane kernel's layout (aflh::timeline_spikes)
}  // namespace twin_rows

namespace afl {
// af_run's lane-pass set-up of the rows (af_engine.cu), then the state machine
template <bool... B, class P, class F>
void run_lane_with_rows(const Mem& m, P pull, F converge) {
    if (twin_rows::rows.n_rows) {
        h_cfg.tl_spikes = twin_rows::lane_spikes.data(); h_cfg.tl_outages = (const OutageP*)twin_rows::rows.outages;
        h_cfg.tl_first = twin_rows::first; h_cfg.tl_rows = twin_rows::rows.n_rows;
    }
    run_lane<B...>(m, pull, converge);
}
}  // namespace afl
namespace afc {
// af_sim_kernel's TimelineArgs for the rows
inline void run_replica_with_rows(State& W, uint64_t local_index, const BandArgs& band) {
    TimelineArgs tl = {};
    if (twin_rows::rows.n_rows) { tl.spikes = twin_rows::rows.spikes; tl.outages = twin_rows::rows.outages; tl.first = twin_rows::first; tl.rows = twin_rows::rows.n_rows; }
    run_replica(W, local_index, band, tl);
}
}  // namespace afc

#define run_lane run_lane_with_rows
#define run_replica run_replica_with_rows
#include "af_twin.cpp"
#undef run_lane
#undef run_replica

// Rows of every later af_twin_run_lane / af_twin_run_warp: row r describes replica first + r (NULL or n_rows = 0: none).
// The checks of af_timeline_upload (the rows against the scenario) and af_run (no AF_FIELD_SPIKE_DELTA column of `sw`);
// AF_ERR_INVALID and af_twin_error() when one fails (the rows are then cleared).  The caller keeps the rows alive.
extern "C" int af_twin_rows_set(const AfScenario* sc, const AfSweep* sw, const AfTimeline* t, uint64_t first) {
    twin_rows::rows = AfTimeline{};
    twin_rows::lane_spikes.clear();
    if (!t || t->n_rows == 0) return AF_OK;
    if (!afh::validate_timeline(*sc, *t, g_err) || !afh::timeline_sweep_fits(sw ? sw->columns : nullptr, sw ? sw->n_columns : 0, g_err))
        return AF_ERR_INVALID;
    aflh::timeline_spikes(*sc, *t, twin_rows::lane_spikes);
    twin_rows::rows = *t;
    twin_rows::first = first;
    return AF_OK;
}

extern "C" int af_twin_rows_sizeof_timeline() { return (int)sizeof(AfTimeline); }
