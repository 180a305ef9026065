// The CPU twin with timeline rows, random streams, admission limits (af_twin_admission.cpp) and request deadlines --
// TEST INFRASTRUCTURE ONLY.
//
// Deadlines and the client timeout reach the state machines through AfServer.deadline, AfScenario.client_timeout and
// the sweep's AF_FIELD_SERVER_DEADLINE / AF_FIELD_CLIENT_TIMEOUT columns, which af_twin.cpp already hands them; what a
// launch adds is the output of the expiry and late counts (afl::Cfg.server_expired / late, afc::BandArgs.server_expired
// / late), which af_run points at its buffers when afh::deadline_launch says the launch has a deadline or a timeout
// somewhere.  This file compiles af_twin_admission.cpp unchanged and routes its two calls into the state machines
// through hooks that set those pointers, and exports af_sweep_upload's and af_scenario_upload's checks of the values.
// Built into tests/host_twin/_build/ and loaded by tests/twin_deadline.py only.
#include <string.h>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

namespace twin_dl {
uint32_t* expired = nullptr;               // [n][n_servers] of every later launch (nullptr: not collected)
uint32_t* late = nullptr;                  // [n]
double client_timeout = 0.0;               // the scenario's, which af_run hands the warp engine in BandArgs
}  // namespace twin_dl

namespace afl {
template <bool... B, class P, class F>
void run_lane_with_deadlines(const Mem& m, P pull, F converge) {
    if (h_cfg.dl) { h_cfg.server_expired = twin_dl::expired; h_cfg.late = twin_dl::late; }
    run_lane<B...>(m, pull, converge);
}
}  // namespace afl
namespace afc {
inline void run_replica_with_deadlines(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl,
                                       const StreamArgs& rs) {
    BandArgs b = band;
    b.server_expired = twin_dl::expired; b.late = twin_dl::late; b.client_timeout = twin_dl::client_timeout;
    run_replica(W, local_index, b, tl, rs);
}
}  // namespace afc

#define run_lane run_lane_with_deadlines
#define run_replica run_replica_with_deadlines
#include "af_twin_admission.cpp"

// Where every later af_twin_run_lane / af_twin_run_warp writes its expiry ([n][n_servers]) and late ([n]) counts (NULL:
// nowhere), and the scenario's client timeout the warp engine gets (af_run: BandArgs.client_timeout; the lane engine
// reads it from the scenario's tables).  The warp engine writes the counts whatever the launch; the lane engine only when
// the launch has a deadline or a timeout somewhere, as on the device (the caller zeroes the buffers, as af_run does).
extern "C" void af_twin_deadline_set(uint32_t* expired, uint32_t* late, double client_timeout) {
    twin_dl::expired = expired; twin_dl::late = late; twin_dl::client_timeout = client_timeout;
}

// 1 when the launch of `sc` + `sw` has a deadline or a client timeout somewhere (afh::deadline_launch), else 0
extern "C" int af_twin_deadline_launch(const AfScenario* sc, const AfSweep* sw) {
    return afh::deadline_launch(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0) ? 1 : 0;
}

// 1 when af_run would take the lean lane build for `sc` + `sw` without traces (aflh::lean_launch), else 0
extern "C" int af_twin_deadline_lean(const AfScenario* sc, const AfSweep* sw) {
    return aflh::lean_launch(*sc, 0, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0) ? 1 : 0;
}

// af_sweep_upload's check of the deadline columns of `sw` (afh::deadline_sweep_fits): 1 when accepted, else 0
extern "C" int af_twin_deadline_sweep_fits(const AfSweep* sw) {
    return afh::deadline_sweep_fits(sw->columns, sw->n_columns, sw->values, sw->n_rows, g_err) ? 1 : 0;
}
