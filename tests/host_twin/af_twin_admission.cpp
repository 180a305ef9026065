// The CPU twin with timeline rows and random streams (af_twin_streams.cpp) and admission limits -- TEST INFRASTRUCTURE ONLY.
//
// Admission limits reach the state machines through the scenario's AfServer.max_in_service and the sweep's
// AF_FIELD_SERVER_MAX_IN_SERVICE columns, which af_twin.cpp already hands them; what a launch adds is the output of the
// rejection counts (afl::Cfg.server_rejected, afc::BandArgs.server_rejected), which af_run points at its buffer when
// afh::admission_launch says the launch has a limit somewhere.  This file compiles af_twin_streams.cpp unchanged and
// routes its two calls into the state machines through hooks that set that pointer, and exports af_sweep_upload's and
// af_scenario_upload's checks of the limits.  Built into tests/host_twin/_build/ and loaded by tests/twin_admission.py only.
#include <string.h>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

namespace twin_adm {
uint32_t* rejected = nullptr;              // [n][n_servers] of every later launch (nullptr: not collected)
}  // namespace twin_adm

namespace afl {
template <bool... B, class P, class F>
void run_lane_with_admission(const Mem& m, P pull, F converge) {
    if (h_cfg.adm) h_cfg.server_rejected = twin_adm::rejected;
    run_lane<B...>(m, pull, converge);
}
}  // namespace afl
namespace afc {
inline void run_replica_with_admission(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl,
                                       const StreamArgs& rs) {
    BandArgs b = band;
    b.server_rejected = twin_adm::rejected;
    run_replica(W, local_index, b, tl, rs);
}
}  // namespace afc

#define run_lane run_lane_with_admission
#define run_replica run_replica_with_admission
#include "af_twin_streams.cpp"

// Where every later af_twin_run_lane / af_twin_run_warp writes its rejection counts ([n][n_servers], NULL: nowhere).
// The warp engine writes them whatever the launch; the lane engine only when the launch has a limit somewhere, as on
// the device (the caller zeroes the buffer, as af_run does).
extern "C" void af_twin_admission_set(uint32_t* rejected) { twin_adm::rejected = rejected; }

// 1 when the launch of `sc` + `sw` has an admission limit somewhere (afh::admission_launch), else 0
extern "C" int af_twin_admission_launch(const AfScenario* sc, const AfSweep* sw) {
    return afh::admission_launch(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0) ? 1 : 0;
}

// af_scenario_upload's check (afh::validate): 1 when `sc` is accepted, else 0 (af_twin_error() says why)
extern "C" int af_twin_admission_validate(const AfScenario* sc) { return afh::validate(*sc, g_err) ? 1 : 0; }

// af_sweep_upload's check of the admission columns of `sw` (afh::admission_sweep_fits): 1 when accepted, else 0
extern "C" int af_twin_admission_sweep_fits(const AfSweep* sw) {
    return afh::admission_sweep_fits(sw->columns, sw->n_columns, sw->values, sw->n_rows, g_err) ? 1 : 0;
}
