// The CPU twin with timeline rows, random streams, admission limits, request deadlines (af_twin_deadline.cpp) and rate
// limits -- TEST INFRASTRUCTURE ONLY.
//
// Rate limits reach the state machines through AfServer.rate_limit / burst, AfScenario.lb_rate_limit / lb_burst and the
// sweep's four rate-limit columns, which af_twin.cpp already hands them (the lane engine reads the scenario's through
// its tables); what a launch adds is the output of the throttle counts (afl::Cfg.throttled, afc::BandArgs.throttled),
// which af_run points at its buffer when afh::ratelimit_launch says the launch has a rate limit somewhere, and the
// scenario's LB rate and burst the warp engine gets in BandArgs.  This file compiles af_twin_deadline.cpp unchanged and
// routes its two calls into the state machines through hooks that set them, and exports the checks and the GCRA rule.
// Built into tests/host_twin/_build/ and loaded by tests/twin_ratelimit.py only.
#include <string.h>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

namespace twin_rl {
uint32_t* throttled = nullptr;             // [n][n_servers + 1] of every later launch (nullptr: not collected)
double lb_rate = 0.0;                      // the scenario's, which af_run hands the warp engine in BandArgs
int32_t lb_burst = 0;
}  // namespace twin_rl

namespace afl {
template <bool... B, class P, class F>
void run_lane_with_ratelimit(const Mem& m, P pull, F converge) {
    if (h_cfg.rl) h_cfg.throttled = twin_rl::throttled;
    run_lane<B...>(m, pull, converge);
}
}  // namespace afl
namespace afc {
inline void run_replica_with_ratelimit(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl,
                                       const StreamArgs& rs) {
    BandArgs b = band;
    b.throttled = twin_rl::throttled; b.lb_rate = twin_rl::lb_rate; b.lb_burst = twin_rl::lb_burst;
    run_replica(W, local_index, b, tl, rs);
}
}  // namespace afc

#define run_lane run_lane_with_ratelimit
#define run_replica run_replica_with_ratelimit
#include "af_twin_deadline.cpp"

// Where every later af_twin_run_lane / af_twin_run_warp writes its throttle counts ([n][n_servers + 1], NULL: nowhere),
// and the scenario's LB rate and burst the warp engine gets (af_run: BandArgs).  The warp engine writes the counts
// whatever the launch; the lane engine only when the launch has a rate limit somewhere, as on the device (the caller
// zeroes the buffer, as af_run does).
extern "C" void af_twin_ratelimit_set(uint32_t* throttled, double lb_rate, int32_t lb_burst) {
    twin_rl::throttled = throttled; twin_rl::lb_rate = lb_rate; twin_rl::lb_burst = lb_burst;
}

// 1 when the launch of `sc` + `sw` has a rate limit somewhere (afh::ratelimit_launch), else 0
extern "C" int af_twin_ratelimit_launch(const AfScenario* sc, const AfSweep* sw) {
    return afh::ratelimit_launch(*sc, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0) ? 1 : 0;
}

// 1 when af_run would take the lean lane build for `sc` + `sw` without traces (aflh::lean_launch), else 0
extern "C" int af_twin_ratelimit_lean(const AfScenario* sc, const AfSweep* sw) {
    return aflh::lean_launch(*sc, 0, sw ? sw->columns : nullptr, sw ? sw->n_columns : 0) ? 1 : 0;
}

// af_sweep_upload's check of the rate-limit columns of `sw` on `sc` (afh::ratelimit_sweep_fits): 1 when accepted, else 0
extern "C" int af_twin_ratelimit_sweep_fits(const AfScenario* sc, const AfSweep* sw) {
    return afh::ratelimit_sweep_fits(*sc, sw->columns, sw->n_columns, sw->values, sw->n_rows, g_err) ? 1 : 0;
}

// The GCRA rule both engines run (afr::rl_params, afr::rl_pass) on one request taken at `now` by a site with `rate` and
// `burst`: 1 when it passes (*tat updated), 0 when it is throttled (*tat unchanged)
extern "C" int af_twin_rl_pass(double* tat, double now, double rate, double burst) {
    double tau, lim;
    afr::rl_params(rate, burst, tau, lim);
    return afr::rl_pass(*tat, now, tau, lim) ? 1 : 0;
}
