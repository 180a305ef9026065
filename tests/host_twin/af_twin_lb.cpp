// The launch checks of load-balancer sweep rows (DESIGN.md §3.11) on the host -- TEST INFRASTRUCTURE ONLY.
//
// af_sweep_upload checks AF_FIELD_LB_COVERED / AF_FIELD_LB_ALGORITHM columns with afh::lb_sweep_fits, and af_run checks
// the rows against the outage marks each replica runs with by afh::lb_cover_fits.  This file exports both, as the CPU
// twin's launches (af_twin_streams.cpp) would apply them, so that the CPU tier tests the rules af_run enforces.  Built into
// tests/host_twin/_build/ and loaded by tests/twin_lb.py only.
#include <stdio.h>
#include "../../asyncflow_b200/csrc/af_host_common.h"

static std::string g_lb_err;
extern "C" const char* af_twin_lb_error() { return g_lb_err.c_str(); }

// 1 when af_sweep_upload accepts the load-balancer columns of `sw`, else 0 (af_twin_lb_error() says why)
extern "C" int af_twin_lb_sweep_fits(const AfScenario* sc, const AfSweep* sw) {
    return afh::lb_sweep_fits(*sc, sw->columns, sw->n_columns, sw->values, sw->n_rows, g_lb_err) ? 1 : 0;
}

// 1 when af_run accepts a launch of replicas [begin, end) with sweep rows from sweep_first and timeline rows `tl`
// (NULL: none) from tl_first, else 0 (af_twin_lb_error() says why)
extern "C" int af_twin_lb_cover_fits(const AfScenario* sc, const AfSweep* sw, uint64_t sweep_first, const AfTimeline* tl,
                                     uint64_t tl_first, uint64_t begin, uint64_t end) {
    return afh::lb_cover_fits(*sc, sw->columns, sw->n_columns, sw->values, sweep_first, sw->n_rows,
                              tl && tl->n_rows ? tl : nullptr, tl_first, begin, end, g_lb_err) ? 1 : 0;
}
