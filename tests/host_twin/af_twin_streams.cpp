// The CPU twin with per-replica timeline rows (af_twin_rows.cpp) and random streams -- TEST INFRASTRUCTURE ONLY.
//
// af_streams_upload's table reaches the kernels as afl::Cfg's stream_* fields (thread per replica) and as
// af_sim_kernel's afc::StreamArgs (warp per replica).  This file compiles af_twin_rows.cpp (and through it af_twin.cpp)
// unchanged and routes the rows library's two calls into the state machines -- afl::run_lane and afc::run_replica --
// through hooks that also hand them the table set by af_twin_streams_set, the way af_run does; every other line of a
// launch is af_twin.cpp's, and the rows are af_twin_rows.cpp's.  With no table set the hooks pass none, and the library
// behaves as libaf_twin_rows.so.  Built into tests/host_twin/_build/ and loaded by tests/twin_streams.py only.
#include <vector>
#include "../../asyncflow_b200/csrc/af_host_common.h"
#include "../../asyncflow_b200/csrc/af_lane_host.h"

namespace twin_streams {
std::vector<uint64_t> table;               // stream of replica first + i (empty: every replica draws as its id)
uint64_t first = 0;
}  // namespace twin_streams

namespace afl {
// af_run's lane-pass set-up of the table (af_engine.cu), then the state machine
template <bool... B, class P, class F>
void run_lane_with_streams(const Mem& m, P pull, F converge) {
    if (!twin_streams::table.empty()) {
        h_cfg.stream_of = twin_streams::table.data(); h_cfg.stream_first = twin_streams::first;
        h_cfg.stream_rows = twin_streams::table.size();
    }
    run_lane<B...>(m, pull, converge);
}
}  // namespace afl
namespace afc {
// af_sim_kernel's StreamArgs for the table
inline void run_replica_with_streams(State& W, uint64_t local_index, const BandArgs& band, const TimelineArgs& tl) {
    StreamArgs rs = {};
    if (!twin_streams::table.empty()) { rs.stream_of = twin_streams::table.data(); rs.first = twin_streams::first; rs.rows = twin_streams::table.size(); }
    run_replica(W, local_index, band, tl, rs);
}
}  // namespace afc

// af_twin_rows.cpp's hooks call run_lane / run_replica: these names reach the hooks above.  (af_twin_rows.cpp then
// points the same names at its own hooks for af_twin.cpp; the preprocessor notes the redefinition, which is intended.)
#define run_lane run_lane_with_streams
#define run_replica run_replica_with_streams
#include "af_twin_rows.cpp"

// The table of every later af_twin_run_lane / af_twin_run_warp: replica first + i, i < n, draws as stream_of[i] (NULL or
// n = 0: every replica as its own id).  The table is copied.
extern "C" void af_twin_streams_set(const uint64_t* stream_of, uint64_t n, uint64_t first) {
    twin_streams::table.assign(stream_of, stream_of + (stream_of ? n : 0));
    twin_streams::first = first;
}
