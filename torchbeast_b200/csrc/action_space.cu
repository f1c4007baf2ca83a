// Factored (multi-discrete) action spaces: the host-side check every factored entry point shares, and the layout query.
// The kernels that take a factored row live beside their flat forms (vtrace.cu, sample.cu, net_kernels.cu).
#include <stddef.h>

#include "common.cuh"

namespace tb {

int action_segments(const tb_action_space* space, int64_t A, const char* who, ActionSegments* out) {
  TB_REQUIRE(space, "%s: null action space", who);
  const int D = space->num_components;
  TB_REQUIRE(D >= 1 && D <= TB_MAX_ACTION_COMPONENTS, "%s: num_components %d outside [1, %d]", who, D,
             TB_MAX_ACTION_COMPONENTS);
  int64_t off = 0;
  out->D = D;
  out->off[0] = 0;
  for (int k = 0; k < D; ++k) {
    TB_REQUIRE(space->dims[k] >= 1, "%s: component %d has %d actions (at least 1)", who, k, space->dims[k]);
    off += space->dims[k];
    TB_REQUIRE(off <= A, "%s: the component sizes add up to more than A = %lld", who, (long long)A);
    out->off[k + 1] = int(off);
  }
  TB_REQUIRE(off == A, "%s: the component sizes add up to %lld, not A = %lld", who, (long long)off, (long long)A);
  for (int k = D + 1; k <= TB_MAX_ACTION_COMPONENTS; ++k) out->off[k] = int(off);
  return 0;
}

}  // namespace tb

extern "C" int tb_action_space_layout(int64_t* out_host) {
  TB_REQUIRE(out_host, "tb_action_space_layout: null pointer");
  out_host[0] = int64_t(sizeof(tb_action_space));
  out_host[1] = int64_t(offsetof(tb_action_space, num_components));
  out_host[2] = int64_t(offsetof(tb_action_space, dims));
  return 0;
}
