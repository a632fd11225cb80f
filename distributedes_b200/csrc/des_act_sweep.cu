// The sweep instantiations of policy_act_kernel (des_policy_act_sweep, des_act.cu), in a translation unit of their own:
// see des_act.cuh.
#include "des_act.cuh"

namespace des {

int act_launch_sweep(const ActSweepArgs &a, int H, int64_t n, cudaStream_t st) { return act_launch(a, H, n, st); }

}  // namespace des
