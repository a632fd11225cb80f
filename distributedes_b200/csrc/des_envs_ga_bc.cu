// The genetic algorithm's behaviour-writing instantiations of rollout_pendulum_kernel (des_rollout_eval_ga_bc,
// des_envs.cu), in a translation unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

int rollout_ga_bc_launch(const GaBcArgs &a, int H, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(GaBcArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rollout_pendulum_kernel<1, false, GaBcArgs>; break;
        case 2: kernel = rollout_pendulum_kernel<2, false, GaBcArgs>; break;
        case 4: kernel = rollout_pendulum_kernel<4, false, GaBcArgs>; break;
        case 6: kernel = rollout_pendulum_kernel<6, false, GaBcArgs>; break;
        default: kernel = rollout_pendulum_kernel<8, false, GaBcArgs>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

}  // namespace des
