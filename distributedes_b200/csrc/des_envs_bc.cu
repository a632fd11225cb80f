// The behaviour-writing instantiations of rollout_pendulum_kernel (des_rollout_eval_bc, des_envs.cu), in a translation
// unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

int rollout_bc_launch(const BcArgs &a, int H, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(BcArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rollout_pendulum_kernel<1, false, BcArgs>; break;
        case 2: kernel = rollout_pendulum_kernel<2, false, BcArgs>; break;
        case 4: kernel = rollout_pendulum_kernel<4, false, BcArgs>; break;
        case 6: kernel = rollout_pendulum_kernel<6, false, BcArgs>; break;
        default: kernel = rollout_pendulum_kernel<8, false, BcArgs>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

}  // namespace des
