// The recording instantiations of rollout_pendulum_kernel (des_rollout_record[_solutions], des_envs.cu), in a translation
// unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

int rollout_record_launch(const RecordArgs &a, int H, bool rows_mode, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(RecordArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rows_mode ? rollout_pendulum_kernel<1, true, RecordArgs> : rollout_pendulum_kernel<1, false, RecordArgs>; break;
        case 2: kernel = rows_mode ? rollout_pendulum_kernel<2, true, RecordArgs> : rollout_pendulum_kernel<2, false, RecordArgs>; break;
        case 4: kernel = rows_mode ? rollout_pendulum_kernel<4, true, RecordArgs> : rollout_pendulum_kernel<4, false, RecordArgs>; break;
        case 6: kernel = rows_mode ? rollout_pendulum_kernel<6, true, RecordArgs> : rollout_pendulum_kernel<6, false, RecordArgs>; break;
        default: kernel = rows_mode ? rollout_pendulum_kernel<8, true, RecordArgs> : rollout_pendulum_kernel<8, false, RecordArgs>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

}  // namespace des
