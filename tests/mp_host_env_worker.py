"""One rank of the 2-GPU host-stepped check (tests/test_gpu_host_env.py): HostEnvEngine on SynthWalk-v0, each rank
stepping only its own members' environments.  `run()` without torch.distributed is the single-GPU reference."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def run():
    import torch
    from distributedes_b200.engine import HostEnvEngine
    from distributedes_b200.envs import GymEnvBatch
    from oracle import nes_oracle as orc
    from oracle import synth_walk as sw
    eng = HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=lambda B: GymEnvBatch(sw.SynthWalkEnv, B, 4), hidden=64,
                        pop_size=13, theta0=orc.synthetic_theta(24, 64, 4), sigma=0.1, learning_rate=0.1,
                        repetitions=4, seed=4)
    fit, steps = [], []
    for _ in range(2):
        eng.generation()
        fit.append(eng.fitness_all.cpu().numpy().copy())
        steps.append(eng.steps_taken)
    torch.cuda.synchronize()
    return dict(fit=np.stack(fit), steps=np.asarray(steps), stats=eng.obs_stats.cpu().numpy(), theta=eng.theta_numpy())


if __name__ == '__main__':
    import torch
    import torch.distributed as dist
    rank = int(os.environ['RANK'])
    torch.cuda.set_device(rank)
    os.environ.setdefault('DES_COMM', 'nccl')
    dist.init_process_group('nccl')
    try:
        np.savez(os.path.join(sys.argv[1], 'rank%d.npz' % rank), **run())
    finally:
        dist.destroy_process_group()
