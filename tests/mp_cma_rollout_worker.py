"""torchrun worker for tests/test_gpu_cma_rollout.py::test_two_gpu_closed_loop_cma_equals_one_gpu (2 ranks, NCCL):
two generations of closed-loop CMA-ES (Pendulum-v0, 16 hidden units, lambda = 37: a ragged 19 + 18 split).
run() is the same run in one process (no process group)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run():
    from distributedes_b200 import cma_es
    from distributedes_b200.config import ClosedLoopPendulumConfig
    cfg = ClosedLoopPendulumConfig(16)
    cfg.pop_size, cfg.sigma, cfg.seed, cfg.max_generations = 37, 0.5, 3, 3
    worker = cma_es.Worker(0, None, None, None, None, cfg)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, cfg.pop_size, seed=cfg.seed, device=worker.device)
    costs = []
    real_run = worker.run

    def spy_run(solutions, member_offset=0, generation=0):
        cost = real_run(solutions, member_offset, generation)
        costs.append(es.gather_cost(cost).cpu().numpy().copy())
        return cost
    worker.run = spy_run
    rewards, _, _ = cma_es.train(cfg, worker=worker, es=es)
    return dict(cost=np.stack(costs), stats=worker.obs_stats.cpu().numpy(), m=es.m.cpu().numpy(),
                rewards=np.asarray(rewards))


if __name__ == '__main__':
    rank = int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl')
    out = run()
    np.savez(os.path.join(sys.argv[1], 'rank%d.npz' % rank), **out)
    dist.destroy_process_group()
