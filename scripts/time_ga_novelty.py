"""Time the genetic algorithm's novelty-search generation against the plain GA generation on the closed-loop Pendulum
(10 episodes x 200 steps per member), with CUDA events after a warm-up, the variants alternated in one process, at
N = 64, 1024 and 4096 members and H = 16, 64 and 128, over a table of T = ceil(0.2 N) parents with 2 elites:

  ga_fused      des_rollout_eval_ga
  ga_bc_fused   des_rollout_eval_ga_bc: the same evaluation, also writing each member's behaviour
  ga_order      des_ga_order: the GA's selection
  ns_order      des_novelty of the N behaviours against an archive of A = 1000 rows (k = 10) + des_ns_ga_order at
                w = 0.5: GA-NSR's selection

Each shape also checks that ga_fused and ga_bc_fused give the same fitness, bit for bit.  Prints the GPU's name, power
limit and maximum SM clock, then one JSON line per shape (milliseconds per call, median of the trials).

    python scripts/time_ga_novelty.py [--trials K]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedes_b200 import ops  # noqa: E402
from distributedes_b200.model import StandardFCNet  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_ga import timed  # noqa: E402
from time_record import gpu  # noqa: E402

ARCHIVE, K_NN, W = 1000, 10, 0.5


def main():
    K = int(sys.argv[sys.argv.index('--trials') + 1]) if '--trials' in sys.argv else 10
    print(json.dumps(dict(gpu=gpu())))
    for N in (64, 1024, 4096):
        for H in (16, 64, 128):
            theta = torch.from_numpy(StandardFCNet(3, 1, H, seed=0).get_weight()).cuda()
            T = -(-N // 5)
            parents = ops.ga_rows(theta.reshape(1, -1), 0, sigma=0.1, seed=1, generation=0, n_local=T)
            stats = torch.tensor([0.1, 0.2, 0.3, 0.5, 0.4, 20.0, 1000.0], dtype=torch.float32, device='cuda')
            env = dict(hidden=H, horizon=200, repetitions=10, clip=2.0, action_noise_std=0.1, seed=7, generation=3,
                       obs_stats=stats)
            f_ga, f_bc = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
            bc = torch.empty((N, 3), device='cuda')
            g = torch.Generator(device='cuda').manual_seed(N + H)
            archive = torch.rand((ARCHIVE, 3), device='cuda', generator=g) * 2 - 1
            nov = torch.empty(N, device='cuda')
            order_ws, ns_ws = ops.ga_order_workspace(N, 'cuda'), ops.ns_ga_order_workspace(N, 'cuda')
            o_ga, o_ns = torch.empty(T, dtype=torch.int32, device='cuda'), torch.empty(T, dtype=torch.int32, device='cuda')

            def ga_fused():
                ops.rollout_eval_ga(parents, 2, sigma=0.1, n_local=N, out=f_ga, **env)

            def ga_bc_fused():
                ops.rollout_eval_ga_bc(parents, 2, sigma=0.1, n_local=N, out=f_bc, bc_out=bc, **env)

            def ga_order():
                ops.ga_order(f_ga, T, workspace=order_ws, out=o_ga)

            def ns_order():
                ops.novelty(bc, archive, K_NN, out=nov)
                ops.ns_ga_order(f_bc, nov, W, T, workspace=ns_ws, out=o_ns)

            variants = dict(ga_fused=ga_fused, ga_bc_fused=ga_bc_fused, ga_order=ga_order, ns_order=ns_order)
            res = {k: [] for k in variants}
            for _ in range(3):                       # alternate the variants
                for k, fn in variants.items():
                    res[k].append(timed(fn, K))
            ms = {k: round(float(np.median(v)), 4) for k, v in res.items()}
            print(json.dumps(dict(N=N, H=H, T=T, ms=ms, bc_equals_ga=bool(torch.equal(f_ga, f_bc)),
                                  bc_over_ga=round(ms['ga_bc_fused'] / ms['ga_fused'], 4),
                                  ns_over_ga=round((ms['ga_bc_fused'] + ms['ns_order']) /
                                                   (ms['ga_fused'] + ms['ga_order']), 4))))


if __name__ == '__main__':
    main()
