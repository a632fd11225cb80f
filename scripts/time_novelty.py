"""Time novelty search's kernels and one NSR-ES generation against one NES generation, with CUDA events after a warm-up.

1. des_novelty over n queries x A archive rows x d dimensions, k = 10: milliseconds per call and distance evaluations
   (n x A) per second, for n = 64, 4096 and 65 536, A = 10^3, 10^4 and 10^5, d = 3 and 24.
2. One generation on the closed-loop Pendulum (10 episodes x 200 steps per member) at N = 64, 1024 and 4096 and H = 16
   and 64, against an archive of 1000 behaviours, split into its phases; the NES and NSR-ES arms alternate trial by trial:
     eval      des_rollout_eval (NES) / des_rollout_eval_bc (NSR-ES)
     shape     des_centered_rank (NES) / des_novelty of the N behaviours + des_ns_shape at w = 0.5 (NSR-ES)
     update    des_nes_grad_partial + des_nes_apply + des_state_advance (the same in both arms)
     test      des_rollout_eval of 10 noiseless test episodes / des_rollout_eval_bc of them
   Each shape also checks that the two arms' evaluation fitness is the same, bit for bit.

Prints the GPU's name, power limit and maximum SM clock, then one JSON line per shape (milliseconds, medians).

    python scripts/time_novelty.py [--trials K]
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
from time_record import gpu  # noqa: E402


def timed(fn, trials):
    """Median milliseconds of fn() over `trials` event-timed calls, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(trials):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def novelty_table(trials):
    g = torch.Generator(device='cuda').manual_seed(0)
    for d in (3, 24):
        for A in (1000, 10000, 100000):
            archive = torch.randn((A, d), device='cuda', generator=g)
            for n in (64, 4096, 65536):
                q = torch.randn((n, d), device='cuda', generator=g)
                out = torch.empty(n, device='cuda')
                ms = timed(lambda: ops.novelty(q, archive, 10, out=out), trials)
                print(json.dumps(dict(op='des_novelty', n=n, A=A, d=d, k=10, ms=round(ms, 4),
                                      distances_per_s=float('%.4g' % (n * A / (ms * 1e-3))))), flush=True)


def generation_table(trials):
    for N in (64, 1024, 4096):
        for H in (16, 64):
            theta = torch.from_numpy(StandardFCNet(3, 1, H, seed=0).get_weight()).cuda()
            P = theta.numel()
            stats = torch.tensor([0.1, 0.2, 0.3, 0.5, 0.4, 20.0, 1000.0], dtype=torch.float32, device='cuda')
            state = ops.new_state('cuda', 3)
            env = dict(hidden=H, horizon=200, clip=2.0, action_noise_std=0.1, seed=7, state=state, obs_stats=stats)
            fit = {arm: torch.empty(N, device='cuda') for arm in ('nes', 'ns')}
            test_fit, episodes = torch.empty(1, device='cuda'), torch.empty(10, device='cuda')
            bc, test_bc = torch.empty((N, 3), device='cuda'), torch.empty((1, 3), device='cuda')
            archive = torch.randn((1000, 3), device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
            nov, shaped = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
            rank_ws, shape_ws = ops.rank_workspace(N, 'cuda', N), ops.ns_shape_workspace(N, 'cuda')
            grad_ws = ops.grad_workspace(N, P, 'cuda')
            partial, update = torch.empty(P, device='cuda'), torch.empty(P, device='cuda')
            m, v = torch.zeros(P, dtype=torch.float64, device='cuda'), torch.zeros(P, dtype=torch.float64, device='cuda')
            th = theta.clone()

            def evaluate(arm):
                kw = dict(repetitions=10, sigma=0.05, n_local=N, out=fit[arm], **env)
                if arm == 'ns':
                    ops.rollout_eval_bc(th, bc_out=bc, **kw)
                else:
                    ops.rollout_eval(th, **kw)

            def shape(arm):
                if arm == 'ns':
                    ops.novelty(bc, archive, 10, out=nov)
                    ops.ns_shape(fit[arm], nov, 0.5, workspace=shape_ws, out=shaped)
                else:
                    ops.centered_rank(fit[arm], workspace=rank_ws, out=shaped)

            def step(arm):
                ops.nes_grad_partial(shaped, P, seed=7, state=state, workspace=grad_ws, out=partial)
                ops.nes_apply(th, m, v, partial, N, state, sigma=0.05, learning_rate=0.01, update_out=update)
                ops.state_advance(state)

            def test(arm):
                kw = dict(repetitions=10, sigma=0.0, n_local=1, noiseless=True, out=test_fit, episodes_out=episodes, **env)
                if arm == 'ns':
                    ops.rollout_eval_bc(th, bc_out=test_bc, **kw)
                else:
                    ops.rollout_eval(th, **kw)

            phases = dict(eval=evaluate, shape=shape, update=step, test=test)
            for arm in ('nes', 'ns'):                                      # warm-up of every shape
                for fn in phases.values():
                    fn(arm)
            evaluate('nes')
            evaluate('ns')
            same = bool(torch.equal(fit['nes'], fit['ns']))
            times = {arm: {p: [] for p in phases} for arm in ('nes', 'ns')}
            torch.cuda.synchronize()
            for _ in range(trials):
                for arm in ('nes', 'ns'):                                  # alternate the arms
                    for p, fn in phases.items():
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        fn(arm)
                        b.record()
                        b.synchronize()
                        times[arm][p].append(a.elapsed_time(b))
            row = dict(op='generation', N=N, H=H, archive=1000, same_fitness=same)
            for arm in ('nes', 'ns'):
                med = {p: round(float(np.median(t)), 4) for p, t in times[arm].items()}
                med['total'] = round(sum(med.values()), 4)
                row[arm] = med
            row['shape_share_of_nes'] = round(row['ns']['shape'] / row['nes']['total'], 4)
            print(json.dumps(row), flush=True)


def main():
    K = int(sys.argv[sys.argv.index('--trials') + 1]) if '--trials' in sys.argv else 10
    print(json.dumps(dict(gpu=gpu())), flush=True)
    novelty_table(K)
    generation_table(K)


if __name__ == '__main__':
    main()
