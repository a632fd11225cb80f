"""Time a genetic-algorithm generation against an NES generation on the closed-loop Pendulum (10 episodes x 200 steps
per member), with CUDA events after a warm-up, the variants alternated in one process, at N = 64, 1024 and 4096 members
and H = 16, 64 and 128:

  nes_rollout    des_rollout_eval (theta + sigma*eps built in shared memory)
  ga_fused       des_rollout_eval_ga over a table of T = ceil(0.2 N) parents, 2 elites
  ga_rows        des_ga_rows of the N rows + des_rollout_eval_solutions on them (the materialised path)
  nes_update     des_centered_rank + des_nes_grad_partial + des_nes_apply + des_state_advance: the rest of an NES step
  ga_select      des_ga_order + des_ga_rows' gather of the T selected members: the rest of a GA step

Each shape also checks that ga_fused and ga_rows give the same fitness, bit for bit.  Prints the GPU's name, power limit
and maximum SM clock, then one JSON line per shape (milliseconds per call, median of the trials).

    python scripts/time_ga.py [--trials K]
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


def main():
    K = int(sys.argv[sys.argv.index('--trials') + 1]) if '--trials' in sys.argv else 10
    print(json.dumps(dict(gpu=gpu())))
    for N in (64, 1024, 4096):
        for H in (16, 64, 128):
            theta = torch.from_numpy(StandardFCNet(3, 1, H, seed=0).get_weight()).cuda()
            P, T = theta.numel(), -(-N // 5)
            parents = ops.ga_rows(theta.reshape(1, -1), 0, sigma=0.1, seed=1, generation=0, n_local=T)
            stats = torch.tensor([0.1, 0.2, 0.3, 0.5, 0.4, 20.0, 1000.0], dtype=torch.float32, device='cuda')
            env = dict(hidden=H, horizon=200, repetitions=10, clip=2.0, action_noise_std=0.1, seed=7, generation=3,
                       obs_stats=stats)
            f_nes, f_fused, f_rows = (torch.empty(N, device='cuda') for _ in range(3))
            rows = torch.empty((N, P), device='cuda')
            nxt = torch.empty((T, P), device='cuda')
            order_ws = ops.ga_order_workspace(N, 'cuda')
            rank_ws, grad_ws = ops.rank_workspace(N, 'cuda', N), ops.grad_workspace(N, P, 'cuda')
            shaped, partial = torch.empty(N, device='cuda'), torch.empty(P, device='cuda')
            m, v = torch.zeros(P, dtype=torch.float64, device='cuda'), torch.zeros(P, dtype=torch.float64, device='cuda')
            state = ops.new_state('cuda')
            th = theta.clone()

            def nes_rollout():
                ops.rollout_eval(theta, sigma=0.1, n_local=N, out=f_nes, **env)

            def ga_fused():
                ops.rollout_eval_ga(parents, 2, sigma=0.1, n_local=N, out=f_fused, **env)

            def ga_rows():
                ops.ga_rows(parents, 2, sigma=0.1, seed=7, generation=3, n_local=N, out=rows)
                ops.rollout_eval_solutions(rows, out=f_rows, **env)

            def nes_update():
                ops.centered_rank(f_nes, 0, N, workspace=rank_ws, out=shaped)
                ops.nes_grad_partial(shaped, P, seed=7, state=state, workspace=grad_ws, out=partial)
                ops.nes_apply(th, m, v, partial, N, state, sigma=0.1, learning_rate=0.01)
                ops.state_advance(state)

            def ga_select():
                order = ops.ga_order(f_fused, T, workspace=order_ws)
                ops.ga_rows(parents, 2, sigma=0.1, seed=7, generation=3, members=order, out=nxt)

            variants = dict(nes_rollout=nes_rollout, ga_fused=ga_fused, ga_rows=ga_rows, nes_update=nes_update,
                            ga_select=ga_select)
            res = {k: [] for k in variants}
            for _ in range(3):                       # alternate the variants
                for k, fn in variants.items():
                    res[k].append(timed(fn, K))
            ms = {k: round(float(np.median(v)), 4) for k, v in res.items()}
            print(json.dumps(dict(N=N, H=H, T=T, ms=ms, fused_equals_rows=bool(torch.equal(f_fused, f_rows)),
                                  ga_over_nes=round((ms['ga_fused'] + ms['ga_select']) /
                                                    (ms['nes_rollout'] + ms['nes_update']), 4))))


if __name__ == '__main__':
    main()
