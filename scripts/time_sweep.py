"""Time a sweep of R NES runs of 64 members on the closed-loop Pendulum three ways: one RolloutRunsEngine with a seed
and hyper-parameters per run (a sweep), one RolloutRunsEngine of R runs of one config (a batch of runs), and R
RolloutEngines one after another.  H in {16, 64}, 10 x 200-step episodes per member, R in {1, 4, 10, 32}.

  generation   ms per generation of all R runs, from CUDA events around `iters` graph-replayed generations after a
               warm-up, with the L2 flushed before each timed window (the sequential arm times each run and sums them).
               The three arms are timed in turn, `rounds` times; the median of each is reported.
  grad         us per call of the sweep's gradient (des_nes_grad_partial_sweep: round keys in registers, set up from each
               run's seed) against the batch's (des_nes_grad_partial_runs: round keys in the parameter bank), same shapes,
               timed in turn the same way; at N = 64 and at N = 2048, where the hot loop dominates.

Prints one JSON line with the card's name and power limit, read in the same call.

    python scripts/time_sweep.py [--iters 20] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distributedes_b200 import ops, ops_runs                            # noqa: E402
from distributedes_b200.engine import RolloutEngine, RolloutRunsEngine   # noqa: E402
from distributedes_b200.model import StandardFCNet                       # noqa: E402
from time_runs import card, timed                                        # noqa: E402

POP = 64


def _hyper(R):
    """A sigma x learning-rate grid of R runs, each with its own seed."""
    return dict(seeds=list(range(1, R + 1)), sigma=[(0.05, 0.1, 0.2)[r % 3] for r in range(R)],
                learning_rate=[(0.02, 0.05, 0.1, 0.2)[r % 4] for r in range(R)])


def _median_rounds(fns, rounds, iters):
    times = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            times[i].append(fn(iters))
    return [statistics.median(t) for t in times]


def generation_ms(H, R, iters, rounds):
    theta0 = StandardFCNet(3, 1, H, seed=0).get_weight()
    kw = dict(hidden=H, pop_size=POP, theta0=theta0, use_graph=True)
    h = _hyper(R)
    sweep = RolloutRunsEngine(runs=R, **kw, **h)
    batch = RolloutRunsEngine(runs=R, sigma=0.1, learning_rate=0.1, seed=1, **kw)
    singles = [RolloutEngine(seed=h['seeds'][r], sigma=h['sigma'][r], learning_rate=h['learning_rate'][r], **kw)
               for r in range(R)]
    for _ in range(3):                                   # warm-up: graph capture, module loading
        sweep.generation()
        batch.generation()
        for e in singles:
            e.generation()
    torch.cuda.synchronize()
    return _median_rounds([lambda n: timed(sweep.generation, n), lambda n: timed(batch.generation, n),
                           lambda n: sum(timed(e.generation, n) for e in singles)], rounds, iters)


def grad_us(H, R, N, iters, rounds):
    P = ops.param_count(3, H, 1)
    shaped = torch.from_numpy(np.random.default_rng(0).uniform(-0.5, 0.5, (R, N)).astype(np.float32)).cuda()
    h = _hyper(R)
    hp = ops_runs.run_table(h['seeds'], h['sigma'], h['learning_rate'], 0.005, 0.0, 'cuda')
    st, ws, out = ops.new_state('cuda', 0), ops_runs.grad_runs_workspace(R, N, P, 'cuda'), torch.empty((R, P), device='cuda')

    def sweep():
        ops_runs.nes_grad_partial_sweep(shaped, P, hp, state=st, workspace=ws, out=out)

    def runs():
        ops_runs.nes_grad_partial_runs(shaped, P, seed=1, state=st, workspace=ws, out=out)
    for fn in (sweep, runs):
        fn()
    torch.cuda.synchronize()
    ms = _median_rounds([lambda n: timed(sweep, n), lambda n: timed(runs, n)], rounds, iters * 10)
    return [1000 * t for t in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_sweep.py measures on a GPU; none is available')
    torch.cuda.set_device(0)
    rows, grads = [], []
    for H in (16, 64):
        for R in (1, 4, 10, 32):
            sw, bat, seq = generation_ms(H, R, a.iters, a.rounds)
            rows.append(dict(hidden=H, runs=R, pop=POP, sweep_generation_ms=round(sw, 4),
                             runs_generation_ms=round(bat, 4), seq_generation_ms=round(seq, 4),
                             sweep_over_runs=round(sw / bat, 3), seq_over_sweep=round(seq / sw, 2)))
            print(json.dumps(rows[-1]), file=sys.stderr)
    for H, R, N in ((64, 10, 64), (64, 32, 64), (64, 10, 2048)):
        sw, rn = grad_us(H, R, N, a.iters, a.rounds)
        grads.append(dict(hidden=H, runs=R, pop=N, sweep_grad_us=round(sw, 2), runs_grad_us=round(rn, 2),
                          sweep_over_runs=round(sw / rn, 3)))
        print(json.dumps(grads[-1]), file=sys.stderr)
    res = dict(card=card(), generation=rows, grad=grads)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
