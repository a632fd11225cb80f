"""Time a sweep of R CMA-ES runs of lambda = 64 two ways: one cma_es.train_sweep generation (CMASweep + SweepWorker: one
launch per step for every run) and R cma_es.train generations one after another (Worker + CMAEvolutionStrategy per
run).  H in {16, 32}, R in {1, 4, 10, 32}, on two environments:

  pendulum  closed-loop Pendulum-v0 on the device (ClosedLoopPendulumConfig: 10 repetitions of 200 steps).
  noop      a vectorised no-op host environment (envs.py protocol, obs 24, action 4, zero observations and rewards,
            every episode 100 steps; HostEnvConfig, 10 repetitions): what the host bridge itself costs.

  generation  ms per generation of all R runs: one generation is train()'s loop body (ask, evaluate, steps, best =
              argmin, test(best), rank, tell, merge), ending in a synchronise.  Each run's eigendecomposition comes every
              eigen_gap generations (CMAEvolutionStrategy.eigen_gap: 1 to 5 here), so a window is the smallest multiple of
              the gap of at least --min-gens generations, after a warm-up of as many: every window then holds the same
              eigendecompositions per run in both arms.  The arms are timed in turn, `rounds` times; the median of each.
  split       ms per phase and generation, averaged over one instrumented gap of sweep generations, a synchronise after
              each phase: ask (noise_fill_sweep and each run's sampling GEMM), eval (the evaluation and the test
              episodes), update (rank + rank-mu + covariance update, with each run's fp64 bookkeeping of tell), eigh
              (each run's step size and cuSOLVER eigendecomposition, amortised over the gap) and host (argmin,
              statistics merge).

Prints one JSON line with the card's name, power limit and SM clock limit, read in the same call.

    python scripts/time_cma_sweep.py [--min-gens 4] [--rounds 3] [--out results.json]
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distributedes_b200 import cma_es                                          # noqa: E402
from distributedes_b200.config import ClosedLoopPendulumConfig, HostEnvConfig  # noqa: E402
from time_runs import card                                                     # noqa: E402

POP, D0, A = 64, 24, 4


class NoopEnv:
    """The shapes the config probes."""
    class _Box:
        def __init__(self, n):
            self.shape = (n,)
    observation_space, action_space = _Box(D0), _Box(A)


class NoopBatch:
    """Zero observations and rewards; every episode lasts `length` steps."""

    def __init__(self, B, length=100):
        self.num_envs, self.length = B, length

    def reset(self, keys):
        self.t = 0
        return np.zeros((self.num_envs, D0))

    def step(self, actions, alive):
        self.t += 1
        return np.zeros((self.num_envs, D0)), np.zeros(self.num_envs), np.full(self.num_envs, self.t >= self.length)


def configs(env, H, R):
    out = []
    for r in range(R):
        c = ClosedLoopPendulumConfig(H) if env == 'pendulum' else HostEnvConfig(NoopEnv, H, batch_env_fn=NoopBatch)
        c.pop_size, c.seed, c.sigma = POP, 1000 + r, 0.5
        c.initial_weight = c.initial_weight.copy()
        out.append(c)
    return out


class Single:
    """R train() runs, one generation each in turn."""

    def __init__(self, cs):
        self.runs = []
        for c in cs:
            w = cma_es.Worker(0, None, None, None, None, c)
            self.runs.append((c, w, cma_es.CMAEvolutionStrategy(c.initial_weight, c.sigma, c.pop_size, seed=c.seed,
                                                                device=w.device, kernels=w.kn)))

    def generation(self):
        for c, worker, es in self.runs:
            solutions = es.ask()
            cost = es.gather_cost(worker.run(solutions, es.offset, es.gen))
            worker.steps_over_ranks(es)
            best = int(torch.argmin(cost))
            cma_es.test(c, solutions[best], None, worker=worker)
            shaped = worker.kn.centered_rank(cost.to(torch.float32).contiguous(), 0, es.lam)
            es.tell(solutions, shaped)
            worker.merge_obs_stats(es)
        torch.cuda.synchronize()


class Sweep:
    """One train_sweep generation of every run; `split` times its phases (CMASweep.tell marks its own)."""

    def __init__(self, cs):
        self.cs = cs
        self.worker, self.es = cma_es.build_sweep(cs)

    def generation(self, split=None):
        worker, es, c, R = self.worker, self.es, self.cs[0], len(self.cs)
        clock = [time.perf_counter()]

        def mark(name):
            if split is not None:
                torch.cuda.synchronize()
                t = time.perf_counter()
                split[name] = split.get(name, 0.0) + (t - clock[0]) * 1e3
                clock[0] = t
        rows = es.ask()
        mark('ask')
        cost = worker.run(rows, es.gen, es.running)
        worker.steps(es.lam)
        mark('eval')
        best = torch.argmin(cost, dim=1)
        best_rows = rows.reshape(R, es.lam, -1)[torch.arange(R, device=rows.device), best].contiguous()
        mark('host')
        worker.test_returns(best_rows, c.test_repetitions, es.running)
        mark('eval')
        es.tell(worker.kn.centered_rank_runs(cost.to(torch.float32).contiguous()), mark=mark if split is not None else None)
        worker.merge_obs_stats(es.running)
        torch.cuda.synchronize()
        mark('host')


def window(arm, gens):
    """ms per generation over `gens` generations, after a warm-up of `gens` generations: with `gens` a multiple of the
    eigen gap, both arms start every window at the same point of the gap and every window holds the same number of
    eigendecompositions per run."""
    for _ in range(gens):
        arm.generation()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(gens):
        arm.generation()
    return (time.perf_counter() - t) * 1e3 / gens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--min-gens', type=int, default=4, help='a window is the smallest multiple of the eigen gap >= this')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rows = []
    for env in ('pendulum', 'noop'):
        for H in (16, 32):
            for R in (1, 4, 10, 32):
                cs = configs(env, H, R)
                single, sweep = Single(copy.deepcopy(cs)), Sweep(cs)
                gap = sweep.es.es[0].eigen_gap
                gens = gap * -(-args.min_gens // gap)
                t_single, t_sweep = [], []
                for _ in range(args.rounds):
                    t_single.append(window(single, gens))
                    t_sweep.append(window(sweep, gens))
                split = {}
                for _ in range(gap):                  # one whole gap: each run's eigh once, amortised over its generations
                    sweep.generation(split=split)
                row = dict(env=env, H=H, R=R, lam=POP, eigen_gap=gap, window_gens=gens,
                           sequential_ms=statistics.median(t_single), sweep_ms=statistics.median(t_sweep),
                           split_ms={k: round(v / gap, 3) for k, v in split.items()})
                row['speedup'] = row['sequential_ms'] / row['sweep_ms']
                print(json.dumps(row), flush=True)
                rows.append(row)
    result = dict(card=card(), rows=rows)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
