"""Time a sweep of R genetic-algorithm runs of N = 64 two ways: one genetic.train_sweep generation (GASweep + SweepWorker:
one launch per step for every run) and R genetic.train generations one after another (Worker + GeneticAlgorithm per
run).  H in {16, 64}, R in {1, 4, 10, 32}, on two environments:

  pendulum  closed-loop Pendulum-v0 on the device (ClosedLoopPendulumConfig: 10 repetitions of 200 steps; the fused
            des_rollout_eval_ga[_sweep] evaluation).
  noop      the vectorised no-op host environment of time_cma_sweep.py (obs 24, action 4, every episode 100 steps;
            HostEnvConfig, 10 repetitions): what the host bridge itself costs.

  generation  ms per generation of all R runs: one generation is train()'s loop body (evaluate, steps, best = max, tell,
              test(row 0), merge), ending in a synchronise.  Each arm runs --gens warm-up generations, then --gens timed
              ones; the arms are timed in turn, `rounds` times; the median of each.
  split       ms per phase and generation of the sweep, averaged over --gens instrumented generations, a synchronise
              after each phase: eval (the generation's evaluation), select (des_ga_order_runs and the gather of the next
              tables), test (the test episodes of every run's row 0) and host (max, step counts, statistics merge).

Prints one JSON line per arm and one with the card's name, power limit and SM clock limit, read in the same call.

    python scripts/time_ga_sweep.py [--gens 4] [--rounds 3] [--out results.json]
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distributedes_b200 import genetic                                         # noqa: E402
from distributedes_b200.config import ClosedLoopPendulumConfig, HostEnvConfig  # noqa: E402
from time_cma_sweep import NoopBatch, NoopEnv                                  # noqa: E402
from time_runs import card                                                     # noqa: E402

POP = 64


def configs(env, H, R):
    out = []
    for r in range(R):
        c = ClosedLoopPendulumConfig(H) if env == 'pendulum' else HostEnvConfig(NoopEnv, H, batch_env_fn=NoopBatch)
        c.pop_size, c.seed, c.sigma = POP, 1000 + r, 0.05
        c.initial_weight = c.initial_weight.copy()
        out.append(c)
    return out


class Single:
    """R train() runs, one generation each in turn."""

    def __init__(self, cs):
        self.runs = [(c,) + genetic.build(c) for c in cs]

    def generation(self):
        for c, worker, ga in self.runs:
            f = worker.run(ga)
            worker.steps(ga.N)
            float(f.max())
            ga.tell(f)
            genetic.test(c, ga.best, None, worker=worker)
            worker.merge_obs_stats(ga.N)
        torch.cuda.synchronize()


class Sweep:
    """One train_sweep generation of every run; `split` times its phases."""

    def __init__(self, cs):
        self.cs = cs
        self.worker, self.ga = genetic.build_sweep(cs)

    def generation(self, split=None):
        worker, ga, c = self.worker, self.ga, self.cs[0]
        clock = [time.perf_counter()]

        def mark(name):
            if split is not None:
                torch.cuda.synchronize()
                t = time.perf_counter()
                split[name] = split.get(name, 0.0) + (t - clock[0]) * 1e3
                clock[0] = t
        f = worker.run(ga)
        mark('eval')
        worker.steps(ga.N)
        f.max(dim=1).values.cpu()
        mark('host')
        ga.tell(f)
        mark('select')
        rows = torch.stack([b.reshape(-1) for b in ga.best]).contiguous()
        worker.test_returns(rows, c.test_repetitions, ga.running)
        mark('test')
        worker.merge_obs_stats(ga.running)
        torch.cuda.synchronize()
        mark('host')


def window(arm, gens):
    """ms per generation over `gens` generations, after a warm-up of `gens` generations."""
    for _ in range(gens):
        arm.generation()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(gens):
        arm.generation()
    return (time.perf_counter() - t) * 1e3 / gens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gens', type=int, default=4)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_ga_sweep.py measures on a GPU; none is available')
    rows = []
    for env in ('pendulum', 'noop'):
        for H in (16, 64):
            for R in (1, 4, 10, 32):
                cs = configs(env, H, R)
                single, sweep = Single(copy.deepcopy(cs)), Sweep(cs)
                t_single, t_sweep = [], []
                for _ in range(args.rounds):
                    t_single.append(window(single, args.gens))
                    t_sweep.append(window(sweep, args.gens))
                split = {}
                for _ in range(args.gens):
                    sweep.generation(split=split)
                row = dict(env=env, H=H, R=R, N=POP, window_gens=args.gens,
                           sequential_ms=round(statistics.median(t_single), 3), sweep_ms=round(statistics.median(t_sweep), 3),
                           split_ms={k: round(v / args.gens, 3) for k, v in split.items()})
                row['speedup'] = round(row['sequential_ms'] / row['sweep_ms'], 2)
                print(json.dumps(row), flush=True)
                rows.append(row)
    result = dict(card=card(), rows=rows)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
