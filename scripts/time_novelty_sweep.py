"""Time a sweep of R NSR-ES runs (w = 0.5, N = 64, one agent each) two ways: one novelty.train_sweep generation
(NoveltySweep: one launch per step for every run) and R novelty.train generations one after another (one NoveltySearch
per run).  A generation is train()'s loop body: the test (behaviour archived), the evaluation (fitness and behaviours),
novelty, shaping, gradient and Adam.

  pendulum  closed-loop Pendulum-v0 on the device (ClosedLoopPendulumConfig: 10 repetitions of 200 steps), H in {16, 64},
            R in {1, 4, 10, 32}.
  host      Pendulum-v0 stepped on the host by oracle.pendulum_oracle.PendulumBatch (HostEnvConfig, 10 repetitions of 200
            steps), H = 16, R = 10: what the host bridge itself costs.

Every shape is warmed up for --warmup generations in both arms; then --trials generations are timed with CUDA events,
the two arms alternating generation by generation, and the medians are printed.  The archive grows by one row a
generation, so it ends at 1 + warmup + trials rows.  After every timed generation the two arms' fitness must be equal bit
for bit, run by run.  Prints one JSON line per shape and one with the card's name, power limit and SM clock limit, read in
the same call.

    python scripts/time_novelty_sweep.py [--warmup 3] [--trials 15] [--out results.json]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from distributedes_b200 import novelty                                         # noqa: E402
from distributedes_b200.config import ClosedLoopPendulumConfig, HostEnvConfig  # noqa: E402
from host_env_support import PendulumProbe                                     # noqa: E402
from oracle import pendulum_oracle as po                                       # noqa: E402
from time_runs import card                                                     # noqa: E402

POP = 64


def configs(env, H, R):
    out = []
    for r in range(R):
        if env == 'pendulum':
            c = ClosedLoopPendulumConfig(H)
        else:
            c = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0,
                              batch_env_fn=lambda B, s=1000 + r: po.PendulumBatch(B, s))
            c.repetitions = c.test_repetitions = 10
        c.pop_size, c.seed, c.sigma, c.ns_reward_weight = POP, 1000 + r, 0.05, 0.5
        c.initial_weight = c.initial_weight.copy()
        out.append(c)
    return out


class Sequential:
    """R novelty.train runs, one generation each in turn."""

    def __init__(self, cs):
        self.cs, self.runs = cs, [novelty.build(c) for c in cs]

    def generation(self):
        for c, ns in zip(self.cs, self.runs):
            _, _, improved = ns.test_agent(0, c.test_repetitions)
            ns.adapt(improved)
            ns.evaluate(0)
            ns.step(0)

    def fitness(self):
        return torch.stack([ns.agents[0].fitness_all for ns in self.runs])


class Sweep:
    """One novelty.train_sweep generation of every run."""

    def __init__(self, cs):
        self.cs, self.ns = cs, novelty.build_sweep(cs)

    def generation(self):
        ns = self.ns
        for r, t in enumerate(ns.test(self.cs[0].test_repetitions)):
            ns.adapt(r, t[2])
        ns.evaluate()
        ns.step()

    def fitness(self):
        return self.ns.engine.fitness_all


def timed(arm):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    arm.generation()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def measure(env, H, R, warmup, trials):
    cs = configs(env, H, R)
    seq, sweep = Sequential(cs), Sweep(configs(env, H, R))
    for _ in range(warmup):
        seq.generation()
        sweep.generation()
    t_seq, t_sweep = [], []
    for _ in range(trials):
        t_seq.append(timed(seq))
        t_sweep.append(timed(sweep))
        if not np.array_equal(seq.fitness().cpu().numpy().view(np.uint32), sweep.fitness().cpu().numpy().view(np.uint32)):
            raise SystemExit('%s H=%d R=%d: the sweep\'s fitness is not the sequential runs\' bit for bit' % (env, H, R))
    row = dict(env=env, H=H, R=R, N=POP, archive_rows=sweep.ns.size, trials=trials,
               sequential_ms=round(statistics.median(t_seq), 3), sweep_ms=round(statistics.median(t_sweep), 3),
               fitness_bit_equal=True)
    row['speedup'] = round(row['sequential_ms'] / row['sweep_ms'], 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--trials', type=int, default=15)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_novelty_sweep.py measures on a GPU; none is available')
    the_card = card()
    rows = []
    shapes = [('pendulum', H, R) for H in (16, 64) for R in (1, 4, 10, 32)] + [('host', 16, 10)]
    for env, H, R in shapes:
        row = measure(env, H, R, args.warmup, args.trials if env == 'pendulum' else max(3, args.trials // 3))
        print(json.dumps(row), flush=True)
        rows.append(row)
    result = dict(card=the_card, rows=rows)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
