"""Time a sweep of R NES runs of 64 members on host-stepped environments two ways: one HostEnvSweepEngine (every
environment step of every run is one des_policy_act_sweep launch, one copy each way and one synchronise) and R
HostEnvEngines one after another (one such step per run).  H in {16, 64}, 10 episodes per member (the reference's
repetitions), R in {1, 4, 10, 32}, on two vectorised batch environments (the envs.py protocol, obs 24, action 4):

  noop       zero observations and rewards, every episode 100 steps: what the bridge itself costs.
  synthwalk  oracle/synth_walk.py's SynthWalk-v0 dynamics stepped for all slots at once in numpy (episodes of 40-160
             steps; the resets seed each slot's state from its key as SynthWalkEnv does).

  generation  ms per generation of all R runs (wall clock; every generation ends in the host loop's synchronise), `iters`
              generations per window after a warm-up generation.  The two arms are timed in turn, `rounds` times; the
              median of each is reported.
  split       us per environment step of one instrumented generation per arm, run apart from the timed windows:
              kernel = CUDA events around each policy launch, env = wall time in the environments' reset and step, and
              rest = everything else in the generation per step (the copies and the synchronise, the host bookkeeping,
              and the per-generation launches: rows, ranking, the gradient, Adam).  For the sequential arm, steps are
              summed over the R runs.

Prints one JSON line with the card's name, power limit and SM clock limit, read in the same call.

    python scripts/time_host_sweep.py [--iters 2] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distributedes_b200 import ops, ops_runs                                  # noqa: E402
from distributedes_b200.engine import HostEnvEngine, HostEnvSweepEngine       # noqa: E402
from distributedes_b200.envs import episode_seed                              # noqa: E402
from distributedes_b200.model import StandardFCNet                            # noqa: E402
from oracle import synth_walk as sw                                          # noqa: E402
from time_runs import card                                                    # noqa: E402

POP, REPS, D0, A = 64, 10, 24, 4
ENV_TIME = [0.0]                  # seconds spent in the environments, summed by the instrumented generations


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


class SynthWalkBatch:
    """SynthWalk-v0 (oracle/synth_walk.py) for all slots at once: slot b resets to reset_state(episode_seed(seed, *key))
    and ends after episode_length of that state."""

    def __init__(self, B, seed):
        self.num_envs, self.seed = B, seed

    def reset(self, keys):
        self.s = np.stack([sw.reset_state(episode_seed(self.seed, *(int(v) for v in k))) for k in keys])
        self.T = np.array([sw.episode_length(s) for s in self.s])
        self.t = 0
        return self.s.copy()

    def step(self, actions, alive):
        a = np.asarray(actions, dtype=np.float64)
        ns = 0.8 * self.s + 0.2 * np.tanh(self.s @ sw.M.T) + a @ sw.B.T
        d = a - np.tanh(self.s @ sw.C.T)
        r = 0.5 * ns[:, 1] - 0.02 * (ns * ns).sum(1) - 0.1 * (d * d).sum(1)
        self.s, self.t = ns, self.t + 1
        return ns.copy(), r, self.t >= self.T


class Timed:
    """A batch environment whose reset and step add their wall time to ENV_TIME."""

    def __init__(self, env):
        self.env, self.num_envs = env, env.num_envs

    def reset(self, keys):
        t0 = time.perf_counter()
        try:
            return self.env.reset(keys)
        finally:
            ENV_TIME[0] += time.perf_counter() - t0

    def step(self, actions, alive):
        t0 = time.perf_counter()
        try:
            return self.env.step(actions, alive)
        finally:
            ENV_TIME[0] += time.perf_counter() - t0


class Kernels:
    """A kernels module whose policy launches are bracketed by CUDA events while `on`."""

    def __init__(self, module):
        self._m, self.__name__, self.on, self.events = module, module.__name__, False, []

    def __getattr__(self, name):
        f = getattr(self._m, name)
        if name not in ('policy_act', 'policy_act_sweep'):
            return f

        def call(*a, **kw):
            if not self.on:
                return f(*a, **kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = f(*a, **kw)
            e1.record()
            self.events.append((e0, e1))
            return out
        return call


def _env_fn(kind, seed):
    return (lambda B: Timed(NoopBatch(B))) if kind == 'noop' else (lambda B: Timed(SynthWalkBatch(B, seed)))


def _arms(kind, H, R):
    theta0 = StandardFCNet(D0, A, H, seed=0).get_weight()
    seeds, sigma = list(range(1, R + 1)), [(0.05, 0.1, 0.2)[r % 3] for r in range(R)]
    lr = [(0.02, 0.05, 0.1, 0.2)[r % 4] for r in range(R)]
    kw = dict(env_fn=None, hidden=H, pop_size=POP, theta0=theta0, state_dim=D0, action_dim=A, repetitions=REPS)
    k_sweep, k_seq = Kernels(ops_runs), Kernels(ops)
    sweep = HostEnvSweepEngine(runs=R, seeds=seeds, sigma=sigma, learning_rate=lr,
                               batch_env_fn=[_env_fn(kind, s) for s in seeds], kernels=k_sweep, **kw)
    singles = [HostEnvEngine(seed=seeds[r], sigma=sigma[r], learning_rate=lr[r], batch_env_fn=_env_fn(kind, seeds[r]),
                             kernels=k_seq, **kw) for r in range(R)]
    return (sweep.generation, k_sweep), (lambda: [e.generation() for e in singles], k_seq)


def _wall_ms(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return 1000 * (time.perf_counter() - t0) / iters


def _split(fn, k):
    """(steps, kernel us, env us, rest us per step) of one instrumented generation."""
    torch.cuda.synchronize()
    k.on, k.events, ENV_TIME[0] = True, [], 0.0
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    k.on = False
    n = len(k.events)
    kern = sum(e0.elapsed_time(e1) for e0, e1 in k.events) / 1000
    return n, 1e6 * kern / n, 1e6 * ENV_TIME[0] / n, 1e6 * (total - kern - ENV_TIME[0]) / n


def measure(kind, H, R, iters, rounds):
    arms = _arms(kind, H, R)
    for fn, _ in arms:                                     # warm-up: module loading, pinned buffers, environments
        fn()
    times = [[], []]
    for _ in range(rounds):
        for i, (fn, _) in enumerate(arms):
            times[i].append(_wall_ms(fn, iters))
    sweep_ms, seq_ms = (statistics.median(t) for t in times)
    row = dict(env=kind, hidden=H, runs=R, pop=POP, reps=REPS, sweep_generation_ms=round(sweep_ms, 3),
               seq_generation_ms=round(seq_ms, 3), seq_over_sweep=round(seq_ms / sweep_ms, 2))
    for name, (fn, k) in zip(('sweep', 'seq'), arms):
        n, kern, env, rest = _split(fn, k)
        row.update({name + '_steps': n, name + '_kernel_us': round(kern, 1), name + '_env_us': round(env, 1),
                    name + '_rest_us': round(rest, 1)})
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--runs', default='1,4,10,32')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_host_sweep.py measures on a GPU; none is available')
    torch.cuda.set_device(0)
    rows = []
    for kind in ('noop', 'synthwalk'):
        for H in (16, 64):
            for R in (int(r) for r in a.runs.split(',')):
                rows.append(measure(kind, H, R, a.iters, a.rounds))
                print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    res = dict(card=card(), generation=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
