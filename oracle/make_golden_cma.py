#!/usr/bin/env python
"""Generate tests/golden/train_cma_closed_pend.npz by running the REFERENCE's own cma_es.train() verbatim.

TEST INFRASTRUCTURE, like oracle/make_golden.py (whose setup it reuses: the reference checkout and the stub gym on
sys.path); it runs only where the reference checkout exists, and the fixture it writes is committed.

    python oracle/make_golden_cma.py        # writes tests/golden/train_cma_closed_pend.npz only

What comes from where: cma_es.train() (cma_es.py:31-111) VERBATIM on the reference's PendulumConfig(hidden_size=16)
over the stub gym's restated Pendulum-v0, with the third-party `cma` package (pycma, absent here) replaced by
oracle/cma_stub: ask() / tell() over oracle/cma_oracle.CMAState, z from the device's counter noise (stream tag 1).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(HERE, 'cma_stub'))

import numpy as np                       # noqa: E402
import torch                             # noqa: E402

from oracle import make_golden as mg     # noqa: E402  (puts the reference and oracle/gym_stub on sys.path)
from oracle import pendulum_oracle as po  # noqa: E402


def golden_cma_closed(tag, H, lam, reps, seed, sigma, gens):
    """cma_es.train() VERBATIM on the reference's own PendulumConfig(hidden_size=H) over the stub gym's Pendulum-v0, with
    oracle/cma_stub standing in for pycma.  Hooks as in make_golden.golden_train_closed: np.random.randn (only the zero action noise
    draws it here), the reset hook (worker episode k -> (generation, member, repetition); the k-th test() call is
    instance first + 2 + k and resets from the test stream with generation word k), and a recording SharedStats.merge.
    fitness_shift is wrapped to record the raw costs it ranks."""
    import gym
    import cma
    ref_cma = __import__('cma_es')                  # the reference's cma_es.py (imports the stub `cma`)
    torch.manual_seed(0)
    first = gym._pendulum_instances[0]
    cfg = mg.ref_config.PendulumConfig(hidden_size=H)
    cfg.repetitions = reps
    cfg.test_repetitions = reps
    cfg.num_workers = 1
    cfg.pop_size = lam
    cfg.sigma = sigma                                # cma_es.py:147
    cfg.max_steps = (gens + 1) * lam * reps * po.HORIZON - 1     # gens + 1 evaluations, `gens` tell()s
    theta0 = cfg.initial_weight.astype(np.float32)
    real_randn = np.random.randn

    def zero_randn(*shape):
        return np.zeros(shape[0])                    # utils.py:133, multiplied by action_noise_std = 0

    def reset_hook(instance, episode):
        if instance == first + 1:                                        # the worker's environment
            g, rest = divmod(episode, lam * reps)
            member, rep = divmod(rest, reps)
        else:                                                            # the k-th test() call
            g, member, rep = instance - (first + 2), po.TEST_MEMBER, episode
        th, thd = po.reset_states(seed, g, [member], reps)
        return th[0, rep], thd[0, rep]

    stats_log, costs_log = [], []
    real_merge = mg.ref_utils.SharedStats.merge
    real_shift = ref_cma.fitness_shift

    def logging_merge(self, B):
        real_merge(self, B)
        stats_log.append(np.concatenate([self.m.numpy(), self.v.numpy(), self.n.numpy()]).copy())

    def logging_shift(x):
        costs_log.append(np.asarray(x, dtype=np.float64).copy())
        return real_shift(x)

    cma.noise_seed = seed
    del cma.instances[:]
    np.random.randn = zero_randn
    gym.pendulum_reset_hook = reset_hook
    mg.ref_utils.SharedStats.merge = logging_merge
    ref_cma.fitness_shift = logging_shift
    try:
        rewards, steps, _ = ref_cma.train(cfg)
    finally:
        np.random.randn = real_randn
        gym.pendulum_reset_hook = None
        mg.ref_utils.SharedStats.merge = real_merge
        ref_cma.fitness_shift = real_shift
    es = cma.instances[-1]
    assert len(es.told) == gens and len(stats_log) == gens
    t = es.told
    np.savez(os.path.join(mg.OUT, 'train_cma_closed_%s.npz' % tag), H=H, lam=lam, reps=reps, seed=seed, sigma=sigma, gens=gens,
             theta0=theta0, test_rewards=np.asarray(rewards, dtype=np.float64), train_steps=np.asarray(steps),
             stats=np.stack(stats_log), costs=np.stack(costs_log), shaped=np.stack([r['cost'] for r in t]),
             solutions=np.stack([r['solutions'] for r in t]).astype(np.float32), m=np.stack([r['m'] for r in t]),
             sigmas=np.asarray([r['sigma'] for r in t]), pc=np.stack([r['pc'] for r in t]),
             ps=np.stack([r['ps'] for r in t]))


if __name__ == '__main__':
    golden_cma_closed('pend', 16, 16, 10, seed=7, sigma=1.0, gens=3)
    print('train_cma_closed_pend.npz', os.path.getsize(os.path.join(mg.OUT, 'train_cma_closed_pend.npz')))
