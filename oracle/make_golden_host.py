#!/usr/bin/env python
"""Generate tests/golden/train_host_walk.npz by running the REFERENCE's natural_es.train() verbatim on 'SynthWalk-v0'
(oracle/synth_walk.py): the golden of training on an environment stepped on the host.

TEST INFRASTRUCTURE.  Runs only where the reference checkout exists; reuses oracle/make_golden.py's setup (paths, the
gym stand-in, the Philox noise for np.random.randn, the recording Adam) without changing it and rewrites no other
fixture.

    python oracle/make_golden_host.py

Hooks, as in make_golden.py::golden_train_closed: Philox noise for np.random.randn, the recording Adam, and a reset hook so
episode k of the single worker starts from the episode seed of (generation, member, repetition) and the master's test()
episodes from the test member's.  'SynthWalk-v0' is added to the gym stand-in's make() for this run only.
H = 64, N = 16, 10 repetitions, 3 generations, normaliser on.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg             # noqa: E402  (sets up sys.path: gym stand-in, reference, repository)

import numpy as np                    # noqa: E402
import torch                          # noqa: E402
import gym                            # noqa: E402  the stand-in
from oracle import synth_walk as sw   # noqa: E402


def golden_train_host(tag, H, N, reps, seed, sigma, lr, gens):
    instances = [0]

    class HookedWalk(sw.SynthWalkEnv):
        def __init__(self, instance):
            sw.SynthWalkEnv.__init__(self)
            self.instance, self.episode = instance, 0

        def reset(self):
            if self.instance == 1:                                       # the worker's environment
                g, rest = divmod(self.episode, N * reps)
                member, rep = divmod(rest, reps)
            else:                                                        # test(g): instance 2 + g
                g, member, rep = self.instance - 2, sw.TEST_MEMBER, self.episode
            self.seed(sw.episode_seed(seed, g, member, rep))
            self.episode += 1
            return sw.SynthWalkEnv.reset(self)

    real_make = gym.make

    def make(task):
        if task == 'SynthWalk-v0':
            instances[0] += 1
            return HookedWalk(instances[0] - 1)                          # 0 = config probe, 1 = worker, 2 + g = test(g)
        return real_make(task)

    class WalkConfig(mg.ref_config.BasicConfig):
        def __init__(self, hidden_size):
            self.task = 'SynthWalk-v0'
            self.action_clip = lambda a: np.clip(a, -1, 1)
            self.target = 10000
            mg.ref_config.BasicConfig.__init__(self, hidden_size)

    gym.make = make
    torch.manual_seed(0)
    try:
        cfg = WalkConfig(H)
    finally:
        gym.make = real_make
    cfg.repetitions = reps
    cfg.test_repetitions = reps
    cfg.num_workers = 1
    cfg.pop_size = N
    cfg.sigma = sigma
    cfg.learning_rate = lr
    cfg.opt = mg.RecordingAdam()
    P = len(cfg.initial_weight)
    theta0 = cfg.initial_weight.astype(np.float32)
    counter = {'k': 0, 'steps': []}
    real_randn = np.random.randn

    def philox_randn(*shape):
        n = shape[0]
        if n == P:
            g, member = divmod(counter['k'], N)
            counter['k'] += 1
            return mg.orc.noise(seed, g, member, 1, P)[0]
        return np.zeros(n)

    stats_log = []
    real_merge = mg.ref_utils.SharedStats.merge

    def logging_merge(self, B):
        real_merge(self, B)
        stats_log.append(np.concatenate([self.m.numpy(), self.v.numpy(), self.n.numpy()]).copy())

    # train() stops once total_steps > max_steps after collecting a generation (natural_es.py:82-84): with episode
    # lengths that vary, stop on the generation count instead — a step budget no generation can reach, then a bound set
    # from the steps actually taken, which only the collection after the `gens`-th update exceeds.
    real_update = cfg.opt.update

    def update_and_budget(g):
        step = real_update(g)
        if len(cfg.opt.rec_g) == gens:
            cfg.max_steps = 1                                            # the next collection ends the run
        return step
    cfg.opt.update = update_and_budget
    cfg.max_steps = 1 << 62
    np.random.randn = philox_randn
    gym.make = make
    mg.ref_utils.SharedStats.merge = logging_merge
    try:
        rewards, steps, _ = mg.ref_nes.train(cfg)
    finally:
        np.random.randn = real_randn
        gym.make = real_make
        mg.ref_utils.SharedStats.merge = real_merge
    assert len(cfg.opt.rec_g) == gens, (len(cfg.opt.rec_g), gens)
    param = torch.FloatTensor(torch.from_numpy(theta0.copy()))
    thetas = []
    for st in cfg.opt.rec_step:
        param.add_(cfg.learning_rate * torch.FloatTensor(st))
        thetas.append(param.numpy().copy())
    np.savez(os.path.join(mg.OUT, 'train_host_%s.npz' % tag), H=H, N=N, reps=reps, seed=seed, sigma=sigma, lr=lr,
             wd=cfg.weight_decay, gens=gens, theta0=theta0, grad_after_wd=np.stack(cfg.opt.rec_g),
             adam_step=np.stack(cfg.opt.rec_step), theta=np.stack(thetas), stats=np.stack(stats_log),
             test_rewards=np.asarray(rewards, dtype=np.float64), train_steps=np.asarray(steps))


if __name__ == '__main__':
    golden_train_host('walk', 64, 16, 10, seed=9, sigma=0.1, lr=0.1, gens=3)
    f = os.path.join(mg.OUT, 'train_host_walk.npz')
    print(f, os.path.getsize(f))
