#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the REFERENCE's own code (imported from /root/reference).

TEST INFRASTRUCTURE.  Runs only where the reference checkout exists; the fixtures it writes are committed so the tests,
which run without the reference, can check the oracle and the CUDA path against the reference's outputs.

    python oracle/make_golden.py                                         # rewrites every fixture in FIXTURES
    python oracle/make_golden.py train_host_walk train_cma_closed_pend   # only the fixtures named

What comes from where:
  * fitness_shift, Adam                  -> /root/reference/utils.py:142-166, called directly
  * StandardFCNet forward / flat codec   -> /root/reference/model.py:7-39, called directly
  * per-member fitness                   -> /root/reference/utils.py:108-139 Evaluator.eval over the stand-in gym's
                                            tape task (oracle/gym_stub)
  * train_*                              -> natural_es.train() (natural_es.py:34-99) or cma_es.train() (cma_es.py:31-111)
                                            run VERBATIM with one worker, on the stand-in gym's tape task,
                                            Pendulum-v0 (the reference's own PendulumConfig) or SynthWalk-v0
                                            (oracle/synth_walk.py); cma_es.py's `cma` (pycma) is oracle/cma_stub.

run_train() installs the hooks of one verbatim run and restores every one of them when it returns or raises:
  * np.random.randn(P) of the worker (natural_es.py:29) serves the Philox row of (generation, member) — plain
    oracle.nes_oracle.noise or the mirrored row of oracle.mirrored_oracle.noise_mirrored; every other draw (the action
    noise, utils.py:133, times action_noise_std = 0; all of cma_es.train()'s draws) returns zeros.  The noise stream is
    the one non-reference ingredient: the reference has no reproducible RNG (natural_es.py:23 seeds from OS entropy).
  * SharedStats.merge is disabled (observation normaliser off, SURVEY §8d) or records the statistics after each merge.
  * gym.reset_hook starts episode (instance, episode) from its (generation, member, repetition) key, episode_key().
  * fitness_shift records the costs it ranks and stops the run after `gens` updates: train() ends once total_steps >
    max_steps after collecting a generation (natural_es.py:82-84, cma_es.py:85-87), so the step budget stays out of
    reach until the gens-th update and drops below the steps taken after it, whatever the episode lengths.
config.opt is a recording subclass of the reference Adam, from whose steps train_nes() replays theta in torch.
Each fixture is one entry of FIXTURES: a driver and its parameters; a closed-loop task is one entry of ENVS.
"""
import contextlib
import itertools
import os
import sys
from unittest import mock

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF = '/root/reference'
sys.path.insert(0, os.path.join(HERE, 'cma_stub'))
sys.path.insert(0, os.path.join(HERE, 'gym_stub'))
sys.path.insert(0, REF)
sys.path.insert(0, REPO)

import numpy as np
import torch

torch.set_num_threads(1)

import cma                           # noqa: E402  oracle/cma_stub
import gym                           # noqa: E402  oracle/gym_stub
import utils as ref_utils            # noqa: E402  /root/reference/utils.py
import model as ref_model            # noqa: E402  /root/reference/model.py
import config as ref_config          # noqa: E402  /root/reference/config.py
import natural_es as ref_nes         # noqa: E402  /root/reference/natural_es.py
import cma_es as ref_cma             # noqa: E402  /root/reference/cma_es.py
from oracle import mirrored_oracle   # noqa: E402
from oracle import nes_oracle as orc  # noqa: E402
from oracle import pendulum_oracle as po  # noqa: E402
from oracle import synth_walk as sw  # noqa: E402

OUT = os.path.join(REPO, 'tests', 'golden')
ref_utils.logger.setLevel('WARNING')


def golden_fitness_shift():
    rs = np.random.RandomState(7)
    out = {}
    for i, n in enumerate([2, 3, 16, 257, 4096]):
        x = rs.randn(n).astype(np.float32)
        assert len(np.unique(x)) == n          # tie-free: the reference's argsort is unstable on ties
        out['x%d' % i] = x
        out['y%d' % i] = ref_utils.fitness_shift(x)
    # list input, as natural_es.py:90 passes a python list
    out['x5'] = np.asarray([3.0, -1.0, 2.5, 0.0, 10.0], dtype=np.float32)
    out['y5'] = ref_utils.fitness_shift([3.0, -1.0, 2.5, 0.0, 10.0])
    return out


def golden_adam():
    rs = np.random.RandomState(11)
    P, steps = 37, 6
    g = rs.randn(steps, P) * np.logspace(-3, 1, P)[None, :]
    opt = ref_utils.Adam()
    outs = np.stack([opt.update(g[t]) for t in range(steps)])
    return dict(g=g, step=outs, m=opt.m, v=opt.v, beta1_t=opt.beta1_t, beta2_t=opt.beta2_t)


def golden_forward():
    out = {}
    rs = np.random.RandomState(3)
    for tag, (d0, H, A, T) in {'pend': (3, 64, 1, 8), 'b64': (24, 64, 4, 8), 'b256': (24, 256, 4, 4)}.items():
        net = ref_model.StandardFCNet(d0, A, H)
        P = orc.param_count(d0, H, A)
        flat = (rs.randn(P) * 0.2).astype(np.float32)
        net.set_weight(flat.astype(np.float64))          # fp64 in, stored fp32 (model.py:23)
        assert np.array_equal(net.get_weight(), flat)    # codec round trip
        obs = rs.randn(T, d0).astype(np.float32)
        act = net(obs).data.numpy()
        out[tag + '_dims'] = np.asarray([d0, H, A, T])
        out[tag + '_flat'] = flat
        out[tag + '_obs'] = obs
        out[tag + '_act'] = act
        # named-parameter view, to pin the flat layout independently of our unflatten()
        out[tag + '_fc1w'] = net.fc1.weight.data.numpy()
        out[tag + '_fc1b'] = net.fc1.bias.data.numpy()
        out[tag + '_fc2w'] = net.fc2.weight.data.numpy()
        out[tag + '_fc2b'] = net.fc2.bias.data.numpy()
        out[tag + '_fc3w'] = net.fc3.weight.data.numpy()
        out[tag + '_fc3b'] = net.fc3.bias.data.numpy()
    return out


class TaskConfig(ref_config.BasicConfig):
    """config.py:34-39's shape on a stand-in task: actions clipped to +-clip, target 10000."""

    def __init__(self, task, clip, hidden):
        self.task = task
        self.action_clip = lambda a: np.clip(a, -clip, clip)
        self.target = 10000
        ref_config.BasicConfig.__init__(self, hidden)


def tape_config(d0, A, T, clip, H):
    return TaskConfig('SynthTape-d%d-a%d-T%d-v0' % (d0, A, T), clip, H)


def pendulum_start(seed, g, member, rep):
    th, thd = po.reset_states(seed, g, [member], rep + 1)
    return th[0, rep], thd[0, rep]


# closed-loop tasks: the reference config for hidden width H, and the start of episode (generation, member, repetition)
ENVS = {
    'Pendulum-v0': (lambda H: ref_config.PendulumConfig(hidden_size=H), pendulum_start),
    'SynthWalk-v0': (lambda H: TaskConfig('SynthWalk-v0', 1, H), sw.episode_seed),
}


def episode_key(instance, episode, N, reps):
    """(generation, member, repetition) of episode `episode` of gym instance `instance` in a one-worker train(): the
    worker (instance 1) runs members in order, `reps` episodes each; test() number g (instance 2 + g) runs the test
    member, whose key is shared by the Pendulum and SynthWalk streams."""
    if instance == 1:
        g, rest = divmod(episode, N * reps)
        return (g,) + divmod(rest, reps)
    return instance - 2, po.TEST_MEMBER, episode


class RecordingAdam(ref_utils.Adam):
    def __init__(self):
        ref_utils.Adam.__init__(self)
        self.rec_g, self.rec_step = [], []

    def update(self, g):
        self.rec_g.append(np.array(g, dtype=np.float64))
        step = ref_utils.Adam.update(self, g)
        self.rec_step.append(np.array(step, dtype=np.float64))
        return step


def golden_eval(d0, H, A, T, clip, N, seed, sigma):
    """Per-member fitness from the reference Evaluator (utils.py:116-124), noise from the oracle."""
    torch.manual_seed(0)
    cfg = tape_config(d0, A, T, clip, H)
    cfg.repetitions = 1
    norm = ref_utils.StaticNormalizer(cfg.state_dim)     # offline n == 0 -> identity (utils.py:48-49)
    ev = ref_utils.Evaluator(cfg, norm)
    theta = cfg.initial_weight.astype(np.float32)
    P = len(theta)
    eps = orc.noise(seed, 0, 0, N, P)
    fit = np.empty(N)
    steps = np.empty(N, dtype=np.int64)
    for i in range(N):
        disturbed = np.copy(theta)                        # natural_es.py:28
        disturbed += sigma * eps[i]                       # natural_es.py:30
        cost, st = ev.eval(disturbed)                     # natural_es.py:31
        fit[i] = -cost                                    # natural_es.py:32
        steps[i] = st
    return dict(dims=np.asarray([d0, H, A, T]), clip=clip, N=N, seed=seed, sigma=sigma, theta=theta, fitness=fit,
                steps=steps)


def run_train(trainer, make_config, *, N, reps, test_reps, seed, sigma, gens, lr=None, noise='plain',
              normalizer=True, episode_start=None, patches=()):
    """trainer.train(cfg) VERBATIM with one worker, inside the hooks of the module docstring.

    noise: 'plain', 'mirrored' or None (zeros only); normalizer: False disables SharedStats.merge, True records it;
    episode_start(seed, g, member, rep): the value gym.reset_hook returns for that episode, or None for no hook;
    patches: further (object, attribute, value) to install for the run.
    Returns (cfg, record): record holds test_rewards, train_steps, theta0 and the merged stats and ranked costs."""
    stats, costs = [], []
    with contextlib.ExitStack() as scope:
        def patch(obj, name, value):
            scope.enter_context(mock.patch.object(obj, name, value))

        patch(gym, 'instances', itertools.count())           # gym.make() numbering starts at the config probe
        torch.manual_seed(0)
        cfg = make_config()
        cfg.repetitions, cfg.test_repetitions, cfg.num_workers, cfg.pop_size = reps, test_reps, 1, N
        cfg.sigma, cfg.learning_rate, cfg.opt = sigma, lr, RecordingAdam()
        cfg.max_steps = 1 << 62
        P = len(cfg.initial_weight) if noise else None
        rows = mirrored_oracle.noise_mirrored if noise == 'mirrored' else orc.noise
        drawn = itertools.count()

        def randn(n):
            if n != P:
                return np.zeros(n)
            g, member = divmod(next(drawn), N)
            return rows(seed, g, member, 1, P)[0]

        real_merge, real_shift = ref_utils.SharedStats.merge, trainer.fitness_shift

        def recording_merge(self, B):
            real_merge(self, B)
            stats.append(np.concatenate([self.m.numpy(), self.v.numpy(), self.n.numpy()]).copy())

        def recording_shift(x):
            costs.append(np.asarray(x, dtype=np.float64).copy())
            if len(costs) == gens:
                cfg.max_steps = 1                            # the next collection ends the run
            return real_shift(x)

        patch(np.random, 'randn', randn)
        patch(ref_utils.SharedStats, 'merge', recording_merge if normalizer else lambda self, B: None)
        patch(trainer, 'fitness_shift', recording_shift)
        if episode_start is not None:
            patch(gym, 'reset_hook', lambda instance, episode:
                  episode_start(seed, *episode_key(instance, episode, N, reps)))
        for p in patches:
            patch(*p)
        rewards, steps, _ = trainer.train(cfg)
    assert len(costs) == gens, (len(costs), gens)
    return cfg, dict(test_rewards=np.asarray(rewards, dtype=np.float64), train_steps=np.asarray(steps),
                     theta0=cfg.initial_weight.astype(np.float32), stats=stats, costs=costs)


def train_nes(make_config, keys, *, gens, lr, **run):
    """natural_es.train() through run_train; returns the entries `keys` of its record, the parameters and the replay."""
    cfg, rec = run_train(ref_nes, make_config, gens=gens, lr=lr, **run)
    assert len(cfg.opt.rec_g) == gens, (len(cfg.opt.rec_g), gens)
    # replay natural_es.py:95-96 with torch to obtain theta after each generation
    param = torch.FloatTensor(torch.from_numpy(rec['theta0'].copy()))
    updates, thetas = [], []
    for st in cfg.opt.rec_step:
        upd = lr * torch.FloatTensor(st)
        param.add_(upd)
        updates.append(upd.numpy().copy())
        thetas.append(param.numpy().copy())
    rec.update(run, gens=gens, lr=lr, wd=cfg.weight_decay, grad_after_wd=np.stack(cfg.opt.rec_g),
               adam_step=np.stack(cfg.opt.rec_step), update=np.stack(updates), theta=np.stack(thetas),
               stats=np.stack(rec['stats']) if rec['stats'] else None)
    return {k: rec[k] for k in keys.split()}


def train_tape(d0, H, A, T, clip, **run):
    """The tape task, one episode per member and two per test()."""
    out = train_nes(lambda: tape_config(d0, A, T, clip, H),
                    'N seed sigma lr wd gens theta0 grad_after_wd adam_step update theta test_rewards train_steps',
                    reps=1, test_reps=2, **run)
    return dict(dims=np.asarray([d0, H, A, T]), clip=clip, **out)


def train_env(task, H, reps, **run):
    """A closed-loop task of ENVS, normaliser on, `reps` episodes per member and per test()."""
    config, start = ENVS[task]
    out = train_nes(lambda: config(H), 'N reps seed sigma lr wd gens theta0 grad_after_wd adam_step theta stats '
                    'test_rewards train_steps', reps=reps, test_reps=reps, episode_start=start, **run)
    return dict(H=H, **out)


def train_cma(task, H, lam, reps, seed, sigma, gens):
    """cma_es.train() through run_train over oracle/cma_stub, whose z comes from the counter noise (stream tag 1)."""
    config, start = ENVS[task]
    es = []
    cfg, rec = run_train(ref_cma, lambda: config(H), N=lam, reps=reps, test_reps=reps, seed=seed, sigma=sigma,
                         gens=gens, noise=None, episode_start=start,
                         patches=[(cma, 'noise_seed', seed), (cma, 'instances', es)])
    t = es[-1].told
    assert len(t) == gens and len(rec['stats']) == gens
    return dict(H=H, lam=lam, reps=reps, seed=seed, sigma=sigma, gens=gens, theta0=rec['theta0'],
                test_rewards=rec['test_rewards'], train_steps=rec['train_steps'], stats=np.stack(rec['stats']),
                costs=np.stack(rec['costs']), shaped=np.stack([r['cost'] for r in t]),
                solutions=np.stack([r['solutions'] for r in t]).astype(np.float32), m=np.stack([r['m'] for r in t]),
                sigmas=np.asarray([r['sigma'] for r in t]), pc=np.stack([r['pc'] for r in t]),
                ps=np.stack([r['ps'] for r in t]))


PEND_TAPE = dict(d0=3, H=64, A=1, T=32, clip=2.0, N=16, seed=5, sigma=0.1)
B64_TAPE = dict(d0=24, H=64, A=4, T=16, clip=1.0, N=24, seed=6, sigma=0.1)

# fixture name -> (driver, parameters); each driver returns the fixture's arrays in the order np.savez writes them
FIXTURES = {
    'fitness_shift': (golden_fitness_shift, {}),
    'adam': (golden_adam, {}),
    'forward': (golden_forward, {}),
    'eval_pend': (golden_eval, PEND_TAPE),
    'eval_b64': (golden_eval, B64_TAPE),
    'train_pend': (train_tape, dict(PEND_TAPE, lr=0.1, gens=3, normalizer=False)),
    'train_b64': (train_tape, dict(B64_TAPE, lr=0.1, gens=3, normalizer=False)),
    # the same with the reference's observation normaliser left on
    'train_norm_pend': (train_tape, dict(PEND_TAPE, lr=0.1, gens=3)),
    'train_norm_b64': (train_tape, dict(B64_TAPE, lr=0.1, gens=3)),
    # mirrored sampling: member m trains on (-1)^(m & 1) * noise(seed, g, m >> 1)
    'train_b64_mirrored': (train_tape, dict(B64_TAPE, lr=0.1, gens=3, normalizer=False, noise='mirrored')),
    # BASELINE configs[0]: Pendulum-v0, 2x64 MLP, population 16, 10 repetitions of 200 steps
    'train_closed_pend': (train_env, dict(task='Pendulum-v0', H=64, N=16, reps=10, seed=7, sigma=0.1, lr=0.1,
                                          gens=2)),
    'train_closed_mirrored_pend': (train_env, dict(task='Pendulum-v0', H=16, N=16, reps=10, seed=7, sigma=0.1,
                                                   lr=0.1, gens=2, noise='mirrored')),
    'train_host_walk': (train_env, dict(task='SynthWalk-v0', H=64, N=16, reps=10, seed=9, sigma=0.1, lr=0.1,
                                        gens=3)),
    'train_cma_closed_pend': (train_cma, dict(task='Pendulum-v0', H=16, lam=16, reps=10, seed=7, sigma=1.0,
                                              gens=3)),
}


if __name__ == '__main__':
    names = sys.argv[1:] or list(FIXTURES)
    unknown = [n for n in names if n not in FIXTURES]
    if unknown:
        sys.exit('unknown fixture(s) %s; known: %s' % (' '.join(unknown), ' '.join(FIXTURES)))
    os.makedirs(OUT, exist_ok=True)
    for name in names:
        driver, params = FIXTURES[name]
        path = os.path.join(OUT, name + '.npz')
        np.savez(path, **driver(**params))
        print(name, os.path.getsize(path))
