"""Minimal stand-in for the ``gym`` package so the reference's config.py, natural_es.py and cma_es.py import and run
verbatim here (``gym`` is not installed; config.py:1 imports it).  TEST INFRASTRUCTURE ONLY — used by
oracle/make_golden.py and oracle/ref_cpu_baseline.py, never by the product package.

``gym.make(task)`` knows three tasks:
  'Pendulum-v0'                    the restated Pendulum (PendulumEnv)
  'SynthWalk-v0'                   oracle/synth_walk.py's host-stepped test environment
  'SynthTape-d<d0>-a<A>-T<T>-v0'   the synthetic observation tape of SURVEY.md §8d: a fixed tape X[T,d0], targets
                                   a*[T,A]; reward r_t = -||a_t - a*_t||^2 for the (already clipped, utils.py:134)
                                   action the agent passes; the episode ends after T steps.
The oracle modules are imported only when a task needs them, so the tape task runs with nothing but numpy.

Episode keys: make() numbers every instance it returns from the counter ``instances``; a run that keys its episodes
installs a fresh ``itertools.count()`` first, so that in a one-worker train() 0 = the config probe, 1 = the worker and
2 + g = test() number g.  ``reset_hook(instance, episode)`` (module attribute), when set, gives the start of every
Pendulum and SynthWalk episode: (theta, theta_dot) for Pendulum, the episode seed for SynthWalk.  Unset, Pendulum draws
uniform(-[pi, 1], [pi, 1]) and SynthWalk resets from its current seed.
"""
import itertools
import re

import numpy as np

reset_hook = None
instances = itertools.count()


class _Box:
    def __init__(self, shape):
        self.shape = shape


class SynthTapeEnv:
    def __init__(self, d0, A, T, seed=1234):
        rs = np.random.RandomState(seed)
        self.obs = rs.randn(T, d0).astype(np.float32)
        self.target = np.tanh(rs.randn(T, A)).astype(np.float32)
        self.T = T
        self.observation_space = _Box((d0,))
        self.action_space = _Box((A,))
        self.t = 0

    def reset(self):
        self.t = 0
        return self.obs[0]

    def step(self, action):
        a = np.asarray(action, dtype=np.float64).reshape(-1)
        d = a - self.target[self.t].astype(np.float64)
        reward = -float(np.dot(d, d))
        self.t += 1
        done = self.t >= self.T
        obs = self.obs[self.t] if not done else np.zeros_like(self.obs[0])
        return obs, reward, done, {}


class PendulumEnv:
    """'Pendulum-v0' of OpenAI gym (classic_control/pendulum.py + the 200-step TimeLimit wrapper): state (theta,
    theta_dot) in float64, stepped by oracle.pendulum_oracle.pendulum_step, the one restatement of its dynamics."""
    horizon = 200

    def __init__(self, instance):
        self.instance = instance
        self.episode = 0
        self.np_random = np.random.RandomState(instance)
        self.observation_space = _Box((3,))
        self.action_space = _Box((1,))

    def _obs(self):
        th, thdot = self.state
        return np.array([np.cos(th), np.sin(th), thdot])

    def reset(self):
        if reset_hook is not None:
            self.state = np.asarray(reset_hook(self.instance, self.episode), dtype=np.float64)
        else:
            high = np.array([np.pi, 1.0])
            self.state = self.np_random.uniform(low=-high, high=high)
        self.episode += 1
        self.t = 0
        return self._obs()

    def step(self, u):
        from oracle.pendulum_oracle import pendulum_step
        th, thdot = self.state
        th, thdot, reward = pendulum_step(th, thdot, u[0])
        self.state = np.array([th, thdot])
        self.t += 1
        return self._obs(), reward, self.t >= self.horizon, {}


class SeededEpisodes:
    """A seed()-able environment (SynthWalk-v0) whose episodes are numbered like PendulumEnv's: reset_hook, when set,
    gives each episode's seed."""

    def __init__(self, env, instance):
        self.env, self.instance, self.episode = env, instance, 0
        self.observation_space, self.action_space = env.observation_space, env.action_space

    def reset(self):
        if reset_hook is not None:
            self.env.seed(reset_hook(self.instance, self.episode))
        self.episode += 1
        return self.env.reset()

    def step(self, action):
        return self.env.step(action)


def make(task):
    instance = next(instances)
    if task == 'Pendulum-v0':
        return PendulumEnv(instance)
    if task == 'SynthWalk-v0':
        from oracle import synth_walk
        return SeededEpisodes(synth_walk.SynthWalkEnv(), instance)
    m = re.fullmatch(r'SynthTape-d(\d+)-a(\d+)-T(\d+)-v0', task)
    if m is None:
        raise ValueError('gym stand-in only knows Pendulum-v0, SynthWalk-v0 and SynthTape-d<d0>-a<A>-T<T>-v0, got %r'
                         % (task,))
    return SynthTapeEnv(int(m.group(1)), int(m.group(2)), int(m.group(3)))
