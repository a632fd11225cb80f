"""Configuration surface of the reference (config.py:5-53): same attribute names, the tape env in place
of gym.  `sigma` and `learning_rate` are set by all_tasks() in the reference (natural_es.py:143-144);
they get those values as defaults here.  New attributes: tape_len (T), seed, precision, device.
"""
from __future__ import annotations

import numpy as np

from .envs import DeviceEnv, TapeEnv
from .fitness import POLICY_WIDTHS
from .model import StandardFCNet
from .utils import Adam


class BasicConfig:
    def __init__(self, hidden_size):
        if not hasattr(self, 'env_fn'):
            self.env_fn = lambda: TapeEnv(self.state_dim_, self.action_dim_, self.tape_len)
        self.repetitions = 1          # the tape is deterministic: one episode per evaluation (reference: 10)
        self.test_repetitions = 1
        env = self.env_fn()
        self.action_dim = env.action_space.shape[0]
        self.state_dim = env.observation_space.shape[0]
        self.hidden_size = hidden_size
        self.model_fn = lambda: StandardFCNet(self.state_dim, self.action_dim, self.hidden_size, seed=0)
        model = self.model_fn()
        self.initial_weight = model.get_weight()
        self.reward_to_fitness = lambda r: r
        self.pop_size = 30
        self.num_workers = 1          # = GPUs (one process per GPU); set by the launcher
        self.max_steps = 0
        self.opt = Adam()
        self.weight_decay = 0.005
        self.action_noise_std = 0
        self.tag = ''
        self.sigma = 0.1              # natural_es.py:143
        self.learning_rate = 0.1      # natural_es.py:144
        self.seed = 0
        self.precision = 'fp32'
        self.max_generations = 0      # 0 = unbounded (stop on max_steps like the reference)
        self.normalize_obs = False    # True = the reference's StaticNormalizer/SharedStats behaviour (utils.py:37-106)
        self.mirrored = False         # True = mirrored sampling for NES: members 2p, 2p+1 are theta +- sigma*eps_p (even pop_size)


class SynthTapeConfig(BasicConfig):
    def __init__(self, hidden_size=64, state_dim=24, action_dim=4, tape_len=256, clip=1.0):
        self.task = 'SynthTape-d%d-a%d-T%d-v0' % (state_dim, action_dim, tape_len)
        self.state_dim_, self.action_dim_, self.tape_len = state_dim, action_dim, tape_len
        self.clip = float(clip)
        self.action_clip = lambda a: np.clip(a, -clip, clip)
        self.target = 10000
        BasicConfig.__init__(self, hidden_size)


class PendulumConfig(SynthTapeConfig):
    """Pendulum-v0 shapes (config.py:26-31): obs 3, action 1, clip 2, 200-step episodes."""

    def __init__(self, hidden_size=16, tape_len=200):
        SynthTapeConfig.__init__(self, hidden_size, 3, 1, tape_len, 2.0)


class ClosedLoopPendulumConfig(BasicConfig):
    """The reference's PendulumConfig (config.py:26-31) with the environment stepped on the device: 10 repetitions of
    200-step episodes per member (config.py:8-9), per-member observations, observation normaliser on."""

    def __init__(self, hidden_size=64):
        # limits of des_rollout_eval (csrc/des_envs.cu): checked here, not at the first generation.  16 is the reference's
        # own PendulumConfig default (config.py:27) and the width its CMA-ES driver uses (cma_es.py:129).
        if hidden_size not in POLICY_WIDTHS:
            raise ValueError('ClosedLoopPendulumConfig: hidden_size must be one of %s on the device path (got %r)'
                             % (POLICY_WIDTHS, hidden_size))
        self.task = 'Pendulum-v0'
        self.clip = 2.0
        self.action_clip = lambda a: np.clip(a, -2, 2)
        self.target = 10000
        self.tape_len = DeviceEnv.SPECS[self.task]['horizon']
        self.env_fn = lambda: DeviceEnv(self.task)
        BasicConfig.__init__(self, hidden_size)
        self.closed_loop = True
        self.repetitions = 10         # config.py:8
        self.test_repetitions = 10    # config.py:9
        self.normalize_obs = True


class BipedalWalkerConfig(SynthTapeConfig):
    """BipedalWalker-v2 shapes (config.py:34-39): obs 24, action 4, clip 1."""

    def __init__(self, hidden_size=16, tape_len=256):
        SynthTapeConfig.__init__(self, hidden_size, 24, 4, tape_len, 1.0)


class HostEnvConfig(BasicConfig):
    """Any environment with the classic gym API (reset() -> obs, step(a) -> (obs, reward, done, info), optionally
    seed(s)), stepped on the host by the user's own code, with the population's policy step on the device
    (fitness.HostRollouts, for NES and CMA-ES).  The reference's BasicConfig (config.py:5-21): env_fn is
    probed for state_dim / action_dim, 10 repetitions and 10 test repetitions (config.py:8-9), the observation
    normaliser on.  `batch_env_fn(num_slots)`, if given, builds a vectorised environment implementing the batch protocol
    of envs.py (otherwise envs.GymEnvBatch wraps num_slots environments from env_fn)."""

    def __init__(self, env_fn, hidden_size=16, clip=1.0, task=None, batch_env_fn=None):
        if hidden_size not in POLICY_WIDTHS:
            raise ValueError('HostEnvConfig: hidden_size must be one of %s (des_policy_act); got %r'
                             % (POLICY_WIDTHS, hidden_size))
        self.env_fn = env_fn
        self.batch_env_fn = batch_env_fn
        self.task = task if task is not None else 'host-env'
        self.clip = float(clip)
        self.action_clip = lambda a: np.clip(a, -self.clip, self.clip)
        self.target = 10000
        BasicConfig.__init__(self, hidden_size)
        if not (1 <= self.state_dim <= 32 and 1 <= self.action_dim <= 8):
            raise ValueError('HostEnvConfig: des_policy_act takes state_dim <= 32 and action_dim <= 8; the environment '
                             'has %d and %d' % (self.state_dim, self.action_dim))
        self.host_env = True
        self.repetitions = 10         # config.py:8
        self.test_repetitions = 10    # config.py:9
        self.normalize_obs = True


class GymConfig(HostEnvConfig):
    """A gym task by name, e.g. GymConfig('BipedalWalker-v2', 64): gym.make(task) with the action clip of the
    reference's config for that task (config.py:29, 37, 44, 51; 1 for tasks it does not list).  Needs the `gym`
    package with the classic API; it is imported when the config is constructed."""

    CLIPS = {'Pendulum-v0': 2.0, 'BipedalWalker-v2': 1.0, 'LunarLanderContinuous-v2': 1.0,
             'BipedalWalkerHardcore-v2': 1.0}

    def __init__(self, task, hidden_size=16):
        try:
            import gym
        except ImportError as e:
            raise ImportError('GymConfig(%r) needs the gym package (classic API: reset() -> obs, step(a) -> '
                              '(obs, reward, done, info)), which is not installed; or pass any such environment '
                              'factory to HostEnvConfig' % (task,)) from e
        HostEnvConfig.__init__(self, lambda: gym.make(task), hidden_size, self.CLIPS.get(task, 1.0), task)
