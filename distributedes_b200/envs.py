"""Environments: the synthetic observation tape of SURVEY.md §8d, the shape descriptor of environments stepped on the
device, and the batch protocol of environments stepped on the host.

The reference steps a gym env per member per step (utils.py:126-139).  For the benchmark workload the
env is a fixed tape: observations X[T, d0] shared by all members, targets a*[T, A], reward
r_t = -||clip(a_t) - a*_t||^2, return = sum_t r_t.  The arrays here are what gets copied to the GPU;
stepping happens inside des_nes_eval.

Host-stepped environments (engine.HostEnvEngine, cma_es.Worker with a `host_env` config) talk to the engines through
one batch protocol and nothing else:

    num_envs                                   B, the number of slots (members x repetitions, member-major)
    reset(keys) -> obs[B, d0]                  keys: int64 [B, 3] = (generation word, global member, repetition)
    step(actions[B, A], alive[B]) -> (obs[B, d0], reward fp64[B], done bool[B])

Slots whose `alive` entry is False are not stepped; what step() returns for them is ignored.  A vectorised environment
implements the protocol directly; GymEnvBatch adapts B single environments with the classic gym API.
"""
from __future__ import annotations

import numpy as np


class _Box:
    def __init__(self, shape):
        self.shape = shape


class TapeEnv:
    def __init__(self, state_dim, action_dim, tape_len, seed=1234):
        rs = np.random.RandomState(seed)
        self.obs = rs.randn(tape_len, state_dim).astype(np.float32)
        self.target = np.tanh(rs.randn(tape_len, action_dim)).astype(np.float32)
        self.observation_space = _Box((state_dim,))
        self.action_space = _Box((action_dim,))
        self.tape_len = int(tape_len)


class DeviceEnv:
    """Shape descriptor of an environment that is stepped INSIDE des_rollout_eval (closed loop, per-member
    observations): there is no host-side step().  SPECS is the table of them; `env` is the library's environment id
    (DES_ENV_PENDULUM = 0).  'Pendulum-v0': config.py:26-31."""
    SPECS = {'Pendulum-v0': dict(env=0, state_dim=3, action_dim=1, horizon=200, clip=2.0)}

    def __init__(self, task):
        if task not in self.SPECS:
            raise ValueError('no device environment %r (available: %s)' % (task, sorted(self.SPECS)))
        spec = self.SPECS[task]
        self.task = task
        self.observation_space = _Box((spec['state_dim'],))
        self.action_space = _Box((spec['action_dim'],))
        self.horizon, self.clip = spec['horizon'], spec['clip']

    def reset(self):
        raise RuntimeError('%s is stepped on the GPU by des_rollout_eval; it has no host-side reset/step' % self.task)

    step = reset


# ---- host-stepped environments -----------------------------------------------------------------------------------------
STREAM_EPISODE_SEED = 4        # Philox stream tag of episode seeds (DESIGN §3)
TEST_MEMBER = 0x40000000       # the member word of test() episodes (natural_es.py:101-110), as in des_rollout_eval


def _philox4x32_7(c0, c1, c2, c3, seed):
    """The library's counter generator (Philox4x32-7, include/des_b200.h) on uint32 scalars/arrays."""
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
    mask = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = [np.asarray(c, dtype=np.uint64) & mask for c in (c0, c1, c2, c3)]
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
    for _ in range(7):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & mask,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & mask)
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def episode_seed(seed, generation, member, repetition):
    """Seed of episode (generation word, global member, repetition) of a run with `seed`: the first two words of
    Philox4x32-7(counter = (repetition, member, generation, 4), key = seed), x0 + 2^32 x1, shifted right by one so the
    result is a non-negative 63-bit int.  A pure function of the key: shards and reruns see the same episodes.
    Vectorised over array arguments (returns int64 then)."""
    x0, x1, _, _ = _philox4x32_7(repetition, member, generation, STREAM_EPISODE_SEED, seed)
    s = ((x1 << np.uint64(32)) | x0) >> np.uint64(1)
    return int(s) if s.ndim == 0 else s.astype(np.int64)


class GymEnvBatch:
    """The batch protocol over B single environments with the classic gym API the reference uses: reset() -> obs,
    step(a) -> (obs, reward, done, info), and optionally seed(s).  Before each reset, slot b's environment is seeded with
    episode_seed(seed, *keys[b]) when it has seed().  Slots that are not alive are not stepped."""

    def __init__(self, env_fn, B, seed=0):
        self.envs = [env_fn() for _ in range(int(B))]
        self.num_envs = len(self.envs)
        self.seed = int(seed)
        e = self.envs[0] if self.envs else env_fn()
        self.state_dim = int(e.observation_space.shape[0])
        self.action_dim = int(e.action_space.shape[0])

    def reset(self, keys):
        keys = np.asarray(keys, dtype=np.int64).reshape(self.num_envs, 3)
        obs = np.empty((self.num_envs, self.state_dim), dtype=np.float64)
        for b, env in enumerate(self.envs):
            if hasattr(env, 'seed'):
                env.seed(episode_seed(self.seed, *(int(v) for v in keys[b])))
            obs[b] = np.asarray(env.reset(), dtype=np.float64).reshape(-1)
        return obs

    def step(self, actions, alive):
        actions = np.asarray(actions).reshape(self.num_envs, -1)
        alive = np.asarray(alive, dtype=bool).reshape(-1)
        obs = np.zeros((self.num_envs, self.state_dim), dtype=np.float64)
        reward = np.zeros(self.num_envs, dtype=np.float64)
        done = np.ones(self.num_envs, dtype=bool)
        for b in np.flatnonzero(alive):
            o, r, d, _ = self.envs[b].step(actions[b].astype(np.float64))
            obs[b] = np.asarray(o, dtype=np.float64).reshape(-1)
            reward[b] = float(r)
            done[b] = bool(d)
        return obs, reward, done
