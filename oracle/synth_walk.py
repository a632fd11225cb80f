"""'SynthWalk-v0': a BipedalWalker-shaped test environment (obs 24, action 4) — TEST INFRASTRUCTURE ONLY.

The host-stepped training path (engine.HostEnvEngine) is pinned with it: oracle/make_golden.py runs the reference's
natural_es.train() verbatim on it (the stand-in gym's make('SynthWalk-v0')), and the tests step the same dynamics
through distributedes_b200.envs.GymEnvBatch.  Its dynamics live here only.

  state s in R^24, fp64; reset state: 24 uniforms in (-1, 1) from the episode seed (below)
  s' = 0.8 s + 0.2 tanh(M s) + B a                       a = the (clipped) action, 4 entries
  r  = 0.5 s'_1 - 0.02 |s'|^2 - 0.1 |a - tanh(C s)|^2    depends on state and action
  obs = s' ; the episode ends after L = 40 + floor(60.5 (s0_0 + 1)) steps, L in [40, 160], a function of the reset state
M, B, C are fixed (RandomState(2024)).

Episode seeds: episode (generation word g, global member m, repetition r) of a run with `seed` is seeded with
episode_seed(seed, g, m, r) = (x0 + 2^32 x1) >> 1 for Philox4x32-7(counter = (r, m, g, 4), key = seed) — the
documented function of distributedes_b200.envs, restated here on oracle.nes_oracle's Philox.  A seed s gives the reset
state u_k = 2 ((w_k & 0x7FFFFF) + 0.5) / 2^23 - 1 for the words w_0..w_23 of Philox4x32-7(counter = (q, 0, 0, 0x5717),
key = s), q = 0..5.
"""
import numpy as np

from oracle import nes_oracle as orc

D0, A = 24, 4
STREAM_EPISODE_SEED = 4
TEST_MEMBER = 0x40000000
_rs = np.random.RandomState(2024)
M = _rs.randn(D0, D0) * (0.8 / np.sqrt(D0))
B = _rs.randn(D0, A) * 0.3
C = _rs.randn(A, D0) * (1.0 / np.sqrt(D0))
del _rs


class _Box:
    def __init__(self, shape):
        self.shape = shape


def episode_seed(seed, generation, member, repetition):
    x0, x1, _, _ = orc.philox4x32(repetition, member, generation, STREAM_EPISODE_SEED, seed & 0xFFFFFFFF,
                                  (seed >> 32) & 0xFFFFFFFF)
    return int((int(x1) << 32 | int(x0)) >> 1)


def reset_state(s):
    s = int(s)
    w = np.stack(orc.philox4x32(np.arange(6), 0, 0, 0x5717, s & 0xFFFFFFFF, (s >> 32) & 0xFFFFFFFF), axis=1).reshape(-1)
    return 2.0 * (((w & np.uint32(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0) - 1.0


def episode_length(state):
    return 40 + int(np.floor(60.5 * (state[0] + 1.0)))


def step(s, a):
    """fp64 dynamics of one step: (next state, reward)."""
    a = np.asarray(a, dtype=np.float64).reshape(A)
    ns = 0.8 * s + 0.2 * np.tanh(M @ s) + B @ a
    d = a - np.tanh(C @ s)
    r = 0.5 * ns[1] - 0.02 * float(ns @ ns) - 0.1 * float(d @ d)
    return ns, float(r)


class SynthWalkEnv:
    """Classic gym API: seed(s), reset() -> obs, step(a) -> (obs, reward, done, info)."""
    observation_space = _Box((D0,))
    action_space = _Box((A,))

    def __init__(self):
        self._seed = 0

    def seed(self, s=None):
        self._seed = int(s or 0)
        return [self._seed]

    def reset(self):
        self.state = reset_state(self._seed)
        self.t, self.T = 0, episode_length(self.state)
        return self.state.copy()

    def step(self, action):
        self.state, r = step(self.state, action)
        self.t += 1
        return self.state.copy(), r, self.t >= self.T, {}
