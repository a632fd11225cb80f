"""Host-stepped environments on CPU: the oracle's host loop against the reference's own natural_es.train() run verbatim
on SynthWalk-v0 (tests/golden/train_host_walk.npz, oracle/make_golden.py::train_env), the batch protocol adapter
envs.GymEnvBatch, des_policy_act's argument checks, GymConfig without gym, and engine.HostEnvEngine on two gloo ranks."""
import os
import sys

import numpy as np
import pytest

import cpu_ops
import host_env_support as hs
from lib_fixture import lib  # noqa: F401
from oracle import nes_oracle as orc
from oracle import synth_walk as sw
from ranks import spawn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(REPO, 'tests', 'golden', 'train_host_walk.npz')


def walk_batch(seed):
    from distributedes_b200.envs import GymEnvBatch
    return lambda B: GymEnvBatch(sw.SynthWalkEnv, B, seed)


def test_oracle_host_loop_matches_verbatim_reference_train_on_synth_walk():
    g = np.load(GOLD)
    H, N, reps, seed, gens = int(g['H']), int(g['N']), int(g['reps']), int(g['seed']), int(g['gens'])
    assert (H, N, reps, gens) == (64, 16, 10, 3)
    recs = list(hs.host_chain(g['theta0'].copy(), 24, H, 4, 1.0, N, reps, seed, float(g['sigma']), float(g['lr']),
                              float(g['wd']), gens, walk_batch(seed)))
    # natural_es.py:75 sums the episodes' real lengths, which vary between slots
    assert list(g['train_steps']) == [0] + list(np.cumsum([r['steps'] for r in recs[:gens]]))
    assert len(set(np.diff(g['train_steps']))) > 1
    for gen, r in enumerate(recs):
        assert abs(r['test'].mean() - g['test_rewards'][gen]) <= 1e-5 * abs(g['test_rewards'][gen])
        if gen == gens:
            break
        assert np.allclose(r['stats'], g['stats'][gen], rtol=2e-4, atol=2e-5)
        scale = np.abs(g['grad_after_wd'][gen]).max()
        assert np.abs(r['grad_after_wd'] - g['grad_after_wd'][gen]).max() <= (1e-12 if gen == 0 else 1e-5) * scale
        assert np.abs(r['theta'] - g['theta'][gen]).max() <= 2e-6


def test_synth_walk_episode_lengths_vary_and_depend_on_the_reset_state_only():
    lengths = []
    for m in range(40):
        e = sw.SynthWalkEnv()
        e.seed(sw.episode_seed(3, 0, m, 0))
        s0 = e.reset()
        n, done = 0, False
        while not done:
            _, _, done, _ = e.step(np.zeros(4))
            n += 1
        assert n == sw.episode_length(s0)
        lengths.append(n)
    assert min(lengths) >= 40 and max(lengths) <= 160 and len(set(lengths)) > 10


class CountingEnv:
    """Classic gym API; records its seeds and steps."""
    class _Box:
        def __init__(self, n):
            self.shape = (n,)
    observation_space, action_space = _Box(2), _Box(1)

    def __init__(self):
        self.seeds, self.steps, self.length = [], 0, 3

    def seed(self, s):
        self.seeds.append(s)
        self.length = 2 + s % 3
        return [s]

    def reset(self):
        self.t = 0
        return [float(self.length), 0.5]

    def step(self, a):
        self.steps += 1
        self.t += 1
        return [float(self.length), float(a[0])], 1.0 + a[0], self.t >= self.length, {}


class NoSeedEnv(CountingEnv):
    seed = None

    def __getattribute__(self, name):
        if name == 'seed':
            raise AttributeError(name)
        return object.__getattribute__(self, name)


def test_gym_env_batch_steps_alive_slots_only_and_seeds_each_reset_from_its_key():
    from distributedes_b200.envs import GymEnvBatch, episode_seed
    b = GymEnvBatch(CountingEnv, 4, seed=7)
    assert b.num_envs == 4 and (b.state_dim, b.action_dim) == (2, 1)
    keys = np.array([[3, 10, 0], [3, 10, 1], [3, 11, 0], [3, 11, 1]])
    obs = b.reset(keys)
    assert obs.shape == (4, 2) and obs.dtype == np.float64
    assert [e.seeds for e in b.envs] == [[episode_seed(7, 3, 10, 0)], [episode_seed(7, 3, 10, 1)],
                                         [episode_seed(7, 3, 11, 0)], [episode_seed(7, 3, 11, 1)]]
    alive = np.array([True, False, True, False])
    obs, r, done = b.step(np.full((4, 1), 0.25), alive)
    assert [e.steps for e in b.envs] == [1, 0, 1, 0]
    assert r.dtype == np.float64 and done.dtype == bool and np.array_equal(r, [1.25, 0, 1.25, 0])
    assert np.array_equal(obs[:, 1], [0.25, 0, 0.25, 0])
    # environments without seed() are reset as they are
    nb = GymEnvBatch(NoSeedEnv, 2)
    assert nb.reset(np.zeros((2, 3), dtype=np.int64)).shape == (2, 2)


def test_episode_seed_is_a_pure_function_of_the_key():
    from distributedes_b200.envs import episode_seed
    keys = [(0, 0, 0), (0, 0, 1), (0, 1, 0), (1, 0, 0), (5, 0x40000000, 9), (2 ** 32 - 1, 2 ** 28 - 1, 15)]
    seeds = [episode_seed(11, *k) for k in keys]
    assert seeds == [episode_seed(11, *k) for k in keys] == [sw.episode_seed(11, *k) for k in keys]
    assert len(set(seeds)) == len(seeds) and all(0 <= s < 2 ** 63 for s in seeds)
    assert episode_seed(12, 0, 0, 0) != seeds[0]
    # vectorised over arrays
    k = np.array(keys, dtype=np.int64)
    assert list(episode_seed(11, k[:, 0], k[:, 1], k[:, 2])) == seeds


@pytest.mark.parametrize('d0,H,A,reps,alive,P,match', [
    (24, 48, 4, 10, True, None, 'hidden must be 16, 32, 64, 96 or 128'),
    (33, 64, 4, 10, True, None, 'state_dim must be in'),
    (24, 64, 9, 10, True, None, 'action_dim must be in'),
    (24, 64, 4, 17, True, None, 'repetitions must be in'),
    (24, 64, 4, 10, False, None, 'NULL alive mask'),
    (24, 64, 4, 10, True, 6021, 'MLP needs 6020'),
])
def test_policy_act_rejects_bad_arguments_without_gpu(lib, d0, H, A, reps, alive, P, match):
    import ctypes as C
    from distributedes_b200._lib import Dims
    if P is None:
        P = max(int(lib.des_param_count(d0, H, A)), 1)
    dummy = C.c_void_p(16)                    # never dereferenced: validation happens before any CUDA work
    rc = lib.des_policy_act(dummy, None, dummy, P, dummy, dummy if alive else None, None, Dims(d0, H, A, 0), reps, 1.0,
                            0.0, 0, 0, 0, 4, 0, None)
    assert rc == -1
    assert match in lib.des_last_error().decode()
    assert lib.des_obs_parts_reduce(dummy, dummy, 4, 0, None) == -1


def test_gym_config_names_gym_when_it_is_missing(monkeypatch):
    from distributedes_b200.config import GymConfig
    monkeypatch.setitem(sys.modules, 'gym', None)          # `import gym` raises ImportError
    with pytest.raises(ImportError, match='gym package'):
        GymConfig('BipedalWalker-v2', 64)


def test_host_env_config_probes_the_environment():
    from distributedes_b200.config import HostEnvConfig
    cfg = HostEnvConfig(sw.SynthWalkEnv, hidden_size=16, task='SynthWalk-v0')
    assert (cfg.state_dim, cfg.action_dim, cfg.hidden_size, cfg.clip) == (24, 4, 16, 1.0)
    assert cfg.host_env and cfg.normalize_obs and cfg.repetitions == cfg.test_repetitions == 10
    assert cfg.initial_weight.size == 24 * 16 + 16 + 16 * 16 + 16 + 4 * 16 + 4
    with pytest.raises(ValueError, match='hidden_size'):
        HostEnvConfig(sw.SynthWalkEnv, hidden_size=48)


def _engine(N, seed, device='cpu'):
    from distributedes_b200.engine import HostEnvEngine
    return HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=walk_batch(seed), hidden=16, pop_size=N,
                         theta0=np.asarray(orc.synthetic_theta(24, 16, 4), dtype=np.float32), sigma=0.1,
                         learning_rate=0.1, repetitions=3, test_repetitions=2, seed=seed, device=device,
                         kernels=cpu_ops)


def _run(N, gens):
    eng = _engine(N, 5)
    out = dict(fit=[], steps=[], stats=[], tests=[])
    for _ in range(gens):
        out['tests'].append(eng.test_returns())
        eng.generation()
        out['fit'].append(eng.fitness_all.numpy().copy())
        out['steps'].append(eng.steps_taken)
        out['stats'].append(eng.obs_stats.numpy().copy())
    out['theta'] = eng.theta.numpy().copy()
    return {k: np.asarray(v) for k, v in out.items()}


def test_host_env_engine_on_two_ranks_equals_the_single_process_run():
    """Ragged 2-rank split: each rank steps only its own members' environments; the fitness all-gather, the fp64
    observation totals and the step count summed over ranks give the single-process run's fitness, steps, statistics
    and parameters."""
    N, gens = 5, 2
    one = _run(N, gens)
    res = spawn(2, _run, N, gens)
    for k in ('fit', 'steps', 'stats', 'tests', 'theta'):
        assert np.array_equal(res[0][k], res[1][k]), k
    for k in ('fit', 'steps', 'stats', 'tests'):
        assert np.array_equal(res[0][k], one[k]), k
    # the fp32 gradient partials are summed per rank, then across ranks: association differs at rounding
    assert np.max(np.abs(res[0]['theta'] - one['theta'])) <= 2e-6
    assert one['steps'][0] != one['steps'][1]
