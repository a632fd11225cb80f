"""The host logic of host-stepped sweeps without a GPU: engine.HostEnvSweepEngine and natural_es.train_sweep over the
oracle-backed stand-in of cpu_ops_host_sweep.py.  One policy launch per environment step whatever the number of runs,
run r is the HostEnvEngine of its own config, train_sweep's run r is train(configs[r]) with runs stopping at different
generations, every run's environments see the calls of its standalone run and none after it stops, and every sweep the
trainer cannot run is refused by name."""
import copy

import numpy as np
import pytest

import cpu_ops
import cpu_ops_host_sweep
import host_env_support as hs
from distributedes_b200 import config as cfg
from distributedes_b200 import natural_es
from distributedes_b200.engine import HostEnvEngine, HostEnvSweepEngine
from distributedes_b200.envs import GymEnvBatch
from oracle import nes_oracle as orc
from oracle import synth_walk as sw
from ranks import spawn
from test_runs_cpu import Calls

SEEDS = [5, 11, 5, 2**40 + 3, 7]
SIGMA = [0.1, 0.05, 0.2, 0.1, 0.15]
LR = [0.05, 0.1, 0.02, 0.05, 0.08]
WD = [0.005, 0.0, 0.01, 0.005, 0.02]
NOISE = [0.0, 0.3, 0.1, 0.0, 0.2]


class FixedBatch:
    """A vectorised batch environment (envs.py protocol) whose episodes last `length` steps: the observation is a
    function of the reset key and the step, the reward -|a|^2."""

    def __init__(self, B, length=5, d0=3, A=2):
        self.num_envs, self.length, self.d0 = B, length, d0

    def reset(self, keys):
        self.t = 0
        self.base = np.asarray(keys, dtype=np.float64).sum(axis=1, keepdims=True) % 7 / 7.0
        return np.tile(self.base, (1, self.d0))

    def step(self, actions, alive):
        self.t += 1
        a = np.asarray(actions, dtype=np.float64)
        obs = np.tile(self.base, (1, self.d0)) + 0.1 * self.t
        return obs, -(a * a).sum(axis=1), np.full(self.num_envs, self.t >= self.length)


class Recording:
    """Records every reset and step a batch environment receives, with copies of its arguments."""

    def __init__(self, env, log):
        self.env, self.log, self.num_envs = env, log, env.num_envs

    def reset(self, keys):
        self.log.append(('reset', np.array(keys)))
        return self.env.reset(keys)

    def step(self, actions, alive):
        self.log.append(('step', np.array(actions), np.array(alive)))
        return self.env.step(actions, alive)


def walk_batch(seed):
    return lambda B: GymEnvBatch(sw.SynthWalkEnv, B, seed)


def _theta0(R):
    return np.stack([np.asarray(orc.synthetic_theta(24, 16, 4, seed=r), dtype=np.float32) for r in range(R)])


def _sweep(R, kernels=cpu_ops_host_sweep, **kw):
    hyper = dict(seeds=SEEDS[:R], sigma=SIGMA[:R], learning_rate=LR[:R], weight_decay=WD[:R], action_noise_std=NOISE[:R],
                 env_fn=sw.SynthWalkEnv, batch_env_fn=[walk_batch(s) for s in SEEDS[:R]])
    hyper.update(kw)
    hyper.setdefault('theta0', _theta0(R))
    return HostEnvSweepEngine(hidden=16, pop_size=4, runs=R, repetitions=2, test_repetitions=3, kernels=kernels,
                              device='cpu', **hyper)


def test_one_policy_launch_per_step_for_one_run_and_for_five():
    traces = []
    for R in (1, 5):
        k = Calls(cpu_ops_host_sweep)
        theta0 = np.random.default_rng(R).standard_normal(cpu_ops.param_count(3, 16, 2)).astype(np.float32) * 0.3
        e = _sweep(R, k, env_fn=hs.PendulumProbe, state_dim=3, action_dim=2, batch_env_fn=FixedBatch, theta0=theta0)
        k.names.clear()
        e.test_returns()
        e.generation()
        traces.append(k.names)
    assert traces[0] == traces[1] == (['policy_act_sweep'] * 5 + ['nes_perturb_sweep'] + ['policy_act_sweep'] * 5 +
                                      ['obs_parts_reduce_runs', 'centered_rank_runs', 'nes_grad_partial_sweep',
                                       'nes_apply_sweep', 'state_advance', 'obs_stats_merge_totals_runs'])


def test_run_r_is_the_hostenvengine_of_its_own_seed_and_hyper_parameters():
    R, gens = 5, 3
    e = _sweep(R)
    out = dict(test=[], fit=[], steps=[], stats=[])
    for _ in range(gens):
        out['test'].append(e.test_returns())
        e.generation()
        out['fit'].append(e.fitness_all.numpy().copy())
        out['steps'].append(e.steps_taken.copy())
        out['stats'].append(e.obs_stats.numpy().copy())
    theta0 = _theta0(R)
    for r in range(R):
        single = HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=walk_batch(SEEDS[r]), hidden=16, pop_size=4,
                               theta0=theta0[r], sigma=SIGMA[r], learning_rate=LR[r], weight_decay=WD[r],
                               action_noise_std=NOISE[r], seed=SEEDS[r], repetitions=2, test_repetitions=3,
                               kernels=cpu_ops, device='cpu')
        for g in range(gens):
            assert np.array_equal(out['test'][g][r], single.test_returns()), (r, g)
            single.generation()
            assert np.array_equal(out['fit'][g][r], single.fitness_all.numpy()), (r, g)
            assert out['steps'][g][r] == single.steps_taken, (r, g)
            assert np.array_equal(out['stats'][g][r], single.obs_stats.numpy()), (r, g)
        assert np.array_equal(e.theta_numpy()[r], single.theta_numpy()), r
        assert np.array_equal(e.adam_m[r].numpy(), single.adam_m.numpy()), r
        assert np.array_equal(e.adam_v[r].numpy(), single.adam_v.numpy()), r
    assert len({s for g in out['steps'] for s in g}) > 1          # the runs' episodes differ in length
    assert not np.array_equal(e.fitness_all[0].numpy(), e.fitness_all[2].numpy())       # one seed, two sigmas


def _config(seed, sigma, lr, log=None, **kw):
    c = cfg.HostEnvConfig(sw.SynthWalkEnv, 16, task='SynthWalk-v0')
    c.pop_size, c.repetitions, c.test_repetitions = 4, 2, 2
    c.seed, c.sigma, c.learning_rate = seed, sigma, lr
    c.max_steps = 1500
    c.initial_weight = np.asarray(orc.synthetic_theta(24, 16, 4, seed=seed % 3), dtype=np.float32)
    if log is not None:
        c.batch_env_fn = lambda B: Recording(GymEnvBatch(sw.SynthWalkEnv, B, seed), log.setdefault(B, []))
    for name, v in kw.items():
        setattr(c, name, v)
    return c


RUNS = ((0, 0.1, 0.1), (3, 0.05, 0.2), (17, 0.2, 0.05), (4, 0.1, 0.1))


def _cpu_sweep_engine(configs):
    return natural_es.build_sweep_engine(configs, kernels=cpu_ops_host_sweep, device='cpu')


def _train(c):
    return natural_es.train(c, engine=natural_es.build_engine(c, kernels=cpu_ops, device='cpu'))


def test_train_sweep_run_r_is_train_of_config_r_and_stops_where_it_does():
    configs = [_config(*h) for h in RUNS]
    out = natural_es.train_sweep(configs, engine=_cpu_sweep_engine(configs))
    assert len(out) == len(configs)
    for c, run in zip(configs, out):
        single = _train(c)
        assert run[:2] == single[:2], c.seed
        assert len(run[2]) == len(single[2])
    assert len({len(run[0]) for run in out}) > 1                   # the runs stop at different generations
    longest = max(out, key=lambda run: len(run[2]))
    for run in out:                                                 # one clock
        assert run[2] == longest[2][:len(run[2])]


def test_every_runs_environments_get_the_calls_of_its_standalone_run_and_none_after_it_stops():
    logs = [({}, {}) for _ in RUNS]
    configs = [_config(*h, log=logs[r][0]) for r, h in enumerate(RUNS)]
    out = natural_es.train_sweep(configs, engine=_cpu_sweep_engine(configs))
    assert len({len(run[0]) for run in out}) > 1
    for r, h in enumerate(RUNS):
        _train(_config(*h, log=logs[r][1]))
        sweep, single = logs[r]
        assert sorted(sweep) == sorted(single) == [2, 8], r       # the test and the member batch environments
        for B in single:
            assert len(sweep[B]) == len(single[B]), (r, B)
            for a, b in zip(sweep[B], single[B]):
                assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])), (r, B)


def _changed(field, value):
    cs = [_config(*h) for h in RUNS[:3]]
    obj = cs[1]
    *path, last = field.split('.')
    for p in path:                     # copy.copy(config) would share config.opt: give configs[1] its own
        obj = copy.copy(getattr(obj, p))
        setattr(cs[1], p, obj)
    setattr(obj, last, value)
    return cs


@pytest.mark.parametrize('field,value', [
    ('hidden_size', 32), ('pop_size', 6), ('state_dim', 12), ('action_dim', 2), ('repetitions', 3),
    ('test_repetitions', 3), ('clip', 2.0), ('normalize_obs', False), ('opt.beta1', 0.8), ('opt.beta2', 0.99),
    ('opt.epsilon', 1e-6), ('max_steps', 1000), ('max_generations', 3),
])
def test_host_sweep_names_the_first_shared_field_that_differs(field, value):
    with pytest.raises(ValueError, match=r'configs differ in %s \(' % field.replace('.', r'\.')):
        natural_es.train_sweep(_changed(field, value))


def test_host_sweep_configs_may_differ_in_their_environments_and_task():
    cs = [_config(*h) for h in RUNS[:2]]
    cs[1].env_fn, cs[1].task = hs.PendulumProbe, 'other'
    cs[1].batch_env_fn = FixedBatch
    natural_es.check_sweep_configs(cs)


@pytest.mark.parametrize('make,match', [
    (lambda: cfg.ClosedLoopPendulumConfig(16), 'configs\\[1\\] is not; .* all host-stepped'),
    (lambda: cfg.PendulumConfig(16), 'host-stepped'),
    (lambda: _config(1, 0.1, 0.1, mirrored=True), 'mirrored sampling'),
    (lambda: _config(1, 0.1, 0.1, pop_size=2049), 'pop_size 2049 > 2048'),
])
def test_host_sweep_refuses_what_it_cannot_train(make, match):
    with pytest.raises(ValueError, match=match):
        natural_es.train_sweep([_config(0, 0.1, 0.1), make()])


def test_host_sweep_engine_needs_a_seed_per_run_and_a_positive_sigma():
    with pytest.raises(ValueError, match='seeds must be a sequence'):
        _sweep(2, seeds=4)
    with pytest.raises(ValueError, match='seeds has 3 entries; a sweep of 2 runs'):
        _sweep(2, seeds=[1, 2, 3])
    with pytest.raises(ValueError, match='batch_env_fn has 1 entries; a sweep of 2 runs'):
        _sweep(2, batch_env_fn=[FixedBatch])
    with pytest.raises(ValueError, match='sigma must be > 0.*run 1 has 0.0'):
        _sweep(2, sigma=[0.1, 0.0])
    with pytest.raises(ValueError, match='pop_size must be in'):
        HostEnvSweepEngine(env_fn=sw.SynthWalkEnv, hidden=16, pop_size=2049, runs=1, theta0=_theta0(1), seeds=[0],
                           sigma=0.1, learning_rate=0.1, kernels=cpu_ops_host_sweep, device='cpu')


def _world_of_two():
    try:
        natural_es.train_sweep([_config(*h) for h in RUNS[:2]])
    except ValueError as e:
        assert 'world size 2' in str(e), e
        return
    raise AssertionError('train_sweep accepted a process group of 2')


def test_host_sweep_refuses_a_process_group_of_several_ranks():
    spawn(2, _world_of_two)
