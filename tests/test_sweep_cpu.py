"""The host logic of sweeps without a GPU: engine.RolloutRunsEngine(seeds=...) and natural_es.train_sweep over the
oracle-backed stand-in of cpu_ops_sweep.py (the single-population stand-ins of cpu_ops applied run by run with each run's
seed and hyper-parameters).  The launches of a generation do not depend on the number of runs, run r is a
RolloutEngine of its own seed and hyper-parameters, train_sweep's run r is train(configs[r]), equal runs are identical,
and every sweep the trainer cannot run is refused by name."""
import copy

import numpy as np
import pytest

import cpu_ops
import cpu_ops_runs
import cpu_ops_sweep
import host_env_support as hs
from distributedes_b200 import config as cfg
from distributedes_b200 import natural_es
from distributedes_b200.engine import RolloutEngine, RolloutRunsEngine
from ranks import spawn
from test_runs_cpu import Calls

SEEDS = [5, 11, 5, 2**40 + 3, 7]
SIGMA = [0.1, 0.05, 0.2, 0.1, 0.15]
LR = [0.05, 0.1, 0.02, 0.05, 0.08]
WD = [0.005, 0.0, 0.01, 0.005, 0.02]
NOISE = [0.0, 0.3, 0.1, 0.0, 0.2]


def _theta0(P, R=None):
    rng = np.random.default_rng(0)
    return (rng.standard_normal(P if R is None else (R, P)) * 0.3).astype(np.float32)


def _engine(R, kernels=cpu_ops_sweep, **kw):
    P = cpu_ops.param_count(3, 16, 1)
    hyper = dict(seeds=SEEDS[:R], sigma=SIGMA[:R], learning_rate=LR[:R], weight_decay=WD[:R], action_noise_std=NOISE[:R])
    hyper.update(kw)
    return RolloutRunsEngine(hidden=16, pop_size=4, runs=R, theta0=_theta0(P, R), repetitions=2, horizon=12,
                             kernels=kernels, device='cpu', **hyper)


def _config(**kw):
    c = cfg.ClosedLoopPendulumConfig(16)
    c.pop_size, c.repetitions, c.test_repetitions, c.max_generations = 4, 2, 2, 2
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_a_sweep_generation_launches_the_same_ops_for_one_run_and_for_five():
    traces = []
    for R in (1, 5):
        k = Calls(cpu_ops_sweep)
        e = _engine(R, k)
        k.names.clear()
        e.generation()
        e.test_returns()
        traces.append(k.names)
    assert traces[0] == traces[1] == ['rollout_eval_sweep', 'centered_rank_runs', 'nes_grad_partial_sweep',
                                      'nes_apply_sweep', 'state_advance', 'obs_stats_merge_totals_runs',
                                      'rollout_eval_sweep']


def test_run_r_is_a_rolloutengine_of_its_own_seed_and_hyper_parameters():
    R = 5
    e = _engine(R)
    theta0 = e.theta_numpy().copy()
    for _ in range(2):
        e.generation()
    test = e.test_returns()
    for r in range(R):
        single = RolloutEngine(hidden=16, pop_size=4, theta0=theta0[r], sigma=SIGMA[r], learning_rate=LR[r],
                               weight_decay=WD[r], action_noise_std=NOISE[r], seed=SEEDS[r], repetitions=2, horizon=12,
                               kernels=cpu_ops, device='cpu')
        for _ in range(2):
            single.generation()
        assert np.array_equal(e.theta_numpy()[r], single.theta_numpy()), r
        assert np.array_equal(e.adam_m[r].numpy(), single.adam_m.numpy()), r
        assert np.array_equal(e.adam_v[r].numpy(), single.adam_v.numpy()), r
        assert np.array_equal(e.fitness_all[r].numpy(), single.fitness_all.numpy()), r
        assert np.array_equal(e.obs_stats[r].numpy(), single.obs_stats.numpy()), r
        assert np.array_equal(test[r], single.test_returns()), r
    assert not np.array_equal(e.theta_numpy()[0], e.theta_numpy()[1])


def test_runs_with_the_same_seed_and_hyper_parameters_are_identical():
    P = cpu_ops.param_count(3, 16, 1)
    e = RolloutRunsEngine(hidden=16, pop_size=4, runs=3, theta0=_theta0(P), sigma=0.1, learning_rate=0.05,
                          repetitions=2, horizon=12, seeds=[9, 9, 4], kernels=cpu_ops_sweep, device='cpu')
    for _ in range(2):
        e.generation()
    assert np.array_equal(e.theta_numpy()[0], e.theta_numpy()[1])
    assert np.array_equal(e.fitness_all[0].numpy(), e.fitness_all[1].numpy())
    assert not np.array_equal(e.fitness_all[0].numpy(), e.fitness_all[2].numpy())


def test_per_run_values_need_seeds_and_one_entry_per_run():
    P = cpu_ops.param_count(3, 16, 1)
    kw = dict(hidden=16, pop_size=4, runs=3, theta0=_theta0(P), kernels=cpu_ops_sweep, device='cpu')
    for name in ('sigma', 'learning_rate', 'weight_decay', 'action_noise_std'):
        hyper = dict(sigma=0.1, learning_rate=0.1)
        hyper[name] = [0.1, 0.2, 0.3]
        with pytest.raises(ValueError, match='%s per run needs seeds=' % name):
            RolloutRunsEngine(**kw, **hyper)
        with pytest.raises(ValueError, match='%s has 2 entries; a sweep of 3 runs' % name):
            RolloutRunsEngine(**kw, **dict(hyper, **{name: [0.1, 0.2]}), seeds=[1, 2, 3])
    with pytest.raises(ValueError, match='seeds has 2 entries; a sweep of 3 runs'):
        RolloutRunsEngine(**kw, sigma=0.1, learning_rate=0.1, seeds=[1, 2])
    with pytest.raises(ValueError, match='seeds must be a sequence'):
        RolloutRunsEngine(**kw, sigma=0.1, learning_rate=0.1, seeds=4)
    with pytest.raises(ValueError, match='sigma must be > 0.*run 1 has 0.0'):
        RolloutRunsEngine(**kw, sigma=[0.1, 0.0, 0.1], learning_rate=0.1, seeds=[1, 2, 3])


def test_without_seeds_the_engine_keeps_the_runs_contract():
    e = _engine(2, kernels=Calls(cpu_ops_runs), seeds=None, sigma=0.1, learning_rate=0.05, weight_decay=0.005,
                action_noise_std=0.0)
    assert e.hp is None and e.seed == 0 and e.sigma == 0.1


def _sweep_configs():
    cs = []
    for s, sigma, lr, wd in ((0, 0.1, 0.1, 0.005), (3, 0.05, 0.2, 0.0), (17, 0.2, 0.05, 0.01)):
        c = copy.copy(_config())
        c.seed, c.sigma, c.learning_rate, c.weight_decay = s, sigma, lr, wd
        cs.append(c)
    cs[2].initial_weight = cs[2].initial_weight * 0.5
    return cs


def _cpu_sweep_engine(configs, **kw):
    return natural_es.build_sweep_engine(configs, kernels=cpu_ops_sweep, device='cpu', **kw)


def test_train_sweep_run_r_is_train_of_config_r():
    configs = _sweep_configs()
    out = natural_es.train_sweep(configs, engine=_cpu_sweep_engine(configs))
    assert len(out) == 3
    for c, run in zip(configs, out):
        single = natural_es.train(c, engine=natural_es.build_engine(c, kernels=cpu_ops, device='cpu'))
        assert run[:2] == single[:2]
        assert len(run[2]) == len(single[2])
    assert out[0][2] == out[1][2]                      # one clock
    assert out[0][0] != out[1][0]


def _changed(field, value):
    def make():
        cs = _sweep_configs()
        obj = cs[1]
        *path, last = field.split('.')
        for p in path:                 # copy.copy(config) shares config.opt: give configs[1] its own
            obj = copy.copy(getattr(obj, p))
            setattr(cs[1], p, obj)
        setattr(obj, last, value)
        return cs
    return make


@pytest.mark.parametrize('field,value', [
    ('task', 'Other-v0'), ('hidden_size', 32), ('pop_size', 6), ('repetitions', 3), ('test_repetitions', 3),
    ('clip', 1.0), ('normalize_obs', False), ('opt.beta1', 0.8), ('opt.beta2', 0.99), ('opt.epsilon', 1e-6),
    ('max_steps', 1000), ('max_generations', 3),
])
def test_train_sweep_names_the_first_shared_field_that_differs(field, value):
    with pytest.raises(ValueError, match=r'configs differ in %s \(' % field.replace('.', r'\.')):
        natural_es.train_sweep(_changed(field, value)())


def test_train_sweep_ignores_the_tag():
    cs = _sweep_configs()
    cs[1].tag = 'another'
    natural_es.check_sweep_configs(cs)


@pytest.mark.parametrize('make,match', [
    (lambda: cfg.PendulumConfig(16), 'tape configs'),
    (lambda: cfg.HostEnvConfig(hs.PendulumProbe, 16), 'host-stepped'),
    (lambda: _config(mirrored=True), 'mirrored sampling'),
    (lambda: _config(pop_size=2049), 'pop_size 2049 > 2048'),
])
def test_train_sweep_refuses_what_train_runs_refuses(make, match):
    with pytest.raises(ValueError, match=match):
        natural_es.train_sweep([_config(), make()])


def _world_of_two():
    try:
        natural_es.train_sweep(_sweep_configs())
    except ValueError as e:
        assert 'world size 2' in str(e), e
        return
    raise AssertionError('train_sweep accepted a process group of 2')


def test_train_sweep_refuses_a_process_group_of_several_ranks():
    spawn(2, _world_of_two)
