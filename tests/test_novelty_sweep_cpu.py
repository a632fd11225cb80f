"""Novelty-search sweeps without a GPU, over the oracle-backed stand-in of cpu_ops_novelty_sweep.py:

  - novelty.train_sweep(configs) is novelty.train(configs[r]) for every r, bit for bit: rewards, steps, final theta, Adam
    moments and statistics, archive, the weights each generation shaped with, best and best_theta.  Closed-loop configs
    mix seeds, sigma, learning rates, action noise, start points and w in {0, 0.5, 1, 'adaptive'}; host-stepped runs have
    their own environments and stop at different generations;
  - with every w = 1 a sweep is natural_es.train_sweep(configs);
  - every refusal names the config and the field, before any device work;
  - the stand-ins' signatures are the front ends'; multi_runs(batched=True) writes the sequential runs' rewards and steps.
"""
import inspect
import pickle
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import cpu_ops
import cpu_ops_novelty
import cpu_ops_novelty_sweep
from host_env_support import PendulumProbe
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from ranks import spawn

H = 16
HORIZON = 6
K = types.SimpleNamespace(**{k: v for m in (cpu_ops, cpu_ops_novelty) for k, v in vars(m).items()
                             if not k.startswith('_') and callable(v)})
# seed, sigma, learning rate, action noise, start point, reward weight of each run
RUNS = ((5, 0.05, 0.05, 0.0, 1, 0.0), (7, 0.1, 0.02, 0.1, 2, 0.5), (2**40 + 3, 0.02, 0.1, 0.0, 3, 1.0),
        (5, 0.05, 0.05, 0.0, 1, 'adaptive'))


def _closed(seed, sigma, lr, noise, x0, w, **kw):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(H)
    c.pop_size, c.max_generations, c.repetitions, c.test_repetitions = 6, 5, 2, 2
    c.seed, c.sigma, c.learning_rate, c.action_noise_std = seed, sigma, lr, noise
    c.initial_weight = np.asarray(orc.synthetic_theta(3, H, 1, seed=x0), dtype=np.float32)
    c.ns_reward_weight, c.ns_k = w, 3
    for name, v in kw.items():
        setattr(c, name, v)
    return c


def _host(seed, sigma, lr, noise, x0, w, horizon=HORIZON, **kw):
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0,
                      batch_env_fn=lambda B: po.PendulumBatch(B, seed, horizon))
    c.pop_size, c.repetitions, c.test_repetitions, c.max_steps = 6, 2, 2, 200
    c.seed, c.sigma, c.learning_rate, c.action_noise_std = seed, sigma, lr, noise
    c.initial_weight = np.asarray(orc.synthetic_theta(3, H, 1, seed=x0), dtype=np.float32)
    c.ns_reward_weight, c.ns_k = w, 3
    for name, v in kw.items():
        setattr(c, name, v)
    return c


def _short_sweep(ns):
    e = ns.engine
    if not ns.host:
        e.horizon = HORIZON
        e.steps_taken = e.N * e.repetitions * HORIZON


def _sweep(configs, kernels=cpu_ops_novelty_sweep):
    from distributedes_b200 import novelty
    ns = novelty.build_sweep(configs, kernels=kernels, device='cpu')
    _short_sweep(ns)
    return novelty.train_sweep(configs, ns), ns


def _train(c):
    from distributedes_b200 import novelty
    ns = novelty.build(c, kernels=K, device='cpu')
    e = ns.agents[0]
    if hasattr(e.source, 'horizon'):
        e.source.horizon = e.source.T = HORIZON
    return novelty.train(c, ns), ns


def _same(a, b):
    return a.numpy().tobytes() == b.numpy().tobytes()


def _assert_run_is_train(run, ns, r, c):
    single, one = _train(c)
    e = one.agents[0]
    assert run[:2] == single[:2], r
    assert len(run[2]) == len(single[2]), r
    assert _same(ns.theta(r), e.theta) and _same(ns.adam_m(r), e.adam_m) and _same(ns.adam_v(r), e.adam_v), r
    if e.obs_stats is not None:
        assert _same(ns.obs_stats(r), e.obs_stats), r
    assert _same(ns.archive(r), one.archive), r
    assert ns.weights[r] == one.weights, r
    assert ns.best[r] == one.best and ns.best_theta[r].tobytes() == one.best_theta.tobytes(), r
    assert (ns.reward_weight[r], ns.stall[r]) == (one.reward_weight, one.stall), r


@pytest.fixture
def quick_adaptation(monkeypatch):
    """NSRA-ES lowers w after one generation without a better test, so that a short run changes its weight."""
    from distributedes_b200 import novelty
    monkeypatch.setattr(novelty, 'ADAPT_PATIENCE', 1)


def test_closed_loop_run_r_is_train_of_config_r(quick_adaptation):
    configs = [_closed(*h) for h in RUNS]
    out, ns = _sweep(configs)
    for r, c in enumerate(configs):
        _assert_run_is_train(out[r], ns, r, c)
    assert len(set(ns.weights[3])) > 1                                 # NSRA-ES changed its weight: the table moved
    assert ns.weights[0] == [0.0] * 5 and ns.weights[2] == [1.0] * 5
    assert out[0][0] != out[3][0]                                      # equal seeds, different weights
    assert ns.archive(0).shape == (6, 3) and len({tuple(run[2]) for run in out}) == 1      # one clock


def test_closed_loop_launches_per_generation_do_not_depend_on_the_runs():
    traces = []
    for R in (1, 4):
        calls = []

        def wrap(name, f):
            def g(*a, **kw):
                calls.append(name)
                return f(*a, **kw)
            return g
        k = types.SimpleNamespace(**{n: wrap(n, f) for n, f in vars(cpu_ops_novelty_sweep).items()
                                     if not n.startswith('_') and callable(f) and not inspect.isclass(f)})
        _sweep([_closed(*h, max_generations=2) for h in RUNS[:R]], kernels=k)
        traces.append(calls)
    gen = ['rollout_eval_bc_sweep', 'rollout_eval_bc_sweep', 'novelty_runs', 'ns_shape_runs', 'nes_grad_partial_sweep',
           'nes_apply_sweep', 'state_advance', 'obs_stats_merge_totals_runs']
    assert traces[0] == traces[1]
    assert traces[0][-len(gen) * 2 - 2:] == gen * 2 + ['rollout_eval_bc_sweep'] * 2


def test_host_stepped_run_r_is_train_of_config_r_and_stops_where_it_does(quick_adaptation):
    configs = [_host(*h, horizon=hz) for h, hz in zip(RUNS, (4, 6, 9, 4))]
    out, ns = _sweep(configs)
    assert len({len(run[0]) for run in out}) > 1                       # the runs stop at different generations
    assert not ns.running.any()
    for r, c in enumerate(configs):
        _assert_run_is_train(out[r], ns, r, c)
    longest = max(out, key=lambda run: len(run[2]))
    for run in out:                                                    # one clock
        assert run[2] == longest[2][:len(run[2])]


@pytest.mark.parametrize('make', [_closed, _host], ids=['closed', 'host'])
def test_every_weight_1_is_natural_es_train_sweep(make):
    from distributedes_b200 import natural_es
    # no action noise: cpu_ops' evaluation, which natural_es's sweep runs on, leaves it out (the GPU test has it)
    configs = [make(*h[:3], 0.0, h[4], 1.0) for h in RUNS[:3]]
    out, ns = _sweep(configs)
    engine = natural_es.build_sweep_engine(configs, kernels=cpu_ops_novelty_sweep, device='cpu')
    if not ns.host:
        engine.horizon, engine.steps_taken = HORIZON, engine.N * engine.repetitions * HORIZON
    want = natural_es.train_sweep(configs, engine)
    for r in range(3):
        assert out[r][:2] == want[r][:2], r
        assert _same(ns.theta(r), engine.theta[r]), r


def test_the_archive_doubles_when_full():
    from distributedes_b200 import novelty
    configs = [_closed(*h, max_generations=70) for h in RUNS[:2]]
    out, ns = _sweep(configs)
    assert ns._archive.shape[1] == 128 and ns.size == 71
    for r, c in enumerate(configs):
        single, one = _train(c)
        assert out[r][:2] == single[:2] and _same(ns.archive(r), one.archive), r
    assert novelty._INITIAL_CAPACITY == 64


def test_a_batch_without_seeds_refuses_behaviours():
    from distributedes_b200.engine import RolloutRunsEngine
    e = RolloutRunsEngine(hidden=H, pop_size=4, runs=2, theta0=orc.synthetic_theta(3, H, 1, seed=0), sigma=0.05,
                          learning_rate=0.01, repetitions=2, horizon=4, kernels=cpu_ops_novelty_sweep, device='cpu')
    with pytest.raises(ValueError, match='sweeps only'):
        e.evaluate(bc_out=torch.zeros((2, 4, 3)))
    with pytest.raises(ValueError, match='sweeps only'):
        e.test_returns(bc_out=torch.zeros((2, 1, 3)))


def test_the_weight_table():
    from distributedes_b200.ops_novelty_sweep import ns_weight_table
    t = ns_weight_table([0.0, 0.3, 1.0], 'cpu').numpy()
    assert t.dtype == np.float32 and t.shape == (3, 2)
    assert t[1].tobytes() == np.array([np.float32(0.3), np.float32(1.0 - 0.3)], dtype=np.float32).tobytes()
    for w in (-0.1, 1.5, float('nan')):
        with pytest.raises(ValueError, match='run 1 has reward weight'):
            ns_weight_table([0.5, w], 'cpu')


def test_stand_ins_have_the_front_ends_signatures():
    from distributedes_b200 import ops_novelty_sweep
    names = [n for n, f in vars(ops_novelty_sweep).items()
             if inspect.isfunction(f) and f.__module__ == ops_novelty_sweep.__name__ and not n.startswith('_')]
    assert sorted(names) == ['novelty_runs', 'ns_shape_runs', 'ns_shape_runs_workspace', 'ns_weight_table',
                             'rollout_eval_bc_sweep']
    for n in names:
        assert inspect.signature(getattr(cpu_ops_novelty_sweep, n)) == inspect.signature(getattr(ops_novelty_sweep, n)), n


def _changed(make, field, value):
    cs = [make(*h) for h in RUNS[:3]]
    setattr(cs[1], field, value)
    return cs


@pytest.mark.parametrize('field,value', [
    ('task', 'Pendulum-v1'), ('hidden_size', 32), ('pop_size', 8), ('repetitions', 3), ('test_repetitions', 3),
    ('clip', 1.0), ('normalize_obs', False), ('max_steps', 1000), ('max_generations', 2), ('ns_k', 4),
])
def test_closed_loop_sweep_names_the_first_shared_field_that_differs(field, value):
    from distributedes_b200 import novelty
    with pytest.raises(ValueError, match=r'configs differ in %s \(.*in configs\[1\]' % field):
        novelty.train_sweep(_changed(_closed, field, value))


@pytest.mark.parametrize('field,value', [
    ('hidden_size', 32), ('pop_size', 8), ('repetitions', 3), ('test_repetitions', 3), ('clip', 1.0),
    ('normalize_obs', False), ('max_steps', 1000), ('max_generations', 3), ('ns_k', 4),
])
def test_host_sweep_names_the_first_shared_field_that_differs(field, value):
    from distributedes_b200 import novelty
    with pytest.raises(ValueError, match=r'configs differ in %s \(.*in configs\[1\]' % field):
        novelty.train_sweep(_changed(_host, field, value))


def test_sweep_configs_may_differ_in_what_the_runs_own():
    from distributedes_b200 import novelty
    novelty.check_sweep_configs([_closed(*h) for h in RUNS])
    hs = [_host(*h) for h in RUNS]
    hs[1].task = 'other'
    novelty.check_sweep_configs(hs)


def _tape():
    from distributedes_b200.config import PendulumConfig
    return PendulumConfig(H)


@pytest.mark.parametrize('first,make,match', [
    (_closed, lambda: _closed(*RUNS[1], ns_agents=2), r'configs\[1\] has ns_agents = 2.*Adam t, beta\^t and generation '
                                                      r'word.*one des_state'),
    (_closed, lambda: _closed(*RUNS[1], mirrored=True), r'configs\[1\]: novelty: mirrored sampling'),
    (_closed, _tape, r'configs\[1\]: novelty: a tape has no episodes'),
    (_closed, lambda: _closed(*RUNS[1], ns_k=33), r'configs\[1\]: novelty: ns_k 33 is not in'),
    (_closed, lambda: _closed(*RUNS[1], ns_reward_weight=1.5), r'configs\[1\]: novelty: ns_reward_weight 1.5 is not in'),
    (_closed, lambda: _closed(*RUNS[1], ns_reward_weight='adapt'), r"configs\[1\]: .*ns_reward_weight.*'adaptive'"),
    (_closed, lambda: _closed(*RUNS[1], pop_size=2049), r'configs\[1\]: train_runs: pop_size 2049 > 2048'),
    (_host, lambda: _host(*RUNS[1], pop_size=2049), r'configs\[1\]: train_sweep: pop_size 2049 > 2048'),
    (_closed, lambda: _host(*RUNS[1]), r'configs\[1\] is host-stepped and configs\[0\] is not'),
    (_host, lambda: _closed(*RUNS[1]), r'configs\[0\] is host-stepped and configs\[1\] is not'),
])
def test_sweep_refuses_what_it_cannot_train(first, make, match):
    from distributedes_b200 import novelty
    with pytest.raises(ValueError, match=match):
        novelty.train_sweep([first(*RUNS[0]), make()])
    with pytest.raises(ValueError, match=match):
        novelty.build_sweep([first(*RUNS[0]), make()], kernels=cpu_ops_novelty_sweep, device='cpu')


def test_sweep_refuses_an_empty_list():
    from distributedes_b200 import novelty
    with pytest.raises(ValueError, match='no configs'):
        novelty.train_sweep([])


def _world_of_two():
    from distributedes_b200 import novelty
    try:
        novelty.train_sweep([_closed(*h) for h in RUNS[:2]])
    except ValueError as e:
        assert 'configs[0]' in str(e) and 'world size 2' in str(e), e
        return
    raise AssertionError('train_sweep accepted a process group of 2')


def test_sweep_refuses_a_process_group_of_several_ranks():
    spawn(2, _world_of_two)


def test_multi_runs_batched_writes_the_rewards_and_steps_of_the_sequential_runs(tmp_path, monkeypatch):
    from distributedes_b200 import novelty
    train, train_sweep = novelty.train, novelty.train_sweep      # multi_runs' trainers, with the short horizon

    def short_train(c, ns):
        ns.agents[0].source.horizon = ns.agents[0].source.T = HORIZON
        return train(c, ns)

    def short_sweep(configs, ns):
        _short_sweep(ns)
        return train_sweep(configs, ns)
    monkeypatch.setattr(novelty, 'train', short_train)
    monkeypatch.setattr(novelty, 'train_sweep', short_sweep)
    config = _closed(5, 0.05, 0.05, 0.1, 0, 0.5, max_generations=3)
    config.tag = 'ns'
    out = {}
    for batched in (False, True):
        d = tmp_path / str(batched)
        stats = novelty.multi_runs(config, runs=3, log_dir=str(d / 'log'), data_dir=str(d / 'data'), batched=batched,
                                   kernels=cpu_ops_novelty_sweep if batched else K, device='cpu')
        with open(d / 'data' / 'ns-stats-Pendulum-v0.bin', 'rb') as f:
            out[batched] = pickle.load(f)
        assert out[batched] == stats and len(stats) == 3
        assert (d / 'log' / 'ns-Pendulum-v0.txt').exists()
    for a, b in zip(out[False], out[True]):
        assert a[:2] == b[:2]
    assert out[False][0][0] != out[False][1][0]                        # seeds config.seed + r: independent runs
    assert config.seed == 5
