"""The host logic of genetic-algorithm sweeps without a GPU: genetic.train_sweep, GASweep and SweepWorker over the
oracle-backed stand-in of cpu_ops_ga_sweep.py.  The same launches per generation for one run and for five, run r equal to
genetic.train(configs[r]) with its final table, order and statistics (closed-loop and host-stepped SynthWalk, with seeds,
sigma, truncation, elites, action noise and start points differing per run, and host-stepped runs stopping at different
generations), every run's environments seeing exactly the calls of its standalone run, one refusal per shared field and
per refused kind, and multi_runs(batched=True) writing what the sequential runs write."""
import pickle
import types

import numpy as np
import pytest
import torch

import cpu_ops
import cpu_ops_ga
import cpu_ops_ga_sweep
from distributedes_b200 import config as cfg
from distributedes_b200 import genetic
from distributedes_b200.envs import GymEnvBatch
from oracle import nes_oracle as orc
from oracle import synth_walk as sw
from ranks import spawn
from test_host_sweep_cpu import Recording
from test_runs_cpu import Calls

K = types.SimpleNamespace(**{k: v for m in (cpu_ops, cpu_ops_ga) for k, v in vars(m).items()
                             if not k.startswith('_') and callable(v)})
HORIZON = 6
# seed, sigma, action noise, x0 seed, truncation, elites of each run (runs 0 and 3 are equal: identical runs)
RUNS = ((0, 0.05, 0.0, 0, 3, 1), (3, 0.1, 0.2, 1, 2, 0), (2**40 + 17, 0.02, 0.1, 2, 4, 2), (0, 0.05, 0.0, 0, 3, 1),
        (9, 0.2, 0.0, 1, 1, 1))


def _closed(seed, sigma, noise, x0, T, E, **kw):
    c = cfg.ClosedLoopPendulumConfig(16)
    c.pop_size, c.repetitions, c.test_repetitions, c.max_generations = 6, 2, 3, 3
    c.seed, c.sigma, c.action_noise_std, c.truncation, c.elites = seed, sigma, noise, T, E
    c.initial_weight = np.asarray(orc.synthetic_theta(3, 16, 1, seed=x0), dtype=np.float32)
    for name, v in kw.items():
        setattr(c, name, v)
    return c


def _walk(seed, sigma, noise, x0, T, E, log=None, **kw):
    c = cfg.HostEnvConfig(sw.SynthWalkEnv, 16, task='SynthWalk-v0')
    c.pop_size, c.repetitions, c.test_repetitions = 5, 2, 2
    c.seed, c.sigma, c.action_noise_std, c.truncation, c.elites = seed, sigma, noise, T, E
    c.max_steps = 900
    c.initial_weight = np.asarray(orc.synthetic_theta(24, 16, 4, seed=x0), dtype=np.float32)
    if log is not None:
        c.batch_env_fn = lambda B: Recording(GymEnvBatch(sw.SynthWalkEnv, B, seed), log.setdefault(B, []))
    for name, v in kw.items():
        setattr(c, name, v)
    return c


def _sweep(configs, kernels=cpu_ops_ga_sweep):
    worker, ga = genetic.build_sweep(configs, kernels=kernels, device='cpu')
    if not worker.host:
        worker.source.horizon = HORIZON
    return genetic.train_sweep(configs, worker=worker, ga=ga), worker, ga


def _train(c):
    worker, ga = genetic.build(c, kernels=K, device='cpu')
    if getattr(c, 'closed_loop', False):
        worker.source.horizon = worker.source.T = HORIZON
    return genetic.train(c, worker, ga), worker, ga


def _assert_run_is_train(run, worker, ga, r, c):
    single, w1, ga1 = _train(c)
    assert run[:2] == single[:2], r
    assert len(run[2]) == len(single[2]), r
    assert torch.equal(ga.parents[r], ga1.parents), r
    assert torch.equal(ga.best[r], ga1.best), r
    assert torch.equal(ga.order[r], ga1.order), r
    assert ga.gens[r] == ga1.gen, r
    if w1.obs_stats is not None:
        assert torch.equal(worker.obs_stats[r], w1.obs_stats), r


def test_the_same_launches_per_generation_for_one_run_and_for_five():
    traces = []
    for R in (1, 5):
        k = Calls(cpu_ops_ga_sweep)
        configs = [_closed(*h, max_generations=2) for h in RUNS[:R]]
        _sweep(configs, kernels=k)
        traces.append(k.names)
    gen = ['rollout_eval_ga_sweep', 'ga_order_runs', 'ga_rows_sweep', 'ga_table', 'rollout_eval_sweep',
           'obs_stats_merge_totals_runs']
    assert traces[0] == traces[1] == ['run_table', 'ga_table', 'rollout_eval_sweep'] + gen * 2


def test_closed_loop_run_r_is_train_of_config_r_with_its_final_table():
    configs = [_closed(*h) for h in RUNS]
    out, worker, ga = _sweep(configs)
    assert ga.rows == 4 and list(ga.T) == [3, 2, 4, 3, 1]
    for r, c in enumerate(configs):
        _assert_run_is_train(out[r], worker, ga, r, c)
    assert out[0][:2] == out[3][:2]                # equal configs, identical runs
    assert out[0][0] != out[1][0]
    assert len({tuple(run[2]) for run in out}) == 1                # one clock


def test_generation_zero_evaluates_one_row_tables():
    configs = [_closed(*h, max_generations=1) for h in RUNS[:3]]
    cpu_ops_ga.CALLS.clear()
    _sweep(configs)
    evals = [x for x in cpu_ops_ga.CALLS if x['op'] == 'rollout_eval_ga']
    assert [(x['n_parents'], x['n_elites'], x['member_offset'], x['seed']) for x in evals] == \
        [(1, 1, 0, 0), (1, 0, 0, 3), (1, 1, 0, 2**40 + 17)]


def test_host_stepped_run_r_is_train_of_config_r_and_stops_where_it_does():
    configs = [_walk(*h) for h in RUNS]
    out, worker, ga = _sweep(configs)
    assert len({len(run[0]) for run in out}) > 1                   # the runs stop at different generations
    for r, c in enumerate(configs):
        _assert_run_is_train(out[r], worker, ga, r, c)
    longest = max(out, key=lambda run: len(run[2]))
    for run in out:                                                 # one clock
        assert run[2] == longest[2][:len(run[2])]


def test_every_runs_environments_get_the_calls_of_its_standalone_run_and_none_after_it_stops():
    logs = [({}, {}) for _ in RUNS]
    configs = [_walk(*h, log=logs[r][0]) for r, h in enumerate(RUNS)]
    out, _, _ = _sweep(configs)
    assert len({len(run[0]) for run in out}) > 1
    for r, h in enumerate(RUNS):
        _train(_walk(*h, log=logs[r][1]))
        sweep, single = logs[r]
        assert sorted(sweep) == sorted(single) == [2, 10], r       # the test and the member batch environments
        for B in single:
            assert len(sweep[B]) == len(single[B]), (r, B)
            for a, b in zip(sweep[B], single[B]):
                assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])), (r, B)


def test_a_stopped_runs_table_and_order_stay_as_they_were():
    configs = [_walk(*h) for h in RUNS]
    worker, ga = genetic.build_sweep(configs, kernels=cpu_ops_ga_sweep, device='cpu')
    f = worker.run(ga)
    ga.tell(f)
    ga.stop(1)
    table, order = ga.parents[1].clone(), ga.order[1].clone()
    for _ in range(2):
        ga.tell(worker.run(ga))
    assert torch.equal(ga.parents[1], table) and torch.equal(ga.order[1], order)
    assert ga.gens[1] == 1 and ga.gens[0] == 3


def _changed(make, field, value):
    cs = [make(*h) for h in RUNS[:3]]
    setattr(cs[1], field, value)
    return cs


@pytest.mark.parametrize('field,value', [
    ('task', 'Pendulum-v1'), ('hidden_size', 32), ('pop_size', 8), ('repetitions', 3), ('test_repetitions', 2),
    ('clip', 1.0), ('normalize_obs', False), ('max_steps', 1000), ('max_generations', 2),
])
def test_closed_loop_sweep_names_the_first_shared_field_that_differs(field, value):
    with pytest.raises(ValueError, match=r'configs differ in %s \(' % field):
        genetic.train_sweep(_changed(_closed, field, value))


@pytest.mark.parametrize('field,value', [
    ('hidden_size', 32), ('pop_size', 6), ('state_dim', 12), ('action_dim', 2), ('repetitions', 3),
    ('test_repetitions', 3), ('clip', 2.0), ('normalize_obs', False), ('max_steps', 1000), ('max_generations', 3),
])
def test_host_sweep_names_the_first_shared_field_that_differs(field, value):
    with pytest.raises(ValueError, match=r'configs differ in %s \(' % field):
        genetic.train_sweep(_changed(_walk, field, value))


def test_sweep_configs_may_differ_in_what_the_runs_own():
    cs = [_closed(*h) for h in RUNS[:3]]
    cs[1].learning_rate, cs[1].weight_decay, cs[1].tag = 0.5, 0.1, 'other'    # not read by the genetic algorithm
    genetic.check_sweep_configs(cs)
    hs = [_walk(*h) for h in RUNS[:2]]
    hs[1].batch_env_fn, hs[1].task = (lambda B: GymEnvBatch(sw.SynthWalkEnv, B, 1)), 'other'
    genetic.check_sweep_configs(hs)


@pytest.mark.parametrize('first,make,match', [
    (_closed, lambda: cfg.PendulumConfig(16), 'configs\\[1\\] is a tape config'),
    (_closed, lambda: _walk(*RUNS[0]), 'configs\\[1\\] is host-stepped and configs\\[0\\] is not'),
    (_walk, lambda: _closed(*RUNS[0]), 'configs\\[0\\] is host-stepped and configs\\[1\\] is not'),
    (_closed, lambda: _closed(*RUNS[1], mirrored=True), 'configs\\[1\\] asks for mirrored sampling'),
    (_closed, lambda: _closed(*RUNS[1], pop_size=2049), 'pop_size 2049 > 2048.*DES_ERR_UNSUPPORTED'),
    (_closed, lambda: _closed(*RUNS[1], pop_size=1), 'configs\\[1\\]: genetic: pop_size 1 < 2'),
    (_closed, lambda: _closed(*RUNS[1], truncation=7), 'configs\\[1\\]: genetic: truncation 7 is not in \\[1, pop_size = 6\\]'),
    (_closed, lambda: _closed(*RUNS[1], truncation=0), 'configs\\[1\\]: genetic: truncation 0 is not in'),
    (_closed, lambda: _closed(*RUNS[1], elites=3), 'configs\\[1\\]: genetic: elites 3 is not in \\[0, truncation = 2\\]'),
    (_closed, lambda: _closed(*RUNS[1], elites=-1), 'configs\\[1\\]: genetic: elites -1 is not in'),
])
def test_sweep_refuses_what_it_cannot_train(first, make, match):
    with pytest.raises(ValueError, match=match):
        genetic.train_sweep([first(*RUNS[0]), make()])


def test_sweep_refuses_an_empty_list():
    with pytest.raises(ValueError, match='no configs'):
        genetic.train_sweep([])


def _world_of_two():
    try:
        genetic.train_sweep([_closed(*h) for h in RUNS[:2]])
    except ValueError as e:
        assert 'world size 2' in str(e), e
        return
    raise AssertionError('train_sweep accepted a process group of 2')


def test_sweep_refuses_a_process_group_of_several_ranks():
    spawn(2, _world_of_two)


def test_multi_runs_batched_writes_the_rewards_and_steps_of_the_sequential_runs(tmp_path, monkeypatch):
    train, train_sweep = genetic.train, genetic.train_sweep       # multi_runs' trainers, with the short horizon

    def short_train(c, worker, ga):
        worker.source.horizon = worker.source.T = HORIZON
        return train(c, worker, ga)

    def short_sweep(configs, worker, ga):
        worker.source.horizon = HORIZON
        return train_sweep(configs, worker, ga)
    monkeypatch.setattr(genetic, 'train', short_train)
    monkeypatch.setattr(genetic, 'train_sweep', short_sweep)
    config = _closed(5, 0.05, 0.1, 0, 3, 1, max_generations=2)
    config.tag = 'ga'
    out = {}
    for batched in (False, True):
        d = tmp_path / str(batched)
        stats = genetic.multi_runs(config, runs=3, log_dir=str(d / 'log'), data_dir=str(d / 'data'),
                                   kernels=cpu_ops_ga_sweep if batched else K, device='cpu', batched=batched)
        with open(d / 'data' / 'ga-stats-Pendulum-v0.bin', 'rb') as f:
            out[batched] = pickle.load(f)
        assert out[batched] == stats and len(stats) == 3
        assert (d / 'log' / 'ga-Pendulum-v0.txt').exists()
    for a, b in zip(out[False], out[True]):
        assert a[:2] == b[:2]
    assert out[False][0][0] != out[False][1][0]                      # seeds config.seed + r: independent runs
    assert config.seed == 5
