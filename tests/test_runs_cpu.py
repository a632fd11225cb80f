"""The host logic of run batches without a GPU: engine.RolloutRunsEngine and natural_es.train_runs over the
oracle-backed stand-in of cpu_ops_runs.py (the single-population stand-ins of cpu_ops applied run by run).  The launches
of a generation do not depend on the number of runs, every config train_runs cannot batch is refused by name, run 0 is
train()'s run, and multi_runs(batched=True) writes the reference's pickle with one entry per run."""
import os
import pickle

import numpy as np
import pytest
import torch
import torch.distributed as dist

import cpu_ops
import cpu_ops_runs
import host_env_support as hs
from distributedes_b200 import config as cfg
from distributedes_b200 import natural_es
from distributedes_b200.engine import RolloutRunsEngine
from ranks import spawn


class Calls:
    """Forwards to `module` and records the name of each function called."""

    def __init__(self, module):
        self._m, self.names = module, []
        self.__name__ = module.__name__

    def __getattr__(self, name):
        f = getattr(self._m, name)
        if not callable(f):
            return f

        def call(*a, **kw):
            self.names.append(name)
            return f(*a, **kw)
        return call


def _engine(R, kernels, **kw):
    P = cpu_ops.param_count(3, 16, 1)
    theta0 = np.random.default_rng(0).standard_normal(P).astype(np.float32) * 0.3
    return RolloutRunsEngine(hidden=16, pop_size=4, runs=R, theta0=theta0, sigma=0.1, learning_rate=0.05, repetitions=2,
                             horizon=12, seed=5, kernels=kernels, device='cpu', **kw)


def _config(**kw):
    c = cfg.ClosedLoopPendulumConfig(16)
    c.pop_size, c.repetitions, c.test_repetitions, c.max_generations = 4, 2, 2, 2
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_a_generation_launches_the_same_ops_for_one_run_and_for_five():
    traces = []
    for R in (1, 5):
        k = Calls(cpu_ops_runs)
        e = _engine(R, k)
        k.names.clear()
        e.generation()
        e.test_returns()
        traces.append(k.names)
    assert traces[0] == traces[1] == ['rollout_eval_runs', 'centered_rank_runs', 'nes_grad_partial_runs',
                                      'nes_apply_runs', 'state_advance', 'obs_stats_merge_totals_runs',
                                      'rollout_eval_runs']


def test_run_r_is_the_single_population_at_member_offset_r_times_n():
    e = _engine(3, cpu_ops_runs)
    theta0 = e.theta_numpy()[0].copy()
    e.generation()
    e.generation()
    for r in range(3):
        theta = torch.from_numpy(theta0.copy())
        st = cpu_ops.new_state('cpu')
        m, v = torch.zeros(e.P, dtype=torch.float64), torch.zeros(e.P, dtype=torch.float64)
        stats, tot = torch.zeros(7), torch.zeros(7, dtype=torch.float64)
        for _ in range(2):
            fit = cpu_ops.rollout_eval(theta, hidden=16, horizon=12, repetitions=2, sigma=0.1, clip=2.0, seed=5, state=st,
                                       member_offset=4 * r, n_local=4, obs_stats=stats, totals_out=tot)
            shaped = cpu_ops.centered_rank(fit, 0, 4)
            part = cpu_ops.nes_grad_partial(shaped, e.P, seed=5, state=st, member_offset=4 * r)
            cpu_ops.nes_apply(theta, m, v, part, 4, st, sigma=0.1, learning_rate=0.05)
            cpu_ops.state_advance(st)
            cpu_ops.obs_stats_merge_totals(stats, tot, 3)
        assert np.array_equal(e.theta_numpy()[r], theta.numpy()), r
        assert np.array_equal(e.fitness_all[r].numpy(), fit.numpy()), r
        assert np.array_equal(e.obs_stats[r].numpy(), stats.numpy()), r


def test_theta0_per_run_and_its_size_check():
    P = cpu_ops.param_count(3, 16, 1)
    shared = _engine(3, cpu_ops_runs)
    assert shared.theta.is_contiguous() and shared.theta.shape == (3, P)        # ops_runs reads it as one [R, P] block
    assert np.array_equal(shared.theta_numpy()[2], shared.theta_numpy()[0])
    rows = np.arange(2 * P, dtype=np.float32).reshape(2, P) * 1e-3
    e = RolloutRunsEngine(hidden=16, pop_size=4, runs=2, theta0=rows, sigma=0.1, learning_rate=0.1, kernels=cpu_ops_runs,
                          device='cpu')
    assert np.array_equal(e.theta_numpy(), rows) and e.theta.is_contiguous()
    with pytest.raises(ValueError, match='theta0 has'):
        RolloutRunsEngine(hidden=16, pop_size=4, runs=3, theta0=rows, sigma=0.1, learning_rate=0.1,
                          kernels=cpu_ops_runs, device='cpu')
    with pytest.raises(ValueError, match=r'pop_size must be in \[2, 2048\]'):
        RolloutRunsEngine(hidden=16, pop_size=2049, runs=1, theta0=rows[0], sigma=0.1, learning_rate=0.1,
                          kernels=cpu_ops_runs, device='cpu')


@pytest.mark.parametrize('make,match', [
    (lambda: cfg.PendulumConfig(16), 'tape configs'),
    (lambda: cfg.HostEnvConfig(hs.PendulumProbe, 16), 'host-stepped'),
    (lambda: _config(mirrored=True), 'mirrored sampling'),
    (lambda: _config(pop_size=2049), 'pop_size 2049 > 2048'),
])
def test_train_runs_names_each_config_it_cannot_batch(make, match):
    with pytest.raises(ValueError, match=match):
        natural_es.train_runs(make(), 2)


def _world_of_two():
    try:
        natural_es.train_runs(_config(), 2)
    except ValueError as e:
        assert 'world size 2' in str(e), e
        return
    raise AssertionError('train_runs accepted a process group of 2')


def test_train_runs_refuses_a_process_group_of_several_ranks():
    spawn(2, _world_of_two)


_build_runs_engine = natural_es.build_runs_engine


def _cpu_runs_engine(config, runs, **kw):
    return _build_runs_engine(config, runs, kernels=cpu_ops_runs, device='cpu', **kw)


def test_run_0_is_train_and_multi_runs_batched_writes_the_reference_pickle(tmp_path, monkeypatch):
    c = _config()
    single = natural_es.train(c, engine=natural_es.build_engine(c, kernels=cpu_ops, device='cpu'))
    monkeypatch.setattr(natural_es, 'build_runs_engine', _cpu_runs_engine)
    stats = natural_es.multi_runs(c, 3, log_dir=str(tmp_path / 'log'), data_dir=str(tmp_path / 'data'), batched=True)
    with open(os.path.join(str(tmp_path / 'data'), '-stats-Pendulum-v0.bin'), 'rb') as f:
        on_disk = pickle.load(f)
    assert isinstance(on_disk, list) and len(on_disk) == 3
    for run in on_disk:
        rewards, steps, stamps = run
        assert len(rewards) == len(steps) == len(stamps) == 3
        assert steps == single[1]
    assert on_disk[0][0] == single[0]
    assert on_disk[1][0] != single[0]                   # another stream of the same seed
    assert [s[0] for s in stats] == [s[0] for s in on_disk]
    assert os.path.exists(os.path.join(str(tmp_path / 'log'), '-Pendulum-v0.txt'))
    assert not dist.is_initialized()
