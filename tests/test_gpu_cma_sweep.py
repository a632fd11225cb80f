"""CMA-ES sweeps on the GPU.  Each sweep entry point is bit-equal, run by run, to the single entry point: the normals
(seeds above 2^32, stream tags 0 and 1), the closed-loop evaluation of explicit rows (every policy width, repetitions 1
and 10, statistics on and off, action noise on and off, a NaN row), the rank-mu partial (n from 1 to 4481 across the
FFMA / tensor-core boundary, lambda from 1 to 100) and the covariance update (a decay per run, pc given or NULL).
cma_es.train_sweep is R cma_es.train calls bit for bit, with each run's final m, sigma, C, p_c, p_sigma and statistics:
closed-loop Pendulum at H = 16 and lambda = 64 (eigen gap 1: eigh every generation) and lambda = 10, a sweep holding the
train_cma_closed_pend golden config, and host-stepped SynthWalk with runs stopping at different generations."""
import copy
import os

import numpy as np
import pytest
import torch

from distributedes_b200.fitness import POLICY_WIDTHS
from oracle import nes_oracle as orc
from oracle import synth_walk as sw

pytestmark = pytest.mark.gpu


def _table(seeds, noise):
    from distributedes_b200 import ops_sweep
    return ops_sweep.run_table(seeds, 1.0, 0.0, 0.0, noise, 'cuda', runs=len(seeds))


def test_noise_fill_sweep_is_the_single_noise_fill_of_each_runs_seed():
    from distributedes_b200 import ops, ops_cma_sweep
    seeds = [3, 2**40 + 5, 2**63 + 11, 3]
    for tag in (0, 1):
        for N, P in ((1, 1), (16, 353), (64, 353), (100, 1217), (2048, 5)):
            z = ops_cma_sweep.noise_fill_sweep(_table(seeds, 0.0), N, P, 7, stream_tag=tag).reshape(len(seeds), N, P)
            for r, s in enumerate(seeds):
                assert torch.equal(z[r], ops.noise_fill(N, P, s, 7, 0, tag)), (tag, N, P, r)
            assert torch.equal(z[0], z[3])


def test_rollout_eval_solutions_sweep_is_the_single_evaluation_of_each_run():
    from distributedes_b200 import ops, ops_cma_sweep
    rng = np.random.default_rng(5)
    seeds = [9, 2**40 + 1, 9]
    for H in POLICY_WIDTHS:
        P = ops.param_count(3, H, 1)
        for reps in (1, 10):
            for stats_on in (False, True):
                for noise in ((0.0, 0.0, 0.0), (0.3, 0.0, 0.1)):
                    R, N = len(seeds), 6
                    rows = torch.from_numpy(rng.standard_normal((R * N, P)).astype(np.float32) * 0.3).cuda()
                    rows[4, 7] = float('nan')
                    stats = torch.from_numpy(np.concatenate(
                        [rng.standard_normal((R, 3)), rng.uniform(0.5, 2.0, (R, 3)), np.full((R, 1), 50.0)],
                        axis=1).astype(np.float32)).cuda() if stats_on else None
                    totals = torch.zeros((R, 7), dtype=torch.float64, device='cuda')
                    episodes = torch.zeros((R, N, reps), dtype=torch.float32, device='cuda')
                    fit = ops_cma_sweep.rollout_eval_solutions_sweep(rows, _table(seeds, list(noise)), hidden=H, clip=2.0,
                                                                     repetitions=reps, generation=3, run_size=N,
                                                                     obs_stats=stats, totals_out=totals,
                                                                     episodes_out=episodes)
                    for r in range(R):
                        t1 = torch.zeros(7, dtype=torch.float64, device='cuda')
                        e1 = torch.zeros((N, reps), dtype=torch.float32, device='cuda')
                        f1 = ops.rollout_eval_solutions(rows[r * N:(r + 1) * N].contiguous(), hidden=H, clip=2.0,
                                                        repetitions=reps, action_noise_std=noise[r], seed=seeds[r],
                                                        generation=3, member_offset=0,
                                                        obs_stats=None if stats is None else stats[r].contiguous(),
                                                        totals_out=t1, episodes_out=e1)
                        key = (H, reps, stats_on, noise, r)
                        assert torch.equal(fit[r], f1) or (torch.isnan(fit[r]) == torch.isnan(f1)).all() and \
                            torch.equal(fit[r].nan_to_num(), f1.nan_to_num()), key
                        assert torch.equal(episodes[r].nan_to_num(), e1.nan_to_num()), key
                        assert torch.equal(totals[r].nan_to_num(), t1.nan_to_num()), key
                    assert torch.isnan(fit[0, 4]), H


@pytest.mark.parametrize('n', [1, 63, 64, 353, 1217, 2047, 2048, 4481])
def test_cma_rank_mu_runs_is_the_single_rank_mu_of_each_run(n):
    from distributedes_b200 import ops, ops_cma_sweep
    rng = np.random.default_rng(n)
    for lam in (1, 16, 64, 100):
        R = 3
        Y = torch.from_numpy(rng.standard_normal((R, lam, n)).astype(np.float32)).cuda()
        Y[1] *= 1e3
        w = torch.from_numpy(rng.uniform(0.0, 1.0, (R, lam)).astype(np.float32)).cuda()
        out = ops_cma_sweep.cma_rank_mu_runs(Y, w)
        for r in range(R):
            assert torch.equal(out[r], ops.cma_rank_mu(Y[r].contiguous(), w[r].contiguous())), (n, lam, r)


def test_cma_cov_apply_runs_is_the_single_update_of_each_run():
    from distributedes_b200 import ops, ops_cma_sweep
    rng = np.random.default_rng(1)
    for n in (1, 63, 353, 2048):
        R = 4
        C0 = torch.from_numpy(rng.standard_normal((R, n, n)).astype(np.float32)).cuda()
        dC = torch.from_numpy(rng.standard_normal((R, n, n)).astype(np.float32)).cuda()
        pc = torch.from_numpy(rng.standard_normal((R, n)).astype(np.float32)).cuda()
        decay = [0.91234567891, 0.95, 0.9123456789, 0.8]
        for with_pc in (True, False):
            C = C0.clone()
            ops_cma_sweep.cma_cov_apply_runs(C, dC, pc if with_pc else None, torch.tensor(decay, dtype=torch.float64,
                                                                                          device='cuda'), c1=1e-3, cmu=2e-2)
            for r in range(R):
                C1 = C0[r].clone()
                ops.cma_cov_apply(C1, dC[r].contiguous(), pc[r].contiguous() if with_pc else None, decay=decay[r],
                                  c1=1e-3, cmu=2e-2)
                assert torch.equal(C[r], C1), (n, with_pc, r)


def _assert_runs_are_train(configs, out, worker, es):
    from distributedes_b200 import cma_es
    for r, c in enumerate(configs):
        w1 = cma_es.Worker(0, None, None, None, None, c)
        es1 = cma_es.CMAEvolutionStrategy(c.initial_weight, c.sigma, c.pop_size, seed=c.seed, device=w1.device,
                                          kernels=w1.kn)
        single = cma_es.train(c, worker=w1, es=es1)
        assert out[r][0] == single[0] and out[r][1] == single[1], r
        mine = es.es[r]
        for name in ('m', 'C', 'pc', 'ps'):
            assert torch.equal(getattr(mine, name), getattr(es1, name)), (r, name)
        assert mine.sigma == es1.sigma and mine.gen == es1.gen, r
        if w1.obs_stats is not None:
            assert torch.equal(worker.obs_stats[r], w1.obs_stats), r


def _closed(seed, sigma, noise, x0, gens=4, lam=64):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(16)
    c.pop_size, c.max_generations, c.seed, c.sigma, c.action_noise_std = lam, gens, seed, sigma, noise
    c.initial_weight = np.asarray(orc.synthetic_theta(3, 16, 1, seed=x0), dtype=np.float32)
    return c


@pytest.mark.parametrize('lam', [64, 10])         # 10 x 353 floats: a run's z starts 8 bytes past a 16-byte boundary
def test_train_sweep_closed_loop_runs_are_train_bit_for_bit(lam):
    from distributedes_b200 import cma_es
    configs = [_closed(*h, lam=lam, gens=4 if lam == 64 else 7) for h in ((1, 1.0, 0.0, 0), (2**40 + 3, 0.5, 0.2, 1),
                                                                          (1, 1.0, 0.0, 0), (7, 2.0, 0.1, 2))]
    worker, es = cma_es.build_sweep(configs)
    assert es.es[0].eigen_gap == (1 if lam == 64 else 6)          # lambda = 10: one eigh, after the sixth tell
    out = cma_es.train_sweep(configs, worker=worker, es=es)
    _assert_runs_are_train(configs, out, worker, es)
    assert out[0][:2] == out[2][:2] and out[0][0] != out[1][0]


def test_train_sweep_runs_the_cma_closed_pend_golden_config_as_train_does():
    from distributedes_b200 import cma_es
    from test_gpu_goldens import device_rollouts
    with np.load(os.path.join(os.path.dirname(__file__), 'golden', 'train_cma_closed_pend.npz'), allow_pickle=False) as z:
        g = {k: z[k] for k in z.files}
    golden = device_rollouts(g)
    configs = []
    for s, sigma, noise in ((int(g['seed']) + 1, 0.5, 0.1), (None, None, None), (int(g['seed']) + 2**33, 2.0, 0.0)):
        c = copy.copy(golden)
        if s is not None:
            c.seed, c.sigma, c.action_noise_std = s, sigma, noise
            c.initial_weight = golden.initial_weight * np.float32(0.5)
        configs.append(c)
    worker, es = cma_es.build_sweep(configs)
    out = cma_es.train_sweep(configs, worker=worker, es=es)
    _assert_runs_are_train(configs, out, worker, es)
    assert out[1][1] == list(g['train_steps'])


def test_train_sweep_host_stepped_runs_are_train_and_stop_where_it_does():
    from distributedes_b200 import cma_es
    from distributedes_b200.config import HostEnvConfig
    configs = []
    for seed, sigma, noise, x0 in ((0, 0.1, 0.0, 0), (3, 0.05, 0.2, 1), (2**40 + 17, 0.2, 0.1, 2), (9, 0.02, 0.0, 1)):
        c = HostEnvConfig(sw.SynthWalkEnv, 16, task='SynthWalk-v0')
        c.pop_size, c.repetitions, c.test_repetitions, c.max_steps = 16, 2, 2, 6000
        c.seed, c.sigma, c.action_noise_std = seed, sigma, noise
        c.initial_weight = np.asarray(orc.synthetic_theta(24, 16, 4, seed=x0), dtype=np.float32)
        configs.append(c)
    worker, es = cma_es.build_sweep(configs)
    out = cma_es.train_sweep(configs, worker=worker, es=es)
    assert len({len(run[0]) for run in out}) > 1
    _assert_runs_are_train(configs, out, worker, es)
