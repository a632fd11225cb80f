"""Sweeps on the GPU.  Every sweep entry point is bit-equal, run by run, to the single-population entry point with run r's
seed and hyper-parameters at member_offset 0 (rollouts, the partial, Adam), across batch shapes from 2 to 2048 members,
every policy width, statistics on and off, action noise off and on, both sources of the generation word and the
noiseless test mode.  RolloutRunsEngine(seeds=...) is R RolloutEngines, graph-replayed; train_sweep's run r is
train(configs[r]), the golden config among them; the first generation's fitness of every run matches the oracle under its
own seed."""
import copy
import os

import numpy as np
import pytest
import torch

from distributedes_b200.fitness import POLICY_WIDTHS
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu

SHAPES = [(1, 2), (3, 2), (4, 64), (3, 257), (2, 2048)]
RTOL = 2e-4                   # closed-loop fitness against the oracle (tests/test_gpu_rollout.py)


def _hyper(R, rng, noise=True):
    """Per-run seeds (two runs share one), sigma, learning rate, weight decay and action noise."""
    seeds = [int(s) for s in rng.integers(0, 2**63, R)]
    if R > 2:
        seeds[2] = seeds[0]
    return dict(seeds=seeds, sigma=list(rng.uniform(0.02, 0.3, R)), learning_rate=list(rng.uniform(0.01, 0.2, R)),
                weight_decay=list(rng.uniform(0.0, 0.02, R)),
                action_noise_std=list(rng.uniform(0.1, 0.5, R)) if noise else [0.0] * R)


def _table(h):
    from distributedes_b200 import ops_sweep
    return ops_sweep.run_table(h['seeds'], h['sigma'], h['learning_rate'], h['weight_decay'], h['action_noise_std'],
                               'cuda')


def _stats(R, rng):
    s = np.zeros((R, 7), np.float32)
    s[:, :3] = rng.normal(0, 0.3, (R, 3))
    s[:, 3:6] = rng.uniform(0.2, 3.0, (R, 3))
    s[:, 6] = rng.integers(100, 10000, R)
    return torch.from_numpy(s).cuda()


def _thetas(R, H, rng):
    P = orc.param_count(3, H, 1)
    return torch.from_numpy((rng.standard_normal((R, P)) * 0.3).astype(np.float32)).cuda()


@pytest.mark.parametrize('R,N', SHAPES)
def test_rollout_sweep_is_the_single_rollout_of_each_runs_seed(R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(R * 1000 + N)
    for i, H in enumerate(POLICY_WIDTHS):
        theta = _thetas(R, H, rng)
        stats = _stats(R, rng) if i % 2 else None
        h = _hyper(R, rng, noise=i % 3 != 1)
        word = dict(state=ops.new_state('cuda', 5)) if i % 2 == 0 else dict(generation=5)
        kw = dict(hidden=H, horizon=40, repetitions=3, clip=2.0, **word)
        tot = torch.empty((R, 7), dtype=torch.float64, device='cuda')
        ep = torch.empty((R, N, 3), dtype=torch.float32, device='cuda')
        fit = ops_sweep.rollout_eval_sweep(theta, _table(h), run_size=N, obs_stats=stats, totals_out=tot,
                                           episodes_out=ep, **kw)
        for r in range(R):
            t1 = torch.empty(7, dtype=torch.float64, device='cuda')
            e1 = torch.empty((N, 3), dtype=torch.float32, device='cuda')
            f1 = ops.rollout_eval(theta[r], member_offset=0, n_local=N, obs_stats=None if stats is None else stats[r],
                                  totals_out=t1, episodes_out=e1, seed=h['seeds'][r], sigma=h['sigma'][r],
                                  action_noise_std=h['action_noise_std'][r], **kw)
            assert torch.equal(fit[r], f1), (H, r)
            assert torch.equal(ep[r], e1), (H, r)
            assert torch.equal(tot[r], t1), (H, r)


@pytest.mark.parametrize('R', (1, 3, 10))
@pytest.mark.parametrize('noise', (False, True))
def test_noiseless_sweep_is_each_runs_test_episodes(R, noise):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(R + 100 * noise)
    for H in POLICY_WIDTHS:
        theta, stats, h = _thetas(R, H, rng), _stats(R, rng), _hyper(R, rng, noise)
        st = ops.new_state('cuda', 7)
        kw = dict(hidden=H, repetitions=10, clip=2.0, state=st, noiseless=True)
        ep = torch.empty((R, 1, 10), dtype=torch.float32, device='cuda')
        ops_sweep.rollout_eval_sweep(theta, _table(h), run_size=1, obs_stats=stats, episodes_out=ep, **kw)
        for r in range(R):
            e1 = torch.empty(10, dtype=torch.float32, device='cuda')
            ops.rollout_eval(theta[r], member_offset=0, n_local=1, obs_stats=stats[r], episodes_out=e1, sigma=0.0,
                             seed=h['seeds'][r], action_noise_std=h['action_noise_std'][r], **kw)
            assert torch.equal(ep[r, 0], e1), (H, r)


@pytest.mark.parametrize('R,N', SHAPES)
def test_grad_sweep_is_the_single_partial_of_each_runs_seed(R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(7 * N + R)
    for H in POLICY_WIDTHS:
        P = orc.param_count(3, H, 1)
        shaped = torch.from_numpy(rng.uniform(-0.5, 0.5, (R, N)).astype(np.float32)).cuda()
        h = _hyper(R, rng)
        for word in (dict(state=ops.new_state('cuda', 3)), dict(generation=3)):
            part = ops_sweep.nes_grad_partial_sweep(shaped, P, _table(h), **word)
            for r in range(R):
                p1 = ops.nes_grad_partial(shaped[r].contiguous(), P, seed=h['seeds'][r], member_offset=0, **word)
                assert torch.equal(part[r], p1), (H, r)


@pytest.mark.parametrize('R,N', SHAPES)
def test_apply_sweep_is_the_single_apply_with_each_runs_optimiser(R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(R + N)
    P = orc.param_count(3, 64, 1)
    st = ops.new_state('cuda', 0)
    for _ in range(3):
        ops.state_advance(st, 0.8, 0.99)

    def t(shape, dtype=np.float32, scale=1.0):
        return torch.from_numpy((rng.standard_normal(shape) * scale).astype(dtype)).cuda()
    theta, m, v = t((R, P)), t((R, P), np.float64, 0.1), t((R, P), np.float64, 0.01).abs()
    partial = t((R, P), scale=5.0)
    th, mm, vv = theta.clone(), m.clone(), v.clone()
    upd, grad = torch.empty_like(theta), torch.empty_like(m)
    h = _hyper(R, rng)
    adam = dict(beta1=0.8, beta2=0.99, epsilon=1e-7)
    ops_sweep.nes_apply_sweep(th, mm, vv, partial, N, st, _table(h), update_out=upd, grad_out=grad, **adam)
    for r in range(R):
        t1, m1, v1 = theta[r].clone(), m[r].clone(), v[r].clone()
        u1, g1 = torch.empty_like(t1), torch.empty_like(m1)
        ops.nes_apply(t1, m1, v1, partial[r].contiguous(), N, st, update_out=u1, grad_out=g1, sigma=h['sigma'][r],
                      learning_rate=h['learning_rate'][r], weight_decay=h['weight_decay'][r], **adam)
        assert torch.equal(th[r], t1) and torch.equal(mm[r], m1) and torch.equal(vv[r], v1), r
        assert torch.equal(upd[r], u1) and torch.equal(grad[r], g1), r


def test_sweep_engine_is_r_rolloutengines():
    from distributedes_b200.engine import RolloutEngine, RolloutRunsEngine
    H, N, R = 64, 64, 4
    rng = np.random.default_rng(4)
    h = _hyper(R, rng)
    theta0 = np.stack([orc.synthetic_theta(3, H, 1, seed=s) for s in range(R)])
    sweep = RolloutRunsEngine(hidden=H, pop_size=N, runs=R, theta0=theta0, use_graph=True, **h)
    singles = [RolloutEngine(hidden=H, pop_size=N, theta0=theta0[r], seed=h['seeds'][r], sigma=h['sigma'][r],
                             learning_rate=h['learning_rate'][r], weight_decay=h['weight_decay'][r],
                             action_noise_std=h['action_noise_std'][r], use_graph=True) for r in range(R)]
    for _ in range(3):
        sweep.generation()
        for e in singles:
            e.generation()
    test = sweep.test_returns()
    for r, e in enumerate(singles):
        for name in ('theta', 'adam_m', 'adam_v', 'fitness_all', 'obs_stats'):
            assert torch.equal(getattr(sweep, name)[r], getattr(e, name)), (name, r)
        assert np.array_equal(test[r], e.test_returns()), r
    assert torch.equal(sweep.state, singles[0].state)


def test_train_sweep_runs_the_golden_config_as_train_does():
    from distributedes_b200 import natural_es
    from test_gpu_goldens import device_rollouts
    with np.load(os.path.join(os.path.dirname(__file__), 'golden', 'train_closed_pend.npz'), allow_pickle=False) as z:
        g = {k: z[k] for k in z.files}
    golden = device_rollouts(g)
    configs = []
    for s in (int(g['seed']) + 1, None, int(g['seed']) + 7):
        c = copy.copy(golden)
        if s is not None:
            c.seed = s
        configs.append(c)
    out = natural_es.train_sweep(configs)
    for c, run in zip(configs, out):
        single = natural_es.train(c)
        assert run[0] == single[0] and run[1] == single[1], c.seed
    assert out[1][0] != out[0][0]


def test_first_generation_fitness_of_every_run_matches_the_oracle_under_its_seed():
    from distributedes_b200.engine import RolloutRunsEngine
    H, N, R = 64, 16, 3
    rng = np.random.default_rng(8)
    h = _hyper(R, rng, noise=False)
    theta0 = orc.synthetic_theta(3, H, 1, seed=6)
    e = RolloutRunsEngine(hidden=H, pop_size=N, runs=R, theta0=theta0, use_graph=False, **h)
    fit = e.evaluate().cpu().numpy().astype(np.float64)
    for r in range(R):
        ref, _ = po.closed_fitness(theta0, H, h['sigma'][r], h['seeds'][r], 0, 0, N, 10)
        assert np.max(np.abs(fit[r] - ref) / np.abs(ref)) < RTOL, r
