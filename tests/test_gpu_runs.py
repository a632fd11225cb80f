"""Run batches on the GPU.  Every run-batched entry point is bit-equal, run by run, to the single-population entry point
it extends (rollouts at member_offset r*N, the rank within a run, the partial at member_offset r*N, Adam, the statistics
merge), across batch shapes, policy widths, statistics, action noise, both sources of the generation word, the
noiseless test mode and ranks with ties and NaN.  RolloutRunsEngine's run 0 is RolloutEngine's run and its other runs
are the single ops composed at their member offsets, eagerly and as a CUDA graph; the first generation's fitness of
every run matches the oracle; train_runs' run 0 is train()."""
import numpy as np
import pytest
import torch

from distributedes_b200.fitness import POLICY_WIDTHS
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu

SHAPES = [(R, N) for R in (1, 3, 10) for N in (2, 64, 257)]
RTOL = 2e-4                   # closed-loop fitness against the oracle (tests/test_gpu_rollout.py)


def _stats(R, rng):
    """Normaliser statistics [R, 7] that differ per run: small means, positive variances, a positive count."""
    s = np.zeros((R, 7), np.float32)
    s[:, :3] = rng.normal(0, 0.3, (R, 3))
    s[:, 3:6] = rng.uniform(0.2, 3.0, (R, 3))
    s[:, 6] = rng.integers(100, 10000, R)
    return torch.from_numpy(s).cuda()


def _thetas(R, H, rng):
    P = orc.param_count(3, H, 1)
    return torch.from_numpy((rng.standard_normal((R, P)) * 0.3).astype(np.float32)).cuda()


@pytest.mark.parametrize('R,N', SHAPES)
def test_rollout_runs_is_the_single_rollout_at_each_run_offset(R, N):
    from distributedes_b200 import ops, ops_runs
    rng = np.random.default_rng(R * 1000 + N)
    for i, H in enumerate(POLICY_WIDTHS):
        theta = _thetas(R, H, rng)
        stats = _stats(R, rng) if i % 2 else None
        noise = 0.3 if i % 3 != 1 else 0.0
        word = dict(state=ops.new_state('cuda', 5)) if i % 2 == 0 else dict(generation=5)
        kw = dict(hidden=H, horizon=40, repetitions=3, sigma=0.1, clip=2.0, action_noise_std=noise, seed=11, **word)
        tot = torch.empty((R, 7), dtype=torch.float64, device='cuda')
        ep = torch.empty((R, N, 3), dtype=torch.float32, device='cuda')
        fit = ops_runs.rollout_eval_runs(theta, run_size=N, obs_stats=stats, totals_out=tot, episodes_out=ep, **kw)
        for r in range(R):
            t1 = torch.empty(7, dtype=torch.float64, device='cuda')
            e1 = torch.empty((N, 3), dtype=torch.float32, device='cuda')
            f1 = ops.rollout_eval(theta[r], member_offset=r * N, n_local=N, obs_stats=None if stats is None else stats[r],
                                  totals_out=t1, episodes_out=e1, **kw)
            assert torch.equal(fit[r], f1), (H, r)
            assert torch.equal(ep[r], e1), (H, r)
            assert torch.equal(tot[r], t1), (H, r)


@pytest.mark.parametrize('R', (1, 3, 10))
@pytest.mark.parametrize('noise', (0.0, 0.3))
def test_noiseless_runs_are_each_runs_test_episodes(R, noise):
    from distributedes_b200 import ops, ops_runs
    rng = np.random.default_rng(R)
    for H in POLICY_WIDTHS:
        theta, stats = _thetas(R, H, rng), _stats(R, rng)
        st = ops.new_state('cuda', 7)
        kw = dict(hidden=H, repetitions=10, sigma=0.0, clip=2.0, action_noise_std=noise, seed=2, state=st, noiseless=True)
        ep = torch.empty((R, 1, 10), dtype=torch.float32, device='cuda')
        ops_runs.rollout_eval_runs(theta, run_size=1, obs_stats=stats, episodes_out=ep, **kw)
        for r in range(R):
            e1 = torch.empty(10, dtype=torch.float32, device='cuda')
            ops.rollout_eval(theta[r], member_offset=r, n_local=1, obs_stats=stats[r], episodes_out=e1, **kw)
            assert torch.equal(ep[r, 0], e1), (H, r)
            if noise == 0.0:              # without action noise, exactly what a single engine's test_returns runs
                e0 = torch.empty(10, dtype=torch.float32, device='cuda')
                ops.rollout_eval(theta[r], member_offset=0, n_local=1, obs_stats=stats[r], episodes_out=e0, **kw)
                assert torch.equal(ep[r, 0], e0), (H, r)


@pytest.mark.parametrize('R,N', SHAPES)
def test_rank_runs_ranks_within_each_run(R, N):
    from distributedes_b200 import ops, ops_runs
    rng = np.random.default_rng(N)
    f = rng.integers(-5, 5, (R, N)).astype(np.float32)          # many ties
    f[rng.random((R, N)) < 0.1] = np.nan
    f[:, 0] = -0.0
    fit = torch.from_numpy(f).cuda()
    shaped, ranks = ops_runs.centered_rank_runs(fit, return_ranks=True)
    for r in range(R):
        s1, k1 = ops.centered_rank(fit[r].contiguous(), return_ranks=True)
        assert torch.equal(shaped[r], s1) and torch.equal(ranks[r], k1), r


@pytest.mark.parametrize('R,N', SHAPES)
def test_grad_runs_is_the_single_partial_at_each_run_offset(R, N):
    from distributedes_b200 import ops, ops_runs
    rng = np.random.default_rng(7 * N + R)
    for H in POLICY_WIDTHS:
        P = orc.param_count(3, H, 1)
        shaped = torch.from_numpy(rng.uniform(-0.5, 0.5, (R, N)).astype(np.float32)).cuda()
        for word in (dict(state=ops.new_state('cuda', 3)), dict(generation=3)):
            part = ops_runs.nes_grad_partial_runs(shaped, P, seed=9, **word)
            for r in range(R):
                p1 = ops.nes_grad_partial(shaped[r].contiguous(), P, seed=9, member_offset=r * N, **word)
                assert torch.equal(part[r], p1), (H, r)


@pytest.mark.parametrize('R,N', SHAPES)
def test_apply_and_merge_runs_are_the_single_ops_per_run(R, N):
    from distributedes_b200 import ops, ops_runs
    rng = np.random.default_rng(R + N)
    P = orc.param_count(3, 64, 1)
    st = ops.new_state('cuda', 0)
    for _ in range(3):
        ops.state_advance(st)

    def t(shape, dtype=np.float32, scale=1.0):
        return torch.from_numpy((rng.standard_normal(shape) * scale).astype(dtype)).cuda()
    theta, m, v = t((R, P)), t((R, P), np.float64, 0.1), t((R, P), np.float64, 0.01).abs()
    partial = t((R, P), scale=5.0)
    th, mm, vv = theta.clone(), m.clone(), v.clone()
    upd, grad = torch.empty_like(theta), torch.empty_like(m)
    kw = dict(sigma=0.05, learning_rate=0.02, weight_decay=0.005)
    ops_runs.nes_apply_runs(th, mm, vv, partial, N, st, update_out=upd, grad_out=grad, **kw)
    stats, totals = _stats(R, rng), torch.from_numpy(np.abs(rng.standard_normal((R, 7))) * 50).cuda()
    merged = ops_runs.obs_stats_merge_totals_runs(stats.clone(), totals, 3)
    for r in range(R):
        t1, m1, v1 = theta[r].clone(), m[r].clone(), v[r].clone()
        u1, g1 = torch.empty_like(t1), torch.empty_like(m1)
        ops.nes_apply(t1, m1, v1, partial[r].contiguous(), N, st, update_out=u1, grad_out=g1, **kw)
        assert torch.equal(th[r], t1) and torch.equal(mm[r], m1) and torch.equal(vv[r], v1), r
        assert torch.equal(upd[r], u1) and torch.equal(grad[r], g1), r
        s1 = ops.obs_stats_merge_totals(stats[r].clone(), totals[r].contiguous(), 3)
        assert torch.equal(merged[r], s1), r


def _single_chain(theta0, r, N, H, gens, seed, sigma, lr):
    """Run r of a batch composed from the single-population ops at member_offset r*N."""
    from distributedes_b200 import ops
    theta = torch.from_numpy(theta0.copy()).cuda()
    P = theta.numel()
    st = ops.new_state('cuda', 0)
    m, v = torch.zeros(P, dtype=torch.float64, device='cuda'), torch.zeros(P, dtype=torch.float64, device='cuda')
    stats, tot = torch.zeros(7, device='cuda'), torch.zeros(7, dtype=torch.float64, device='cuda')
    for _ in range(gens):
        fit = ops.rollout_eval(theta, hidden=H, repetitions=10, sigma=sigma, clip=2.0, seed=seed, state=st,
                               member_offset=r * N, n_local=N, obs_stats=stats, totals_out=tot)
        shaped = ops.centered_rank(fit)
        part = ops.nes_grad_partial(shaped, P, seed=seed, state=st, member_offset=r * N)
        ops.nes_apply(theta, m, v, part, N, st, sigma=sigma, learning_rate=lr)
        ops.state_advance(st)
        ops.obs_stats_merge_totals(stats, tot, 3)
    return theta, fit, stats


def test_runs_engine_run_0_is_rollout_engine_and_runs_1_to_3_the_composed_ops():
    from distributedes_b200.engine import RolloutEngine, RolloutRunsEngine
    H, N, R, seed, sigma, lr = 64, 64, 4, 3, 0.1, 0.05
    theta0 = orc.synthetic_theta(3, H, 1, seed=4)
    kw = dict(hidden=H, pop_size=N, theta0=theta0, sigma=sigma, learning_rate=lr, seed=seed)
    eager = RolloutRunsEngine(runs=R, use_graph=False, **kw)
    graph = RolloutRunsEngine(runs=R, use_graph=True, **kw)
    single = RolloutEngine(**kw)
    for _ in range(3):
        eager.generation()
        graph.generation()
        single.generation()
        assert torch.equal(eager.theta[0], single.theta) and torch.equal(eager.fitness_all[0], single.fitness_all)
        assert torch.equal(eager.obs_stats[0], single.obs_stats)
    for name in ('theta', 'fitness_all', 'obs_stats', 'adam_m', 'adam_v', 'state'):
        assert torch.equal(getattr(eager, name), getattr(graph, name)), name
    for r in range(1, R):
        theta, fit, stats = _single_chain(theta0, r, N, H, 3, seed, sigma, lr)
        assert torch.equal(eager.theta[r], theta) and torch.equal(eager.fitness_all[r], fit), r
        assert torch.equal(eager.obs_stats[r], stats), r
    assert not torch.equal(eager.theta[1], eager.theta[0])
    test = eager.test_returns()
    assert test.shape == (R, 10)
    assert np.array_equal(test[0], single.test_returns())


def test_first_generation_fitness_of_every_run_matches_the_oracle():
    from distributedes_b200.engine import RolloutRunsEngine
    H, N, R = 64, 16, 3
    theta0 = orc.synthetic_theta(3, H, 1, seed=6)
    e = RolloutRunsEngine(hidden=H, pop_size=N, runs=R, theta0=theta0, sigma=0.1, learning_rate=0.05, seed=8,
                          use_graph=False)
    fit = e.evaluate().cpu().numpy().astype(np.float64)
    for r in range(R):
        ref, _ = po.closed_fitness(theta0, H, 0.1, 8, 0, r * N, N, 10)
        assert np.max(np.abs(fit[r] - ref) / np.abs(ref)) < RTOL, r


def test_train_runs_run_0_is_train():
    from distributedes_b200 import config as cfg
    from distributedes_b200 import natural_es
    c = cfg.ClosedLoopPendulumConfig(64)
    c.pop_size, c.max_generations = 64, 3
    single = natural_es.train(c)
    runs = natural_es.train_runs(c, 5)
    assert len(runs) == 5
    assert runs[0][0] == single[0] and runs[0][1] == single[1]
    assert all(run[1] == single[1] for run in runs)
    assert runs[1][0] != single[0]
