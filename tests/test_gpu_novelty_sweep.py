"""Novelty-search sweeps on the GPU, every entry point run by run against its single-run call, bit for bit:

  - des_rollout_eval_bc_sweep equals des_rollout_eval_bc of each run (its seed, sigma and action noise, member offset 0)
    at every width, members and test episodes, statistics on, R = 3; its fitness, returns and totals equal
    des_rollout_eval_sweep's;
  - des_novelty_runs equals des_novelty of each run on the integer and real cases of test_gpu_novelty.py (NaN rows, A < k,
    A across a 256-row tile, A < capacity with NaN in the unused rows), and at run counts where a run spans many CTAs;
  - des_ns_shape_runs equals des_ns_shape of each run with w in {0, 0.3, 0.5, 1}, and des_centered_rank_runs with every
    w = 1;
  - novelty.train_sweep equals sequential novelty.train, closed-loop (H = 32, N = 64, four runs mixing w and 'adaptive')
    and host-stepped; with every w = 1 it equals natural_es.train_sweep.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from host_env_support import PendulumProbe
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from test_gpu_novelty import CASES, _integer_rows, _same

pytestmark = pytest.mark.gpu
WIDTHS = (16, 32, 64, 96, 128)
# seed, sigma, action noise of each run
HP = ((11, 0.05, 0.1), (2**40 + 5, 0.02, 0.0), (3, 0.1, 0.3))


def _ops():
    from distributedes_b200 import ops, ops_runs
    return ops, ops_runs


def _bytes(t):
    return t.cpu().numpy().tobytes()


@pytest.mark.parametrize('noiseless', [False, True])
@pytest.mark.parametrize('H', WIDTHS)
def test_rollout_eval_bc_sweep_is_des_rollout_eval_bc_run_by_run(H, noiseless):
    ops, runs = _ops()
    R, reps, T = len(HP), 7, 120
    N = 1 if noiseless else 37
    theta = torch.from_numpy(np.stack([orc.synthetic_theta(3, H, 1, seed=H + r) for r in range(R)])).cuda()
    stats = torch.tensor([[0.1, -0.2, 0.3, 0.5, 0.4, 2.0, 1000.0], [0.0, 0.1, -0.1, 1.0, 0.9, 3.0, 50.0],
                          [0.2, 0.2, 0.2, 0.3, 0.3, 0.3, 7.0]], dtype=torch.float32).cuda()
    hp = runs.run_table([h[0] for h in HP], [h[1] for h in HP], 0.01, 0.005, [h[2] for h in HP], 'cuda')
    state = ops.new_state('cuda', 4)
    kw = dict(hidden=H, horizon=T, repetitions=reps, clip=2.0, state=state, run_size=N, noiseless=noiseless,
              obs_stats=stats)
    outs = []
    for bc in (None, torch.full((R, N, 3), np.nan, device='cuda')):
        fit, ep = torch.empty((R, N), device='cuda'), torch.empty((R, N, reps), device='cuda')
        tot = None if noiseless else torch.empty((R, 7), dtype=torch.float64, device='cuda')
        if bc is None:
            runs.rollout_eval_sweep(theta, hp, out=fit, episodes_out=ep, totals_out=tot, **kw)
        else:
            runs.rollout_eval_bc_sweep(theta, hp, out=fit, episodes_out=ep, totals_out=tot, bc_out=bc, **kw)
        outs.append((fit, ep, tot, bc))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert x is None and y is None or _bytes(x) == _bytes(y)
    for r, (seed, sigma, noise) in enumerate(HP):
        fit, ep, bc = torch.empty(N, device='cuda'), torch.empty((N, reps), device='cuda'), torch.empty((N, 3), device='cuda')
        tot = None if noiseless else torch.empty(7, dtype=torch.float64, device='cuda')
        ops.rollout_eval_bc(theta[r], hidden=H, horizon=T, repetitions=reps, sigma=0.0 if noiseless else sigma, clip=2.0,
                            action_noise_std=noise, seed=seed, state=state, member_offset=0, n_local=N,
                            noiseless=noiseless, obs_stats=stats[r], totals_out=tot, out=fit, episodes_out=ep, bc_out=bc)
        got = outs[1]
        assert _bytes(got[0][r]) == _bytes(fit) and _bytes(got[1][r]) == _bytes(ep), r
        assert _bytes(got[3][r]) == _bytes(bc) and bool(torch.isfinite(bc).all()), r
        if tot is not None:
            assert _bytes(got[2][r]) == _bytes(tot), r


def _archives(rs, R, A, d, capacity, integer):
    rows = (lambda n: _integer_rows(rs, n, d)) if integer else (lambda n: rs.randn(n, d).astype(np.float32))
    arch = np.full((R, capacity, d), np.nan, dtype=np.float32)          # rows past A: never read
    for r in range(R):
        arch[r, :A] = rows(A)
        if integer:
            arch[r, :A][rs.rand(A) < 0.05, rs.randint(d)] = np.nan
    return arch


def _check_novelty_runs(q, arch, A, k):
    ops, runs = _ops()
    qd, ad = torch.from_numpy(q).cuda(), torch.from_numpy(arch).cuda()
    got = runs.novelty_runs(qd, ad, k, size=A).cpu().numpy()
    for r in range(q.shape[0]):
        want = ops.novelty(qd[r], ad[r, :A].contiguous(), k).cpu().numpy()
        _same(got[r], want)


@pytest.mark.parametrize('n,A,d,k', CASES)
def test_novelty_runs_on_integer_behaviours_is_des_novelty_run_by_run(n, A, d, k):
    rs = np.random.RandomState(n + A + d + k)
    n, R = min(n, 2048), 3
    q = np.stack([_integer_rows(rs, n, d) for _ in range(R)])
    if n > 1:
        q[:, rs.rand(n) < 0.05, 0] = np.nan
    arch = _archives(rs, R, A, d, A + 37, True)
    _check_novelty_runs(q, arch, A, k)


@pytest.mark.parametrize('n,A,d,k', [(64, 500, 24, 10), (33, 300, 3, 32), (7, 1000, 32, 1), (64, 3, 3, 10),
                                     (64, 257, 3, 10)])
def test_novelty_runs_on_real_behaviours_is_des_novelty_run_by_run(n, A, d, k):
    rs = np.random.RandomState(n + A)
    R = 4
    q = rs.randn(R, n, d).astype(np.float32)
    _check_novelty_runs(q, _archives(rs, R, A, d, 2 * A, False), A, k)


@pytest.mark.parametrize('R,n', [(300, 64), (5, 2048), (1000, 2)])
def test_novelty_runs_where_each_run_spans_many_ctas(R, n):
    rs = np.random.RandomState(R)
    q = rs.randn(R, n, 3).astype(np.float32)
    _check_novelty_runs(q, _archives(rs, R, 70, 3, 128, False), 70, 10)


def test_novelty_runs_limits():
    _, runs = _ops()
    q, a = torch.zeros((2, 2049, 3), device='cuda'), torch.zeros((2, 8, 3), device='cuda')
    with pytest.raises(RuntimeError, match='run_size 2049 > 2048'):
        runs.novelty_runs(q, a, 3, size=8)
    with pytest.raises(RuntimeError, match='capacity'):
        runs.novelty_runs(q[:, :4].contiguous(), a, 3, size=9)
    out = torch.full((0, 4), 1.0, device='cuda')
    runs.novelty_runs(torch.zeros((0, 4, 3), device='cuda'), torch.zeros((0, 8, 3), device='cuda'), 3, size=8, out=out)


@pytest.mark.parametrize('N', [2, 64, 2048])
def test_ns_shape_runs_is_des_ns_shape_run_by_run(N):
    ops, runs = _ops()
    rs = np.random.RandomState(N)
    W = (0.0, 0.3, 1.0, 0.5, 0.05)
    R = len(W)
    f = np.round(rs.randn(R, N), 1).astype(np.float32)                 # ties
    f[rs.rand(R, N) < 0.01] = np.nan
    nov = np.abs(np.round(rs.randn(R, N), 2)).astype(np.float32)
    fd, nd = torch.from_numpy(f).cuda(), torch.from_numpy(nov).cuda()
    got = runs.ns_shape_runs(fd, nd, runs.ns_weight_table(W, 'cuda'))
    for r, w in enumerate(W):
        assert _bytes(got[r]) == _bytes(ops.ns_shape(fd[r], nd[r], w)), (r, w)
    ones = runs.ns_shape_runs(fd, nd, runs.ns_weight_table([1.0] * R, 'cuda'))
    assert _bytes(ones) == _bytes(runs.centered_rank_runs(fd))


def _closed(seed, sigma, lr, noise, w, x0):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(32)
    c.pop_size, c.max_generations = 64, 4
    c.seed, c.sigma, c.learning_rate, c.action_noise_std = seed, sigma, lr, noise
    c.initial_weight = np.asarray(orc.synthetic_theta(3, 32, 1, seed=x0), dtype=np.float32)
    c.ns_reward_weight = w
    return c


def _host(seed, sigma, lr, noise, w, x0, horizon=40):
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=16, clip=2.0, batch_env_fn=lambda B: po.PendulumBatch(B, seed, horizon))
    c.pop_size, c.max_steps, c.seed, c.sigma, c.learning_rate = 16, 3000, seed, sigma, lr
    c.action_noise_std = noise
    c.repetitions = c.test_repetitions = 3
    c.initial_weight = np.asarray(orc.synthetic_theta(3, 16, 1, seed=x0), dtype=np.float32)
    c.ns_reward_weight = w
    return c


RUNS = ((3, 0.05, 0.05, 0.05, 0.5, 0), (4, 0.1, 0.02, 0.0, 'adaptive', 1), (3, 0.05, 0.05, 0.05, 0.0, 0),
        (9, 0.02, 0.1, 0.1, 1.0, 2))


def _assert_sweep_is_train(configs):
    from distributedes_b200 import novelty
    ns = novelty.build_sweep(configs)
    out = novelty.train_sweep(configs, ns)
    for r, c in enumerate(configs):
        one = novelty.build(c)
        single = novelty.train(c, one)
        e = one.agents[0]
        assert out[r][:2] == single[:2], r
        assert torch.equal(ns.theta(r), e.theta) and torch.equal(ns.adam_m(r), e.adam_m), r
        assert torch.equal(ns.obs_stats(r), e.obs_stats), r
        assert _bytes(ns.archive(r)) == _bytes(one.archive) and ns.weights[r] == one.weights, r
        assert ns.best[r] == one.best and ns.best_theta[r].tobytes() == one.best_theta.tobytes(), r
    return out, ns


def test_closed_loop_train_sweep_is_sequential_train():
    out, ns = _assert_sweep_is_train([_closed(*h) for h in RUNS])
    assert ns.archive(0).shape == (5, 3) and out[0][0] != out[2][0]


def test_host_stepped_train_sweep_is_sequential_train():
    out, _ = _assert_sweep_is_train([_host(*h, horizon=hz) for h, hz in zip(RUNS, (40, 60, 40, 90))])
    assert len({len(run[0]) for run in out}) > 1                       # the runs stop at different generations


@pytest.mark.parametrize('make', [_closed, _host], ids=['closed', 'host'])
def test_every_weight_1_is_natural_es_train_sweep(make):
    from distributedes_b200 import natural_es, novelty
    configs = [make(*h[:4], 1.0, h[5]) for h in RUNS]
    ns = novelty.build_sweep(configs)
    out = novelty.train_sweep(configs, ns)
    engine = natural_es.build_sweep_engine(configs)
    want = natural_es.train_sweep(configs, engine)
    for r in range(len(configs)):
        assert out[r][:2] == want[r][:2], r
    if make is _closed:
        assert torch.equal(ns.engine.theta, engine.theta)
