"""The genetic algorithm on the GPU, bit for bit against entry points that already exist:

  - des_ga_rows with a one-row table and no elites is des_nes_perturb; with a larger table, row i is
    des_nes_perturb(parents[p_i]) at member i, p_i the oracle's parent draw, and an elite's row is its parent row;
  - des_rollout_eval_ga is des_rollout_eval_solutions on des_ga_rows' rows at every width (member_offset != 0, action
    noise and statistics on: fitness, episode returns, totals), and with a one-row table and no elites des_rollout_eval;
  - des_ga_order is a stable numpy argsort of -f with NaN last, over ties, +-0 and NaN, on both rank paths;
  - genetic.train on the closed loop: the fused path equals the materialised rows, run to run; its orders and tables
    equal the oracle's chain fed the GPU's fitness; host-stepped SynthWalk and the tape train end to end.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import ga_oracle as gao
from oracle import nes_oracle as orc
from oracle.synth_walk import SynthWalkEnv

pytestmark = pytest.mark.gpu
WIDTHS = (16, 32, 64, 96, 128)


def _ops():
    from distributedes_b200 import ops
    return ops


def _table(n, H, seed=0):
    P = orc.param_count(3, H, 1)
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.standard_normal((n, P)).astype(np.float32) * 0.3).cuda()


def test_one_row_without_elites_is_des_nes_perturb():
    ops = _ops()
    theta = _table(1, 64)
    rows = ops.ga_rows(theta, 0, sigma=0.07, seed=13, generation=5, member_offset=3, n_local=300)
    want = ops.nes_perturb(theta.reshape(-1), 300, 0.07, 13, 5, member_offset=3)
    assert torch.equal(rows, want)


@pytest.mark.parametrize('T,E', [(5, 0), (5, 2), (13, 13)])
def test_rows_are_their_parents_perturbation(T, E):
    ops = _ops()
    parents, N = _table(T, 32, seed=T), 40
    rows = ops.ga_rows(parents, E, sigma=0.05, seed=7, generation=3, n_local=N)
    p = gao.parents_of(7, 3, np.arange(N), T, E)
    for m in range(N):
        want = parents[m] if m < E else ops.nes_perturb(parents[p[m]], 1, 0.05, 7, 3, member_offset=m)[0]
        assert torch.equal(rows[m], want), m
    members = torch.tensor([17, 0, 39, 1, 17], dtype=torch.int32, device='cuda')
    gathered = ops.ga_rows(parents, E, sigma=0.05, seed=7, generation=3, members=members)
    assert torch.equal(gathered, rows[members.long()])


def _stats():
    return torch.tensor([0.1, -0.2, 0.3, 0.5, 0.6, 2.0, 50.0], dtype=torch.float32, device='cuda')


@pytest.mark.parametrize('H', WIDTHS)
def test_rollout_eval_ga_is_rollout_eval_solutions_on_the_rows(H):
    ops = _ops()
    parents, off, n, reps = _table(4, H, seed=H), 1, 37, 3
    env = dict(hidden=H, horizon=40, repetitions=reps, clip=2.0, action_noise_std=0.2, seed=21, generation=6,
               member_offset=off, obs_stats=_stats())
    f, ep, tot = (torch.empty(n, device='cuda'), torch.empty(n * reps, device='cuda'),
                  torch.empty(7, dtype=torch.float64, device='cuda'))
    ops.rollout_eval_ga(parents, 2, sigma=0.04, n_local=n, out=f, episodes_out=ep, totals_out=tot, **env)
    rows = ops.ga_rows(parents, 2, sigma=0.04, seed=21, generation=6, member_offset=off, n_local=n)
    f2, ep2, tot2 = torch.empty_like(f), torch.empty_like(ep), torch.empty_like(tot)
    ops.rollout_eval_solutions(rows, out=f2, episodes_out=ep2, totals_out=tot2, **env)
    assert torch.equal(f, f2) and torch.equal(ep, ep2) and torch.equal(tot, tot2)


@pytest.mark.parametrize('H', (16, 64))
def test_one_row_without_elites_is_des_rollout_eval(H):
    ops = _ops()
    theta = _table(1, H, seed=3)
    env = dict(hidden=H, horizon=60, repetitions=10, sigma=0.05, clip=2.0, action_noise_std=0.1, seed=4, generation=2,
               member_offset=5, n_local=64, obs_stats=_stats())
    assert torch.equal(ops.rollout_eval_ga(theta, 0, **env), ops.rollout_eval(theta.reshape(-1), **env))


@pytest.mark.parametrize('N', [2, 2048, 2049, 65536])
def test_ga_order_is_a_stable_descending_argsort(N):
    ops = _ops()
    rng = np.random.default_rng(N)
    f = rng.integers(-20, 20, N).astype(np.float32)         # many ties
    f[rng.random(N) < 0.1] = 0.0
    f[rng.random(N) < 0.1] = -0.0
    if N > 2:
        f[rng.random(N) < 0.05] = np.nan
        f[rng.random(N) < 0.01] = np.inf
    for T in sorted({1, max(1, N // 5), N}):
        got = ops.ga_order(torch.from_numpy(f).cuda(), T).cpu().numpy()
        assert got.tolist() == gao.order(f, T).tolist(), (N, T)


def _closed(gens=4, seed=3):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(16)
    c.pop_size, c.max_generations, c.seed, c.sigma, c.action_noise_std = 64, gens, seed, 0.1, 0.05
    return c


def _train(c, fused):
    from distributedes_b200 import genetic
    worker, ga = genetic.build(c, fused=fused)
    out = genetic.train(c, worker, ga)
    return out, ga, worker


def test_closed_loop_fused_equals_rows_and_reproduces():
    c = _closed()
    (r1, s1, _), ga1, w1 = _train(c, True)
    (r2, s2, _), ga2, w2 = _train(c, False)
    (r3, s3, _), ga3, _ = _train(c, True)
    assert r1 == r2 == r3 and s1 == s2 == s3 and len(r1) == c.max_generations + 1
    assert torch.equal(ga1.parents, ga2.parents) and torch.equal(ga1.parents, ga3.parents)
    assert torch.equal(w1.obs_stats, w2.obs_stats)


def test_orders_and_tables_are_the_oracle_chain_fed_the_gpu_fitness():
    from distributedes_b200 import genetic
    c = _closed()
    worker, ga = genetic.build(c)
    ops = _ops()
    for g in range(4):
        prev, E = ga.parents.clone(), ga.n_elites
        f = worker.run(ga).clone()
        worker.merge_obs_stats(ga.N)
        want = gao.order(f.cpu().numpy(), ga.T)
        ga.tell(f)
        assert ga.order.cpu().numpy().tolist() == want.tolist()
        p = gao.parents_of(c.seed, g, want, prev.shape[0], E)
        for k, m in enumerate(want):
            row = prev[m] if m < E else ops.nes_perturb(prev[p[k]], 1, c.sigma, c.seed, g, member_offset=int(m))[0]
            assert torch.equal(ga.parents[k], row), (g, k)


def test_host_stepped_and_tape_train_end_to_end():
    from distributedes_b200 import genetic
    from distributedes_b200.config import HostEnvConfig, PendulumConfig
    h = HostEnvConfig(SynthWalkEnv, hidden_size=16)
    h.pop_size, h.max_generations, h.repetitions, h.test_repetitions = 12, 3, 2, 2
    t = PendulumConfig(16, tape_len=32)
    t.pop_size, t.max_generations = 20, 3
    for c in (h, t):
        rewards, steps, stamps = genetic.train(c)
        assert len(rewards) == len(steps) == len(stamps) == 4 and np.all(np.isfinite(rewards))
        assert steps[0] == 0 and all(b > a for a, b in zip(steps, steps[1:]))


def test_record_returns_are_the_test_returns():
    from distributedes_b200 import genetic
    c = _closed()
    sol = c.initial_weight
    tr = genetic.record(c, sol, None)
    mean, _ = genetic.test(c, sol, None)
    assert tr.returns.shape == (c.test_repetitions,)
    assert np.mean(tr.returns.astype(np.float64)) == mean
