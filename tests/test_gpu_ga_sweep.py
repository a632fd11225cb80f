"""Genetic-algorithm sweeps on the GPU, bit for bit against the single-run entry points and trainers:

  - des_rollout_eval_ga_sweep run r is des_rollout_eval_ga of its table, counts, seed, sigma and action noise at member
    offset 0, at every width, with statistics and action noise on (fitness, episode returns, totals), runs of different
    T and E and one run at generation 0 (a one-row table);
  - des_ga_rows_sweep is des_ga_rows per run, in rows mode and in gather mode (rows of -1 left as they were);
  - des_ga_order_runs is des_ga_order per run over ties, +-0, NaN and inf at N = 2, 64 and 2048, -1 past each T_r;
  - genetic.train_sweep run r is genetic.train(configs[r]): closed-loop at H = 16 and 64, host-stepped SynthWalk with
    runs stopping at different generations, and multi_runs batched against sequential.
"""
import copy
import pickle

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc  # noqa: E402
from oracle import synth_walk as sw  # noqa: E402

pytestmark = pytest.mark.gpu
WIDTHS = (16, 32, 64, 96, 128)
# seed, sigma, action noise, n_parents, n_elites, truncation of each run; run 2 is at generation 0 (one-row table)
RUNS = ((21, 0.04, 0.2, 4, 2, 4), (2**40 + 5, 0.1, 0.0, 3, 0, 3), (7, 0.05, 0.1, 1, 1, 4), (21, 0.04, 0.2, 4, 2, 4))


def _ops():
    from distributedes_b200 import ops, ops_runs
    return ops, ops_runs


def _tables(H, rows=4, seed=0):
    P = orc.param_count(3, H, 1)
    rng = np.random.default_rng(seed)
    t = torch.from_numpy(rng.standard_normal((len(RUNS), rows, P)).astype(np.float32) * 0.3).cuda()
    t[3] = t[0]                                   # run 3 repeats run 0
    return t


def _hp_ga(ops_runs, rows=4):
    hp = ops_runs.run_table([r[0] for r in RUNS], [r[1] for r in RUNS], 0.0, 0.0, [r[2] for r in RUNS], 'cuda')
    ga = ops_runs.ga_table([r[3] for r in RUNS], [r[4] for r in RUNS], [r[5] for r in RUNS], rows, 'cuda')
    return hp, ga


def _stats():
    s = torch.tensor([0.1, -0.2, 0.3, 0.5, 0.6, 2.0, 50.0], dtype=torch.float32, device='cuda')
    return torch.stack([s, s * 0, s * 1.5, s])


@pytest.mark.parametrize('H', WIDTHS)
def test_rollout_eval_ga_sweep_is_rollout_eval_ga_per_run(H):
    ops, ops_runs = _ops()
    parents, (hp, ga) = _tables(H, seed=H), _hp_ga(ops_runs)
    R, N, reps = len(RUNS), 37, 3
    stats = _stats()
    env = dict(hidden=H, horizon=40, repetitions=reps, clip=2.0, generation=6)
    f, ep = torch.empty((R, N), device='cuda'), torch.empty((R, N, reps), device='cuda')
    tot = torch.empty((R, 7), dtype=torch.float64, device='cuda')
    ops_runs.rollout_eval_ga_sweep(parents, ga, hp, run_size=N, obs_stats=stats, out=f, episodes_out=ep, totals_out=tot,
                                   **env)
    for r, (seed, sigma, noise, T, E, _) in enumerate(RUNS):
        f1, ep1 = torch.empty(N, device='cuda'), torch.empty(N * reps, device='cuda')
        tot1 = torch.empty(7, dtype=torch.float64, device='cuda')
        ops.rollout_eval_ga(parents[r, :T].contiguous(), E, sigma=sigma, action_noise_std=noise, seed=seed,
                            member_offset=0, n_local=N, obs_stats=stats[r].contiguous(), out=f1, episodes_out=ep1,
                            totals_out=tot1, **env)
        assert torch.equal(f[r], f1) and torch.equal(ep[r].reshape(-1), ep1) and torch.equal(tot[r], tot1), r
    assert torch.equal(f[0], f[3])


def test_ga_rows_sweep_is_ga_rows_per_run_in_both_modes():
    ops, ops_runs = _ops()
    parents, (hp, ga) = _tables(32, seed=1), _hp_ga(ops_runs)
    N = 50
    rows = ops_runs.ga_rows_sweep(parents, ga, hp, generation=4, run_size=N)
    members = torch.tensor([[17, 0, 49, 3], [5, 5, -1, -1], [1, 0, 2, 3], [-1, -1, -1, -1]], dtype=torch.int32,
                           device='cuda')
    out = torch.full_like(parents, 7.0)
    ops_runs.ga_rows_sweep(parents, ga, hp, generation=4, run_size=N, members=members, out=out)
    for r, (seed, sigma, _, T, E, _) in enumerate(RUNS):
        want = ops.ga_rows(parents[r, :T].contiguous(), E, sigma=sigma, seed=seed, generation=4, n_local=N)
        assert torch.equal(rows[r * N:(r + 1) * N], want), r
        for k in range(4):
            m = int(members[r, k])
            assert torch.equal(out[r, k], want[m] if m >= 0 else torch.full_like(out[r, k], 7.0)), (r, k)


@pytest.mark.parametrize('N', (2, 64, 2048))
def test_ga_order_runs_is_ga_order_per_run(N):
    ops, ops_runs = _ops()
    rng = np.random.default_rng(N)
    R = 5
    f = rng.integers(-3, 4, size=(R, N)).astype(np.float32)           # ties
    specials = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, np.nan], dtype=np.float32)
    for r in range(R):
        at = rng.choice(N, size=min(N, len(specials)), replace=False)
        f[r, at] = specials[:len(at)]
    T = [1, N, max(1, N // 5), min(2, N), max(1, N // 2)]
    rows = max(T)
    ga = ops_runs.ga_table([1] * R, [0] * R, T, rows, 'cuda')
    fit = torch.from_numpy(f).cuda()
    order = ops_runs.ga_order_runs(fit, ga, rows)
    for r in range(R):
        want = ops.ga_order(fit[r].contiguous(), T[r])
        assert torch.equal(order[r, :T[r]], want), r
        assert bool((order[r, T[r]:] == -1).all()), r


# ---- train_sweep against train ---------------------------------------------------------------------------------------
TRAIN_RUNS = ((0, 0.05, 0.0, 0, 13, 2), (3, 0.1, 0.2, 1, 6, 0), (11, 0.02, 0.1, 2, 20, 20))


def _closed(H, seed, sigma, noise, x0, T, E):
    from distributedes_b200 import config as cfg
    c = cfg.ClosedLoopPendulumConfig(H)
    c.pop_size, c.repetitions, c.test_repetitions, c.max_generations = 64, 3, 4, 3
    c.seed, c.sigma, c.action_noise_std, c.truncation, c.elites = seed, sigma, noise, T, E
    c.initial_weight = np.asarray(orc.synthetic_theta(3, H, 1, seed=x0), dtype=np.float32)
    return c


def _walk(seed, sigma, noise, x0, T, E):
    from distributedes_b200 import config as cfg
    c = cfg.HostEnvConfig(sw.SynthWalkEnv, 16, task='SynthWalk-v0')
    c.pop_size, c.repetitions, c.test_repetitions = 5, 2, 2
    c.seed, c.sigma, c.action_noise_std, c.truncation = seed, sigma, noise, 1 + T % 5
    c.elites = min(E, c.truncation)
    c.max_steps = 900
    c.initial_weight = np.asarray(orc.synthetic_theta(24, 16, 4, seed=x0), dtype=np.float32)
    return c


def _assert_runs_are_train(configs, out, worker, ga):
    from distributedes_b200 import genetic
    for r, c in enumerate(configs):
        w1, ga1 = genetic.build(c)
        single = genetic.train(c, w1, ga1)
        assert out[r][:2] == single[:2], r
        assert torch.equal(ga.parents[r], ga1.parents) and torch.equal(ga.order[r], ga1.order), r
        if w1.obs_stats is not None:
            assert torch.equal(worker.obs_stats[r], w1.obs_stats), r


@pytest.mark.parametrize('H', (16, 64))
def test_closed_loop_train_sweep_run_r_is_train(H):
    from distributedes_b200 import genetic
    configs = [_closed(H, *h) for h in TRAIN_RUNS]
    worker, ga = genetic.build_sweep(configs)
    out = genetic.train_sweep(configs, worker, ga)
    _assert_runs_are_train(configs, out, worker, ga)


def test_host_stepped_train_sweep_run_r_is_train_and_stops_where_it_does():
    from distributedes_b200 import genetic
    configs = [_walk(*h) for h in TRAIN_RUNS]
    worker, ga = genetic.build_sweep(configs)
    out = genetic.train_sweep(configs, worker, ga)
    assert len({len(run[0]) for run in out}) > 1
    _assert_runs_are_train(configs, out, worker, ga)


def test_multi_runs_batched_writes_the_rewards_and_steps_of_the_sequential_runs(tmp_path):
    from distributedes_b200 import genetic
    config = copy.copy(_closed(16, *TRAIN_RUNS[1]))
    config.max_generations, config.tag = 2, 'ga'
    out = {}
    for batched in (False, True):
        d = tmp_path / str(batched)
        genetic.multi_runs(config, runs=3, log_dir=str(d / 'log'), data_dir=str(d / 'data'), batched=batched)
        with open(d / 'data' / 'ga-stats-Pendulum-v0.bin', 'rb') as f:
            out[batched] = pickle.load(f)
    assert len(out[True]) == len(out[False]) == 3
    for a, b in zip(out[False], out[True]):
        assert a[:2] == b[:2]
    assert out[False][0][0] != out[False][1][0]
