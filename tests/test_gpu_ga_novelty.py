"""The genetic algorithm's novelty search on the GPU:

  - des_rollout_eval_ga_bc's fitness, episode returns and totals are des_rollout_eval_ga's bit for bit at every width,
    with elites and children, statistics and action noise on; its behaviour is the mean of the observations a recording
    of des_ga_rows' rows, one step longer, writes at that step, bit for bit, and numpy's cos / sin of the recorded final
    state within one fp32 ulp;
  - des_ns_ga_order is tests/ga_novelty_oracle.py's order bit for bit on both rank paths, with ties, NaN, +-0 and +-inf
    in both inputs, and at w = 1 it is des_ga_order;
  - novelty.train_ga at w = 1 is genetic.train bit for bit, closed-loop and host-stepped (rewards, steps, final table,
    order, statistics);
  - GA-NSR and GA-NSRA run: each generation's novelty and order equal the oracle's fed the GPU's own fitness,
    behaviours and archive, the weights follow the NSRA-ES schedule of the GPU's test means, and the archive grows by
    one row per generation.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

import ga_novelty_oracle as gno  # noqa: E402
from host_env_support import PendulumProbe  # noqa: E402
from oracle import ga_oracle as gao  # noqa: E402
from oracle import nes_oracle as orc  # noqa: E402
from oracle import novelty_oracle as no  # noqa: E402
from oracle import pendulum_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu
WIDTHS = (16, 32, 64, 96, 128)


def _ops():
    from distributedes_b200 import ops
    return ops


def _table(n, H, seed=0):
    P = orc.param_count(3, H, 1)
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.standard_normal((n, P)).astype(np.float32) * 0.3).cuda()


def _stats():
    return torch.tensor([0.1, -0.2, 0.3, 0.5, 0.6, 2.0, 50.0], dtype=torch.float32, device='cuda')


@pytest.mark.parametrize('H', WIDTHS)
def test_rollout_eval_ga_bc_is_rollout_eval_ga_and_its_behaviour_the_final_observation(H):
    ops = _ops()
    parents, E, off, n, reps, T = _table(4, H, seed=H), 2, 1, 37, 7, 120
    env = dict(hidden=H, horizon=T, repetitions=reps, clip=2.0, action_noise_std=0.2, seed=21, generation=6,
               member_offset=off, obs_stats=_stats())
    outs = []
    for bc in (None, torch.full((n, 3), np.nan, device='cuda')):
        f, ep, tot = (torch.empty(n, device='cuda'), torch.empty(n * reps, device='cuda'),
                      torch.empty(7, dtype=torch.float64, device='cuda'))
        if bc is None:
            ops.rollout_eval_ga(parents, E, sigma=0.04, n_local=n, out=f, episodes_out=ep, totals_out=tot, **env)
        else:
            ops.rollout_eval_ga_bc(parents, E, sigma=0.04, n_local=n, out=f, episodes_out=ep, totals_out=tot, bc_out=bc,
                                   **env)
        outs.append((f, ep, tot, bc))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
    bc = outs[1][3].cpu().numpy()
    assert bool(np.isfinite(bc).all())
    # des_ga_rows' rows recorded one step longer: the observation at t = T is the state after step T - 1
    rows = ops.ga_rows(parents, E, sigma=0.04, seed=21, generation=6, member_offset=off, n_local=n)
    steps = n * reps * (T + 1)
    states = torch.empty(steps * 2, dtype=torch.float64, device='cuda')
    obs = torch.empty(steps * 3, device='cuda')
    ops.rollout_record_solutions(rows, states_out=states, obs_out=obs, **dict(env, horizon=T + 1))
    final_obs = obs.cpu().numpy().reshape(n, reps, T + 1, 3)[:, :, T]
    assert bc.tobytes() == no.behaviours(final_obs, n, reps).tobytes()
    # numpy's cos and sin of the recorded fp64 state: at most one fp32 ulp apart (test_gpu_novelty's argument)
    th = states.cpu().numpy().reshape(n, reps, T + 1, 2)[:, :, T]
    want = no.behaviours(po.pendulum_obs(th[..., 0], th[..., 1]).astype(np.float32), n, reps)
    np.testing.assert_allclose(bc[:, :2], want[:, :2], rtol=0, atol=2.0 ** -23)
    assert bc[:, 2].tobytes() == want[:, 2].tobytes()


def _inputs(N, rng):
    """fitness and novelty [N] fp32 with ties, +-0, NaN and +-inf."""
    f = rng.integers(-20, 20, N).astype(np.float32)
    nov = np.abs(rng.integers(0, 12, N)).astype(np.float32) / 4
    for x in (f, nov):
        x[rng.random(N) < 0.1] = 0.0
        x[rng.random(N) < 0.1] = -0.0
        if N > 2:
            x[rng.random(N) < 0.05] = np.nan
            x[rng.random(N) < 0.01] = np.inf
            x[rng.random(N) < 0.01] = -np.inf
    if N == 2:
        f[:], nov[:] = (np.nan, 1.0), (-0.0, np.inf)
    return f, nov


@pytest.mark.parametrize('w', [0.0, 0.3, 0.5, 1.0])
@pytest.mark.parametrize('N', [2, 64, 2048, 2049, 65536])
def test_ns_ga_order_is_the_oracle_s(N, w):
    ops = _ops()
    f, nov = _inputs(N, np.random.default_rng(N))
    fd, nd = torch.from_numpy(f).cuda(), torch.from_numpy(nov).cuda()
    ws = ops.ns_ga_order_workspace(N, 'cuda')
    for T in sorted({1, -(-N // 5), N}):
        got = ops.ns_ga_order(fd, nd, w, T, workspace=ws).cpu().numpy()
        assert got.tolist() == gno.ns_ga_order(f, nov, w, T).tolist(), (N, T, w)
        if w == 1.0:
            assert got.tolist() == ops.ga_order(fd, T).cpu().numpy().tolist()
            assert got.tolist() == gao.order(f, T).tolist()


# ---- training ----------------------------------------------------------------------------------------------------------
def _closed(w=1.0, gens=4):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(16)
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = 64, 13, 2, gens, 3, 0.1
    c.action_noise_std = 0.05
    c.ns_reward_weight, c.ns_k = w, 10
    return c


def _host(w=1.0, gens=3):
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=16, clip=2.0, batch_env_fn=lambda B: po.PendulumBatch(B, 3, 40))
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = 16, 4, 1, gens, 3, 0.1
    c.repetitions = c.test_repetitions = 3
    c.ns_reward_weight, c.ns_k = w, 5
    return c


@pytest.mark.parametrize('make', [_closed, _host], ids=['closed', 'host'])
def test_train_ga_at_weight_1_is_genetic_train(make):
    from distributedes_b200 import genetic, novelty
    c = make()
    worker, ga = genetic.build(c)
    want = genetic.train(c, worker, ga)
    nsga = novelty.build_ga(c)
    got = novelty.train_ga(c, nsga)
    assert got[0] == want[0] and got[1] == want[1]
    assert torch.equal(nsga.ga.parents, ga.parents) and torch.equal(nsga.ga.order, ga.order)
    assert nsga.worker.obs_stats.cpu().numpy().tobytes() == worker.obs_stats.cpu().numpy().tobytes()
    assert nsga.archive.shape == (1 + c.max_generations, 3) and nsga.weights == [1.0] * c.max_generations


@pytest.mark.parametrize('make', [_closed, _host], ids=['closed', 'host'])
@pytest.mark.parametrize('w', [0.5, 'adaptive'])
def test_novelty_and_order_follow_the_oracle_fed_the_gpu_s_values(make, w):
    from distributedes_b200 import novelty
    c = make(w=w, gens=5)
    nsga = novelty.build_ga(c)
    seen, select = [], nsga.select

    def recorded(fitness):
        archive = nsga.archive.clone()
        order = select(fitness)
        seen.append((fitness.cpu().numpy().copy(), nsga.bc.cpu().numpy().copy(), archive.cpu().numpy(),
                     nsga.novelty.cpu().numpy().copy(), order.cpu().numpy().copy(), nsga.weights[-1]))
        return order
    nsga.select = recorded
    rewards, steps, _ = novelty.train_ga(c, nsga)
    assert len(seen) == c.max_generations and len(rewards) == c.max_generations + 1
    assert nsga.archive.shape == (1 + c.max_generations, 3) and bool(torch.isfinite(nsga.archive).all())
    wt, stall, best = (1.0 if w == 'adaptive' else w), 0, rewards[0]
    for g, (f, bc, archive, nov, order, weight) in enumerate(seen):
        assert archive.shape == (1 + g, 3)
        assert nov.tobytes() == no.novelty_fp32(bc, archive, c.ns_k).tobytes(), g
        assert weight == wt, g
        assert order.tolist() == gno.ns_ga_order(f, nov, weight, c.truncation).tolist(), g
        improved = bool(rewards[g + 1] > best)
        best = rewards[g + 1] if improved else best
        if w == 'adaptive':
            wt, stall = no.adapt(wt, stall, improved)
    assert nsga.weights == [s[5] for s in seen]
    assert np.all(np.isfinite(rewards)) and steps[0] == 0 and all(a < b for a, b in zip(steps, steps[1:]))
