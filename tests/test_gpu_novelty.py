"""Novelty search on the GPU:

  - des_novelty on integer-valued behaviours, where every fp32 operation of the contract is exact and ties are common,
    equals the oracle bit for bit over n, A, d and k, with NaN archive rows and NaN queries;
  - des_novelty on real-valued behaviours equals the oracle's fp32 restatement bit for bit, and lies within (d + 8) fp32
    ulps of the exact fp64 novelty;
  - des_rollout_eval_bc's fitness, episode returns and totals are des_rollout_eval's bit for bit at every width, members
    and test episodes, statistics on; its behaviour is the mean of the observations a recording of one more step
    writes at that step, bit for bit, and numpy's cos / sin of the recorded final state within one fp32 ulp;
  - des_ns_shape at w = 1 is des_centered_rank bit for bit, and the oracle's blend at w = 0, 0.3 and 0.5 on both rank
    paths;
  - novelty.train with one agent at w = 1 is natural_es.train bit for bit, closed-loop and host-stepped; NSR-ES with three
    agents runs and archives one behaviour per generation after the three start points.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from host_env_support import PendulumProbe
from oracle import nes_oracle as orc
from oracle import novelty_oracle as no
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu
WIDTHS = (16, 32, 64, 96, 128)


def _ops():
    from distributedes_b200 import ops
    return ops


def _integer_rows(rs, n, d):
    return rs.randint(-8, 9, size=(n, d)).astype(np.float32)      # |diff| <= 16: d2 <= 32 * 256 < 2^24


CASES = [(1, 1, 3, 10), (1, 100000, 3, 1), (64, 5, 1, 10), (64, 10, 3, 10), (64, 10, 24, 32), (64, 100000, 32, 32),
         (64, 4097, 24, 10), (4096, 4097, 32, 32), (4096, 10, 3, 1), (4096, 100000, 3, 10), (4096, 5, 24, 32),
         (1, 4097, 32, 1)]


@pytest.mark.parametrize('n,A,d,k', CASES)
def test_novelty_on_integer_behaviours_is_the_oracle_s_bit_for_bit(n, A, d, k):
    rs = np.random.RandomState(n + A + d + k)
    q, a = _integer_rows(rs, n, d), _integer_rows(rs, A, d)
    a[rs.rand(A) < 0.05, rs.randint(d)] = np.nan
    if n > 1:
        q[rs.rand(n) < 0.05, 0] = np.nan
    got = _ops().novelty(torch.from_numpy(q).cuda(), torch.from_numpy(a).cuda(), k).cpu().numpy()
    want = no.novelty_integer(q, a, k)
    _same(got, want)


def _same(got, want):
    """Bit for bit, except that a NaN is any NaN: the device's is 0x7fffffff, numpy's 0x7fc00000."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert got[~nan].tobytes() == want[~nan].tobytes()


def test_novelty_on_real_behaviours():
    rs = np.random.RandomState(1)
    ops = _ops()
    for n, A, d, k in ((64, 500, 24, 10), (33, 300, 3, 32), (7, 1000, 32, 1)):
        q, a = rs.randn(n, d).astype(np.float32), rs.randn(A, d).astype(np.float32)
        got = ops.novelty(torch.from_numpy(q).cuda(), torch.from_numpy(a).cuda(), k).cpu().numpy()
        assert got.tobytes() == no.novelty_fp32(q, a, k).tobytes()
        # Against exact distances: the d squares, d sums and d differences of d2 round at most ~(d + 2) u relatively
        # (all terms are non-negative), the sqrt halves that and rounds once more, the fp64 mean adds nothing visible and
        # the final fp32 store rounds once: (d + 8) u with u = 2^-24 bounds it.  Swapped near-ties change the sum of
        # the k smallest by no more than the distances themselves move.
        np.testing.assert_allclose(got, no.novelty(q, a, k), rtol=(d + 8) * 2.0 ** -24, atol=0)


def _bc_case(H, noiseless):
    P = orc.param_count(3, H, 1)
    theta = torch.from_numpy(orc.synthetic_theta(3, H, 1, seed=H)).cuda()
    stats = torch.tensor([0.1, -0.2, 0.3, 0.5, 0.4, 2.0, 1000.0], dtype=torch.float32).cuda()
    n = 1 if noiseless else 37
    kw = dict(hidden=H, horizon=120, repetitions=7, sigma=0.0 if noiseless else 0.05, clip=2.0, action_noise_std=0.1,
              seed=11, generation=3, member_offset=0 if noiseless else 5, n_local=n, noiseless=noiseless,
              obs_stats=stats)
    return P, theta, n, kw


@pytest.mark.parametrize('noiseless', [False, True])
@pytest.mark.parametrize('H', WIDTHS)
def test_rollout_eval_bc_is_des_rollout_eval_and_its_behaviour_the_final_observation(H, noiseless):
    ops = _ops()
    P, theta, n, kw = _bc_case(H, noiseless)
    reps, T = kw['repetitions'], kw['horizon']
    outs = []
    for bc in (None, torch.full((n, 3), np.nan, device='cuda')):
        fit = torch.empty(n, device='cuda')
        ep = torch.empty((n, reps), device='cuda')
        tot = torch.empty(7, dtype=torch.float64, device='cuda')
        if bc is None:
            ops.rollout_eval(theta, out=fit, episodes_out=ep, totals_out=tot, **kw)
        else:
            ops.rollout_eval_bc(theta, out=fit, episodes_out=ep, totals_out=tot, bc_out=bc, **kw)
        outs.append((fit, ep, tot, bc))
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
    bc = outs[1][3].cpu().numpy()
    # one more step recorded: its observation at t = T is the state after step T - 1 of the T-step episodes
    rec = dict(kw, horizon=T + 1)
    steps = n * reps * (T + 1)
    states = torch.empty(steps * 2, dtype=torch.float64, device='cuda')
    obs = torch.empty(steps * 3, device='cuda')
    ops.rollout_record(theta, mirrored=False, states_out=states, obs_out=obs, actions_out=None, rewards_out=None,
                       **rec)
    final_obs = obs.cpu().numpy().reshape(n, reps, T + 1, 3)[:, :, T]
    assert bc.tobytes() == no.behaviours(final_obs, n, reps).tobytes()
    # numpy's cos and sin of the recorded fp64 state: the device's fp64 sincos may differ by an ulp, which the fp32
    # rounding of an observation in [-1, 1] turns into at most one fp32 ulp (2^-24 near 1), kept by the mean
    th = states.cpu().numpy().reshape(n, reps, T + 1, 2)[:, :, T]
    want = no.behaviours(po.pendulum_obs(th[..., 0], th[..., 1]).astype(np.float32), n, reps)
    np.testing.assert_allclose(bc[:, :2], want[:, :2], rtol=0, atol=2.0 ** -23)
    assert bc[:, 2].tobytes() == want[:, 2].tobytes()


@pytest.mark.parametrize('N', [64, 4096, 65536])
def test_ns_shape(N):
    ops = _ops()
    rs = np.random.RandomState(N)
    f = np.round(rs.randn(N), 1).astype(np.float32)                   # ties
    f[rs.rand(N) < 0.01] = np.nan
    nov = np.abs(np.round(rs.randn(N), 2)).astype(np.float32)
    fd, nd = torch.from_numpy(f).cuda(), torch.from_numpy(nov).cuda()
    ranked = ops.centered_rank(fd)
    assert ops.ns_shape(fd, nd, 1.0).cpu().numpy().tobytes() == ranked.cpu().numpy().tobytes()
    for w in (0.0, 0.3, 0.5):
        got = ops.ns_shape(fd, nd, w).cpu().numpy()
        assert got.tobytes() == no.blend(f, nov, w).tobytes(), w


def _closed(M=1, w=1.0, gens=3):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(32)
    c.pop_size, c.max_generations, c.seed, c.sigma, c.learning_rate = 64, gens, 3, 0.05, 0.05
    c.action_noise_std = 0.05
    c.ns_agents, c.ns_reward_weight = M, w
    return c


def _host():
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=16, clip=2.0, batch_env_fn=lambda B: po.PendulumBatch(B, 3, 40))
    c.pop_size, c.max_generations, c.seed, c.sigma, c.learning_rate = 16, 2, 3, 0.05, 0.05
    c.repetitions = c.test_repetitions = 3
    c.ns_reward_weight = 1.0
    return c


@pytest.mark.parametrize('make', [_closed, _host], ids=['closed', 'host'])
def test_one_agent_at_weight_1_trains_as_natural_es(make):
    from distributedes_b200 import natural_es, novelty
    c = make()
    engine = natural_es.build_engine(c)
    want = natural_es.train(c, engine)
    ns = novelty.build(c)
    got = novelty.train(c, ns)
    assert got[0] == want[0] and got[1] == want[1]
    assert torch.equal(ns.agents[0].theta, engine.theta)


def test_nsr_es_with_three_agents_runs():
    from distributedes_b200 import novelty
    c = _closed(M=3, w=0.5, gens=4)
    ns = novelty.build(c)
    rewards, steps, _ = novelty.train(c, ns)
    assert len(rewards) == 5 and steps == [64 * 10 * 200 * g for g in range(5)]
    assert ns.archive.shape == (3 + 4, 3) and bool(torch.isfinite(ns.archive).all())
    assert all(0 <= m < 3 for m in ns.selected) and len(ns.selected) == 5
    assert ns.weights == [0.5] * 4
    assert np.all(np.isfinite(rewards))
