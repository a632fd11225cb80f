"""des_policy_act (the population's policy step for environments stepped on the host) and the engine over it: the fp64
forward, the action-noise stream, dead slots, the statistics order, shard invariance and host-stepped Pendulum-v0
against the oracle.  natural_es.train and cma_es.train over host-stepped episodes meet the reference's goldens in
tests/test_gpu_goldens.py.

Tolerance of the actions: the fp32 forward differs from the fp64 one by fp32 rounding of the FMA chains plus the MUFU
tanh's ~2e-7 absolute error per unit; |W3| sums to O(1) for these weights, so |da| stays below ~1e-5 (3e-5 (1 + |a|) is
used).  Action noise adds the MUFU Box-Muller error, <= 4e-6 (1 + |z|) times the std."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

import host_env_support as hs
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu
RTOL = 2e-4


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


def _rows(d0, H, A, n, seed):
    theta = orc.synthetic_theta(d0, H, A, seed=seed)
    return orc.perturb(theta, 0.1, orc.noise(seed, 0, 0, n, theta.size))


def _stats(d0, rs):
    return (rs.randn(d0).astype(np.float32) * 0.3, (rs.rand(d0) + 0.5).astype(np.float32), np.float32(1000))


@pytest.mark.parametrize('H', [16, 32, 64, 96, 128])
@pytest.mark.parametrize('d0,A', [(3, 1), (8, 2), (24, 4), (32, 8)])
@pytest.mark.parametrize('reps', [1, 10, 16])
def test_policy_act_matches_fp64_forward(H, d0, A, reps):
    from distributedes_b200 import ops
    n, seed, gen, off = 7, 3 + H, 2, 5
    rs = np.random.RandomState(H * 100 + d0 * 10 + reps)
    rows = _rows(d0, H, A, n, seed)
    obs = (rs.randn(n, reps, d0) * 2).astype(np.float32)
    alive = rs.rand(n, reps) < 0.7
    alive[0] = True
    stats = _stats(d0, rs)
    for use_stats in (False, True):
        for noise in (0.0, 0.3):
            st = dev(np.concatenate([stats[0], stats[1], [stats[2]]])) if use_stats else None
            part = torch.zeros((n, 2 * d0 + 1), dtype=torch.float64, device='cuda')
            act = ops.policy_act(dev(rows), dev(obs), dev(alive, torch.uint8), state_dim=d0, hidden=H, action_dim=A,
                                 repetitions=reps, clip=1.5, action_noise_std=noise, seed=seed, generation=gen,
                                 member_offset=off, t=4, obs_stats=st, stat_part=part).cpu().numpy()
            ref = po.policy_actions(rows, obs, alive, d0, H, A, 1.5, stats if use_stats else None, noise, seed, gen, off,
                                    4)
            assert act.shape == (n, reps, A)
            assert np.all(act[~alive] == 0.0)
            assert np.max(np.abs(act - ref) / (1 + np.abs(ref))) < 3e-5, (use_stats, noise)
            want = np.zeros((n, 2 * d0 + 1))
            po.accumulate_stats(want, obs, alive)
            assert np.array_equal(part.cpu().numpy(), want)


def test_action_noise_is_the_counter_stream_and_statistics_accumulate_in_step_order():
    """Zero weights: the action is clip(std * z), z the documented counter normals (quads beyond the fourth action
    included); two launches accumulate the statistics in (step, repetition) order, bit for bit."""
    from distributedes_b200 import ops
    d0, H, A, reps, n = 5, 32, 8, 16, 3
    P = orc.param_count(d0, H, A)
    rows = dev(np.zeros((n, P)))
    rs = np.random.RandomState(1)
    part = torch.zeros((n, 2 * d0 + 1), dtype=torch.float64, device='cuda')
    want = np.zeros((n, 2 * d0 + 1))
    for t in (0, 7):
        obs = rs.randn(n, reps, d0).astype(np.float32)
        alive = rs.rand(n, reps) < 0.8
        act = ops.policy_act(rows, dev(obs), dev(alive, torch.uint8), state_dim=d0, hidden=H, action_dim=A,
                             repetitions=reps, clip=10.0, action_noise_std=1.0, seed=99, generation=6, member_offset=11,
                             t=t, stat_part=part).cpu().numpy()
        z = po.action_noise(99, 6, np.arange(11, 11 + n), reps, t, A)
        assert np.all(np.abs(act - z)[alive] <= 4e-6 * (1 + np.abs(z[alive])))
        assert np.all(act[~alive] == 0)
        po.accumulate_stats(want, obs, alive)
        assert np.array_equal(part.cpu().numpy(), want)
    tot = ops.obs_parts_reduce(part, d0).cpu().numpy()
    assert np.array_equal(tot, want[0] + want[1] + want[2])


def test_policy_act_is_shard_invariant():
    from distributedes_b200 import ops
    d0, H, A, reps, n = 24, 64, 4, 10, 9
    rows = dev(_rows(d0, H, A, n, 4))
    rs = np.random.RandomState(2)
    obs, alive = dev(rs.randn(n, reps, d0)), dev(rs.rand(n, reps) < 0.6, torch.uint8)
    st = dev(np.concatenate(list(_stats(d0, rs)[:2]) + [[50.0]]))
    kw = dict(state_dim=d0, hidden=H, action_dim=A, repetitions=reps, clip=1.0, action_noise_std=0.1, seed=3,
              generation=1, t=12, obs_stats=st)
    parts = [torch.zeros((k, 2 * d0 + 1), dtype=torch.float64, device='cuda') for k in (n, 4, n - 4)]
    whole = ops.policy_act(rows, obs, alive, member_offset=0, stat_part=parts[0], **kw)
    a = ops.policy_act(rows[:4].contiguous(), obs[:4].contiguous(), alive[:4].contiguous(), member_offset=0,
                       stat_part=parts[1], **kw)
    b = ops.policy_act(rows[4:].contiguous(), obs[4:].contiguous(), alive[4:].contiguous(), member_offset=4,
                       stat_part=parts[2], **kw)
    assert torch.equal(whole, torch.cat([a, b])) and torch.equal(parts[0], torch.cat(parts[1:]))


def test_policy_act_rejects_bad_arguments():
    from distributedes_b200 import ops
    rows = dev(np.zeros((2, orc.param_count(24, 64, 4))))
    obs, alive = dev(np.zeros((2, 17, 24))), dev(np.ones((2, 17)), torch.uint8)
    with pytest.raises(RuntimeError, match='repetitions must be in'):
        ops.policy_act(rows, obs, alive, state_dim=24, hidden=64, action_dim=4, repetitions=17, clip=1.0, seed=0,
                       generation=0, t=0)
    with pytest.raises(RuntimeError, match='MLP needs'):
        ops.policy_act(rows, obs[:, :2].contiguous(), alive[:, :2].contiguous(), state_dim=24, hidden=32, action_dim=4,
                       repetitions=2, clip=1.0, seed=0, generation=0, t=0)


# ---- host-stepped Pendulum-v0 against the device rollout's oracle ----------------------------------------------------
def _pendulum_engine(H, N, reps, seed, theta0, **kw):
    from distributedes_b200.engine import HostEnvEngine
    return HostEnvEngine(env_fn=hs.PendulumProbe, batch_env_fn=lambda B: po.PendulumBatch(B, seed), hidden=H, pop_size=N,
                         theta0=theta0, sigma=0.1, learning_rate=0.1, repetitions=reps, clip=2.0, seed=seed, **kw)


def test_host_stepped_pendulum_matches_the_rollout_oracle():
    H, N, reps, seed = 64, 12, 10, 4
    theta = orc.synthetic_theta(3, H, 1, seed=2)
    eng = _pendulum_engine(H, N, reps, seed, theta)
    stats = (np.array([-0.2, 0.01, 0.3], np.float32), np.array([0.5, 0.4, 20.0], np.float32), np.float32(32000))
    eng.obs_stats.copy_(dev(np.concatenate([stats[0], stats[1], [stats[2]]])))
    eng.generation_index = 1
    fit = eng.evaluate().cpu().numpy().astype(np.float64)
    ref, (osum, osq, cnt) = po.closed_fitness(theta, H, 0.1, seed, 1, 0, N, reps, stats)
    assert np.max(np.abs(fit - ref) / np.abs(ref)) < RTOL
    assert eng.steps_taken == N * reps * 200
    t = eng.obs_totals.cpu().numpy()
    assert t[6] == cnt and np.allclose(t[:3], osum, rtol=RTOL, atol=1e-3 * cnt ** 0.5) and np.allclose(t[3:6], osq,
                                                                                                      rtol=RTOL)
    ref_t = po.test_returns(theta, H, seed, 1, reps, stats)
    assert np.max(np.abs(eng.test_returns() - ref_t) / np.abs(ref_t)) < RTOL


def test_two_shards_on_one_gpu_equal_one_shard():
    """Episodes keyed by the global member: two shards' fitness and statistics rows equal the whole population's."""
    from distributedes_b200 import ops
    from distributedes_b200.engine import HostEpisodes
    H, N, reps, seed, gen = 32, 11, 10, 6, 3
    rows = ops.nes_perturb(dev(orc.synthetic_theta(3, H, 1, seed=1)), N, 0.1, seed, gen)
    out = []
    for lo, hi in ((0, N), (0, 5), (5, N)):
        part = torch.zeros((hi - lo, 7), dtype=torch.float64, device='cuda')
        ep = HostEpisodes(ops, 'cuda', po.PendulumBatch((hi - lo) * reps, seed, horizon=60), hi - lo, reps, 3, H, 1, 2.0,
                          0.2, seed)
        ret, steps = ep.run(rows[lo:hi].contiguous(), generation=gen, member_offset=lo, stat_part=part)
        out.append((ret.mean(1).astype(np.float32), part.cpu().numpy(), steps))
    assert np.array_equal(out[0][0], np.concatenate([out[1][0], out[2][0]]))
    assert np.array_equal(out[0][1], np.concatenate([out[1][1], out[2][1]]))
    assert out[0][2] == out[1][2] + out[2][2] == N * reps * 60
