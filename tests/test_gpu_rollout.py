"""des_rollout_eval (closed-loop Pendulum-v0 on the device, SURVEY 8f row 3) through the C ABI against
oracle/pendulum_oracle.py.

Tolerances: the policy is evaluated in fp32 on the device and in fp64 by the oracle; an episode is 200 steps of a
feedback loop, so per-step differences of ~1e-7 grow along the trajectory.  Observed |dR|/|R| <= ~1e-5 on returns of
magnitude ~1e3; the bound used is 2e-4."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu
RTOL = 2e-4


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


@pytest.mark.parametrize('H,n,reps,horizon', [(64, 24, 10, 200), (32, 9, 3, 50), (96, 5, 1, 120), (128, 6, 4, 200)])
def test_rollout_fitness_matches_oracle(H, n, reps, horizon):
    from distributedes_b200 import ops
    theta = orc.synthetic_theta(3, H, 1, seed=H)
    seed, gen, off = 21, 3, 5
    totals = torch.zeros(7, dtype=torch.float64, device='cuda')
    eps_out = torch.empty(n * reps, dtype=torch.float32, device='cuda')
    fit = ops.rollout_eval(dev(theta), hidden=H, horizon=horizon, repetitions=reps, sigma=0.1, clip=2.0, seed=seed,
                           generation=gen, member_offset=off, n_local=n, totals_out=totals, episodes_out=eps_out)
    ref, (osum, osq, cnt) = po.closed_fitness(theta, H, 0.1, seed, gen, off, n, reps, None, horizon)
    got = fit.cpu().numpy().astype(np.float64)
    assert np.max(np.abs(got - ref) / np.abs(ref)) < RTOL
    t = totals.cpu().numpy()
    assert t[6] == cnt == n * reps * horizon
    assert np.allclose(t[:3], osum, rtol=1e-4, atol=1e-3 * cnt ** 0.5) and np.allclose(t[3:6], osq, rtol=1e-4)
    # per-episode returns average to the fitness
    assert np.allclose(eps_out.cpu().numpy().reshape(n, reps).mean(1), got, rtol=1e-6)


def test_rollout_with_normaliser_statistics_and_test_episodes():
    from distributedes_b200 import ops
    H, n, reps = 64, 12, 10
    theta = orc.synthetic_theta(3, H, 1, seed=2)
    stats = (np.array([-0.2, 0.01, 0.3], np.float32), np.array([0.5, 0.4, 20.0], np.float32), np.float32(32000))
    st = dev(np.concatenate([stats[0], stats[1], [stats[2]]]))
    fit = ops.rollout_eval(dev(theta), hidden=H, repetitions=reps, sigma=0.1, clip=2.0, seed=4, generation=1,
                           member_offset=0, n_local=n, obs_stats=st)
    ref, _ = po.closed_fitness(theta, H, 0.1, 4, 1, 0, n, reps, stats)
    assert np.max(np.abs(fit.cpu().numpy() - ref) / np.abs(ref)) < RTOL
    # identity while n == 0 (utils.py:48-49)
    st0 = dev(np.concatenate([stats[0], stats[1], [0.0]]))
    fit0 = ops.rollout_eval(dev(theta), hidden=H, repetitions=reps, sigma=0.1, clip=2.0, seed=4, generation=1,
                            member_offset=0, n_local=n, obs_stats=st0)
    fit_none = ops.rollout_eval(dev(theta), hidden=H, repetitions=reps, sigma=0.1, clip=2.0, seed=4, generation=1,
                                member_offset=0, n_local=n)
    assert torch.equal(fit0, fit_none) and not torch.equal(fit0, fit)
    # test() episodes: unperturbed theta, the test reset stream
    ep = torch.empty(reps, dtype=torch.float32, device='cuda')
    ops.rollout_eval(dev(theta), hidden=H, repetitions=reps, sigma=0.1, clip=2.0, seed=4, generation=1, member_offset=0,
                     n_local=1, noiseless=True, obs_stats=st, episodes_out=ep)
    ref_t = po.test_returns(theta, H, 4, 1, reps, stats)
    assert np.max(np.abs(ep.cpu().numpy() - ref_t) / np.abs(ref_t)) < RTOL


def test_rollout_is_shard_invariant_and_deterministic():
    """Members are addressed globally: evaluating [0,20) in one launch or as [0,7)+[7,20) gives identical bits."""
    from distributedes_b200 import ops
    theta = dev(orc.synthetic_theta(3, 64, 1, seed=9))
    kw = dict(hidden=64, repetitions=10, sigma=0.1, clip=2.0, seed=8, generation=2)
    whole = ops.rollout_eval(theta, member_offset=0, n_local=20, **kw)
    again = ops.rollout_eval(theta, member_offset=0, n_local=20, **kw)
    a = ops.rollout_eval(theta, member_offset=0, n_local=7, **kw)
    b = ops.rollout_eval(theta, member_offset=7, n_local=13, **kw)
    assert torch.equal(whole, again) and torch.equal(whole, torch.cat([a, b]))


def test_rollout_action_noise_matches_oracle():
    from distributedes_b200 import ops
    H, n, reps = 32, 6, 2
    theta = orc.synthetic_theta(3, H, 1, seed=1)
    fit = ops.rollout_eval(dev(theta), hidden=H, horizon=60, repetitions=reps, sigma=0.1, clip=2.0, action_noise_std=0.3,
                           seed=17, generation=0, member_offset=2, n_local=n)
    eps = orc.noise(17, 0, 2, n, orc.param_count(3, H, 1))
    ret, _, _, _ = po.rollouts(orc.perturb(theta, 0.1, eps), H, 17, 0, np.arange(2, 2 + n), reps, None, 60, 2.0, 0.3)
    ref = ret.mean(1)
    assert np.max(np.abs(fit.cpu().numpy() - ref) / np.abs(ref)) < 5e-4      # MUFU normals (2^-21 abs) feed the loop


def test_rollout_rejects_bad_arguments():
    from distributedes_b200 import ops
    theta = dev(orc.synthetic_theta(3, 64, 1))
    with pytest.raises(RuntimeError, match='multiple of 32'):
        ops.rollout_eval(dev(orc.synthetic_theta(3, 48, 1)), hidden=48, sigma=0.1, clip=2.0, seed=0, n_local=2)
    with pytest.raises(RuntimeError, match='repetitions'):
        ops.rollout_eval(theta, hidden=64, repetitions=11, sigma=0.1, clip=2.0, seed=0, n_local=2)
    with pytest.raises(RuntimeError, match='unknown environment'):
        ops.rollout_eval(theta, env=5, hidden=64, sigma=0.1, clip=2.0, seed=0, n_local=2)
    with pytest.raises(RuntimeError, match='workspace'):
        ops.rollout_eval(theta, hidden=64, sigma=0.1, clip=2.0, seed=0, n_local=4,
                         totals_out=torch.zeros(7, dtype=torch.float64, device='cuda'),
                         workspace=torch.empty(3, dtype=torch.float64, device='cuda'))
