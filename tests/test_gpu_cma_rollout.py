"""des_rollout_eval_solutions (explicit solution rows rolled out on the device), the rows closed-loop CMA-ES evaluates:
bit identity with the NES rollout of the same weights, the oracle, shard invariance and the device's ask() noise.

Tolerances: as tests/test_gpu_rollout.py for rollouts of sigma = 0.1 perturbations (2e-4)."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu
RTOL = 2e-4


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


def _stats():
    return (np.array([-0.2, 0.01, 0.3], np.float32), np.array([0.5, 0.4, 20.0], np.float32), np.float32(32000))


def _run_both(H, n, off, reps, horizon, stats, act_noise, seed=11, gen=4, sigma=0.1):
    from distributedes_b200 import ops
    theta = dev(orc.synthetic_theta(3, H, 1, seed=H + 1))
    st = dev(np.concatenate([stats[0], stats[1], [stats[2]]])) if stats is not None else None
    outs = []
    for mode in ('nes', 'rows'):
        totals = torch.zeros(7, dtype=torch.float64, device='cuda')
        eps = torch.empty(n * reps, dtype=torch.float32, device='cuda')
        kw = dict(hidden=H, horizon=horizon, repetitions=reps, clip=2.0, action_noise_std=act_noise, seed=seed,
                  generation=gen, member_offset=off, obs_stats=st, totals_out=totals, episodes_out=eps)
        if mode == 'nes':
            fit = ops.rollout_eval(theta, sigma=sigma, n_local=n, **kw)
        else:
            rows = ops.nes_perturb(theta, n, sigma, seed, gen, member_offset=off)
            fit = ops.rollout_eval_solutions(rows, **kw)
        outs.append((fit, eps, totals))
    return outs


@pytest.mark.parametrize('H', [16, 32, 64, 128])
@pytest.mark.parametrize('stats,act_noise', [(None, 0.0), ('stats', 0.0), ('stats', 0.3)])
def test_solution_rows_equal_the_nes_rollout_bit_for_bit(H, stats, act_noise):
    """Rows fp32(theta + sigma*eps_m) from des_nes_perturb evaluate to the same bits as des_rollout_eval's own
    perturbation: both compute fmaf(sigma, eps, theta), and every counter is keyed by the global member index."""
    (f0, e0, t0), (f1, e1, t1) = _run_both(H, 19, 6, 10, 80, _stats() if stats else None, act_noise)
    assert torch.equal(f0, f1) and torch.equal(e0, e1) and torch.equal(t0, t1)


@pytest.mark.parametrize('H,n,reps,horizon', [(16, 24, 10, 200), (32, 9, 3, 50), (64, 12, 10, 200), (96, 5, 1, 120),
                                              (128, 6, 4, 200)])
def test_solution_rows_match_oracle(H, n, reps, horizon):
    from distributedes_b200 import ops
    seed, gen, off = 21, 3, 5
    P = orc.param_count(3, H, 1)
    rows = (orc.synthetic_theta(3, H, 1, seed=H)[None, :]
            + 0.1 * np.random.RandomState(H).randn(n, P)).astype(np.float32)
    stats = _stats() if H in (16, 64) else None
    st = dev(np.concatenate([stats[0], stats[1], [stats[2]]])) if stats is not None else None
    totals = torch.zeros(7, dtype=torch.float64, device='cuda')
    eps = torch.empty(n * reps, dtype=torch.float32, device='cuda')
    fit = ops.rollout_eval_solutions(dev(rows), hidden=H, horizon=horizon, repetitions=reps, clip=2.0, seed=seed,
                                     generation=gen, member_offset=off, obs_stats=st, totals_out=totals, episodes_out=eps)
    ret, osum, osq, cnt = po.rollouts(rows, H, seed, gen, np.arange(off, off + n), reps, stats, horizon)
    got = fit.cpu().numpy().astype(np.float64)
    assert np.max(np.abs(got - ret.mean(1)) / np.abs(ret.mean(1))) < RTOL
    ep = eps.cpu().numpy().reshape(n, reps).astype(np.float64)
    assert np.max(np.abs(ep - ret) / np.abs(ret)) < RTOL
    t = totals.cpu().numpy()
    assert t[6] == cnt == n * reps * horizon
    assert np.allclose(t[:3], osum, rtol=RTOL, atol=1e-3 * cnt ** 0.5) and np.allclose(t[3:6], osq, rtol=RTOL)


def test_nes_rollout_at_16_hidden_units_matches_oracle():
    from distributedes_b200 import ops
    theta = orc.synthetic_theta(3, 16, 1, seed=5)
    stats = _stats()
    totals = torch.zeros(7, dtype=torch.float64, device='cuda')
    fit = ops.rollout_eval(dev(theta), hidden=16, repetitions=10, sigma=0.1, clip=2.0, seed=9, generation=2,
                           member_offset=3, n_local=20, obs_stats=dev(np.concatenate([stats[0], stats[1], [stats[2]]])),
                           totals_out=totals)
    ref, (osum, osq, cnt) = po.closed_fitness(theta, 16, 0.1, 9, 2, 3, 20, 10, stats)
    assert np.max(np.abs(fit.cpu().numpy() - ref) / np.abs(ref)) < RTOL
    t = totals.cpu().numpy()
    assert t[6] == cnt and np.allclose(t[3:6], osq, rtol=RTOL)
    ep = torch.empty(10, dtype=torch.float32, device='cuda')
    ops.rollout_eval(dev(theta), hidden=16, repetitions=10, sigma=0.1, clip=2.0, seed=9, generation=2, member_offset=0,
                     n_local=1, noiseless=True, episodes_out=ep)
    ref_t = po.test_returns(theta, 16, 9, 2, 10)
    assert np.max(np.abs(ep.cpu().numpy() - ref_t) / np.abs(ref_t)) < RTOL


def test_width_48_is_still_rejected_by_both_entry_points():
    from distributedes_b200 import ops
    th = dev(orc.synthetic_theta(3, 48, 1))
    with pytest.raises(RuntimeError, match='multiple of 32'):
        ops.rollout_eval(th, hidden=48, sigma=0.1, clip=2.0, seed=0, n_local=2)
    with pytest.raises(RuntimeError, match='multiple of 32'):
        ops.rollout_eval_solutions(th.reshape(1, -1).repeat(2, 1).contiguous(), hidden=48, clip=2.0, seed=0)
    with pytest.raises(RuntimeError, match='MLP needs'):
        ops.rollout_eval_solutions(dev(np.zeros((2, 354))), hidden=16, clip=2.0, seed=0)


def test_solution_rows_are_shard_invariant_and_deterministic():
    from distributedes_b200 import ops
    P = orc.param_count(3, 16, 1)
    rows = dev(np.random.RandomState(1).randn(20, P) * 0.5)
    kw = dict(hidden=16, repetitions=10, clip=2.0, seed=8, generation=2, action_noise_std=0.1)
    whole = ops.rollout_eval_solutions(rows, member_offset=0, **kw)
    again = ops.rollout_eval_solutions(rows, member_offset=0, **kw)
    a = ops.rollout_eval_solutions(rows[:7].contiguous(), member_offset=0, **kw)
    b = ops.rollout_eval_solutions(rows[7:].contiguous(), member_offset=7, **kw)
    assert torch.equal(whole, again) and torch.equal(whole, torch.cat([a, b]))


def test_noise_of_device_ask_is_the_stub_s_within_mufu_error():
    """The golden's pycma stand-in draws z from the same counter stream; the device's MUFU normals differ from the fp64
    restatement by at most 4e-6 * (1 + |z|)."""
    from distributedes_b200 import ops
    z = ops.noise_fill(16, 353, 7, 0, stream_tag=1).cpu().numpy().astype(np.float64)
    ref = orc.noise(7, 0, 0, 16, 353, stream=orc.STREAM_CMA_Z)
    assert np.max(np.abs(z - ref) / (1 + np.abs(ref))) <= 4e-6
