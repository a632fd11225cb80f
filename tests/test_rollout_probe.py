"""The rollout probe (oracle/rollout_probe.py) and the closed-loop error bound (oracle/forward_error.py, 'mufu') on the
CPU: trajectories made by oracle/pendulum_oracle.py, summed into fp64 totals in the kernel's order and differenced as
the GPU test differences the device's totals."""
import numpy as np
import pytest

from oracle import forward_error as fe
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import rollout_probe as rp

SEED, GEN = 21, 3


def _flat(H, member=5, sigma=0.1):
    theta = orc.synthetic_theta(3, H, 1, seed=H)
    return orc.perturb(theta, sigma, orc.noise(SEED, GEN, member, 1, orc.param_count(3, H, 1)))[0]


@pytest.mark.parametrize('H,steps,clip,noise', [(32, range(0, 60), 2.0, 0.0), (16, list(range(0, 8)) + list(range(150, 170)), 0.5, 0.3),
                                                (64, range(0, 40), 3.0, 0.0)])
def test_recovery_is_exact_to_its_resolution(H, steps, clip, noise):
    """Observations come back within their stated error (in practice exactly), torques within their resolution at
    every non-saturated step, and the step-0 observations are the reset states'."""
    member = 5
    flat = _flat(H, member)
    hs = rp.horizons(steps)
    totals = rp.simulate_totals(flat, H, SEED, GEN, member, hs, clip=clip, act_noise=noise)
    obs, err = rp.observations(totals, hs)
    _, _, _, _, (o_true, u_true) = po.rollouts(flat.reshape(1, -1), H, SEED, GEN, [member], rp.EPISODES, None, max(hs),
                                               clip, noise, trace=True)
    o_true, u_true = o_true[0].astype(np.float64), u_true[0]
    known = np.isfinite(obs)
    assert known[:, list(steps)].all()
    assert np.all(np.abs(obs - o_true)[known] <= err[known])
    assert np.max(err[known]) < 1e-11
    assert np.array_equal(obs[:, 0].astype(np.float32), rp.reset_observations(SEED, GEN, member))
    u, res, valid = rp.torques(obs, err)
    t = np.asarray(list(steps))
    u, res, valid, ut = u[:, t], res[:, t], valid[:, t], u_true[:, t]
    assert valid.mean() > 0.5
    assert np.all(np.abs(u - ut)[valid] <= res[valid])
    assert np.max(res[valid]) < 5e-6
    # the dynamics step predicts the next observation from the recovered torque
    pred = rp.predict(obs, np.where(np.isfinite(u_true[:, :obs.shape[1] - 1]), u_true[:, :obs.shape[1] - 1], 0))
    tol = rp.predict_tolerance(obs)
    ok = np.isfinite(pred).all(-1) & np.isfinite(obs[:, 1:]).all(-1)
    assert np.all((np.abs(pred - obs[:, 1:]) <= tol)[ok])


def test_resolution_catches_a_wrong_torque():
    """A torque off by 3x the resolution at one step shows in the recovered torque of that step."""
    H, member, steps = 16, 2, range(0, 12)
    flat = _flat(H, member)
    hs = rp.horizons(steps)
    obs, err = rp.observations(rp.simulate_totals(flat, H, SEED, GEN, member, hs), hs)
    u, res, valid = rp.torques(obs, err)
    _, _, _, _, (_, ut) = po.rollouts(flat.reshape(1, -1), H, SEED, GEN, [member], rp.EPISODES, None, max(hs), 2.0,
                                      trace=True)
    e, t = np.argwhere(valid[:, :10])[0]
    assert abs(u[e, t] + 3 * res[e, t] - ut[0, e, t]) > res[e, t]


def test_mufu_bound_covers_an_emulated_kernel():
    """The fp32 FFMA chains and the butterfly of rollout_pendulum_kernel emulated in numpy, with tanh off by up to
    TANH_MUFU_ABS, the normaliser in fp32 and the noise added by one FMA: every action within B of a*."""
    rs = np.random.RandomState(0)
    for H in (16, 32, 96, 128):
        R = H // 16
        flat = _flat(H).astype(np.float32)
        W1, b1, W2, b2, W3, b3 = orc.unflatten(flat, 3, H, 1)
        obs = np.concatenate([np.stack([np.cos(th := rs.uniform(-np.pi, np.pi, 200)), np.sin(th)], 1),
                              rs.uniform(-8, 8, (200, 1))], 1).astype(np.float32)
        stats = (np.float32([-0.2, 0.01, 0.3]), np.float32([0.5, 0.4, 20.0]), np.float32(3200))
        z = rs.randn(200).astype(np.float32)
        std = np.float32(0.3)

        def fma(a, b, c):
            return np.float32(np.float64(a) * np.float64(b) + np.float64(c))

        def tanh(v):
            return np.float32(np.tanh(np.float64(v)) + rs.uniform(-1, 1) * fe.TANH_MUFU_ABS)

        a = np.empty(200)
        for t in range(200):
            s = np.sqrt(stats[1] + np.float32(1e-6)).astype(np.float32)
            x = ((obs[t] - stats[0]) / s).astype(np.float32)
            h1 = [tanh(fma(W1[j, 2], x[2], fma(W1[j, 1], x[1], fma(W1[j, 0], x[0], b1[j])))) for j in range(H)]
            h2 = []
            for j in range(H):
                acc = b2[j]
                for pk in range(H):
                    k = (pk % 16) * R + pk // 16
                    acc = fma(W2[j, k], h1[k], acc)
                h2.append(tanh(acc))
            p = [np.float32(0)] * 16
            for g in range(16):
                for r in range(R):
                    p[g] = fma(W3[0, g * R + r], h2[g * R + r], p[g])
            for st in (1, 2, 4, 8):
                for q in range(0, 16, 2 * st):
                    p[q] = np.float32(p[q] + p[q + st])
            a[t] = fma(z[t], std, np.float32(p[0] + b3[0]))
        noise = (np.float64(z) * np.float64(std))[:, None]
        ref = fe.closed_loop_actions(flat, obs, 3, H, 1, stats, noise)[:, 0]
        B = fe.closed_loop_bound(flat, obs, 3, H, 1, stats, noise)[:, 0]
        assert np.all(np.abs(a - ref) <= B), np.max(np.abs(a - ref) / B)
        assert np.max(np.abs(a - ref) / B) > 1e-3                       # the bound is not vacuous either


def test_mufu_bound_shrinks_to_the_roundings_when_w2_is_zero():
    """With W2 = 0 layer 2 is tanh(b2) whatever the observation: B is the same for every observation and is made of the
    roundings alone — tanh_mufu's absolute error and the bias chain through W3, and layer 3's own roundings."""
    H = 64
    flat = _flat(H).astype(np.float64)
    W1, b1, W2, b2, W3, b3 = orc.unflatten(flat, 3, H, 1)
    W2[...] = 0.0
    rs = np.random.RandomState(1)
    obs = rs.uniform(-1, 1, (50, 3))
    B = fe.closed_loop_bound(flat, obs, 3, H, 1)[:, 0]
    assert np.allclose(B, B[0], rtol=1e-12)
    u = 2.0 ** -24
    aW3 = np.abs(W3[0])
    expect = aW3 @ ((H + 3) * u * np.abs(b2) + fe.TANH_MUFU_ABS) + (H // 16 + 6) * u * (aW3.sum() + abs(b3[0]))
    assert B[0] <= expect * 1.001
    flat0 = _flat(H).astype(np.float64)
    assert B[0] < fe.closed_loop_bound(flat0, obs, 3, H, 1)[:, 0].min() / 5
    # and the normaliser adds its 4 roundings only when statistics are in use
    stats = (np.float32([0.1, 0.0, 0.2]), np.float32([0.5, 0.5, 10.0]), np.float32(100))
    off = (np.float32([0.1, 0.0, 0.2]), np.float32([0.5, 0.5, 10.0]), np.float32(0))
    assert np.array_equal(fe.closed_loop_bound(flat0, obs, 3, H, 1, off), fe.closed_loop_bound(flat0, obs, 3, H, 1))
    assert not np.array_equal(fe.closed_loop_bound(flat0, obs, 3, H, 1, stats), fe.closed_loop_bound(flat0, obs, 3, H, 1))


def test_oracle_keeps_nan_actions_nan():
    """np.clip keeps NaN, in the action clip and in gym's Pendulum: a NaN b3 gives NaN returns; an infinite W3 entry
    gives an infinite action, which clips like any other."""
    H = 16
    flat = _flat(H)[None].repeat(3, 0)
    P = flat.shape[1]
    flat[0, P - 1] = np.nan                                            # b3
    flat[1, P - 1 - H + 3] = np.inf                                    # one W3 entry
    ret, _, _, _ = po.rollouts(flat, H, SEED, GEN, [0, 1, 2], 4, horizon=20)
    assert np.isnan(ret[0]).all() and np.isfinite(ret[1:]).all()
    assert np.isnan(rp.applied(np.array([np.nan]), 0.5)).all()
    assert np.array_equal(rp.applied(np.array([np.inf, -np.inf, 1.0]), 3.0), [2.0, -2.0, 1.0])
