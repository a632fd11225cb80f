"""CPU stand-ins for the mirrored-sampling ops (same names and arguments as distributedes_b200.ops), on top of
tests/fake_kernels.py, for the gloo runs of NESEngine / RolloutEngine with mirrored=True.  TEST-ONLY."""
import numpy as np
import torch

from fake_kernels import *          # noqa: F401,F403  the plain NESEngine ops on CPU tensors
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po


def _gen(state, generation):
    return int(state[0]) if state is not None else generation


def nes_eval_mirrored(theta, obs, target, *, hidden, sigma, clip, seed, generation=0, state=None, member_offset=0,
                      n_local, precision='fp32', out=None, workspace=None):
    T, d0 = obs.shape
    f = mo.evaluate_population(theta.numpy(), obs.numpy(), target.numpy(), sigma, clip, seed, _gen(state, generation),
                               member_offset, n_local, d0, hidden, target.shape[1])
    out.copy_(torch.from_numpy(f.astype(np.float32)))
    return out


def nes_grad_partial_mirrored(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None,
                              out=None):
    assert member_offset % 2 == 0 and shaped_local.numel() % 2 == 0, 'a mirrored shard holds whole pairs'
    s = shaped_local.numpy().astype(np.float64)
    c = (s[0::2] - s[1::2])
    part = c @ orc.noise(seed, _gen(state, generation), member_offset // 2, c.size, P) if c.size else np.zeros(P)
    out.copy_(torch.from_numpy(part.astype(np.float32)))
    return out


def rollout_eval_mirrored(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                          generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None,
                          totals_out=None, workspace=None, out=None, episodes_out=None):
    assert not noiseless and member_offset % 2 == 0 and n_local % 2 == 0
    stats = None
    if obs_stats is not None:
        a = obs_stats.numpy()
        stats = (a[:3], a[3:6], a[6])
    fit, (osum, osq, cnt) = mo.closed_fitness(theta.numpy(), hidden, sigma, seed, _gen(state, generation), member_offset,
                                              n_local, repetitions, stats, horizon, clip)
    out.copy_(torch.from_numpy(fit.astype(np.float32)))
    if totals_out is not None:
        totals_out.copy_(torch.from_numpy(np.concatenate([osum, osq, [cnt]])))
    return out


def nes_perturb_mirrored(theta, n_members, sigma, seed, generation, member_offset=0, out=None):
    P = theta.numel()
    rows = orc.perturb(theta.numpy(), sigma, mo.noise_mirrored(seed, generation, member_offset, n_members, P))
    res = torch.from_numpy(np.asarray(rows, dtype=np.float32).reshape(n_members, P))
    if out is None:
        return res
    out.copy_(res)
    return out


def closed_chain(theta, H, N, reps, seed, sigma, lr, wd, gens, horizon=po.HORIZON):
    """Single-process chain of mirrored closed-loop generations with the oracle; yields per-generation records."""
    P = theta.size
    stats = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    opt = orc.Adam()
    for gen in range(gens):
        test = po.test_returns(theta, H, seed, gen, reps, stats, horizon)
        fit, (osum, osq, cnt) = mo.closed_fitness(theta, H, sigma, seed, gen, 0, N, reps, stats, horizon)
        stats = po.merge_totals(stats, osum, osq, cnt)
        grad = mo.nes_gradient_streamed(orc.fitness_shift(fit), sigma, seed, gen, P)
        theta, _ = orc.nes_update(theta, grad, opt, wd, lr)
        yield dict(test=test, fitness=fit, stats=np.concatenate([stats[0], stats[1], [stats[2]]]),
                   grad_after_wd=grad - wd * grad, theta=theta)
