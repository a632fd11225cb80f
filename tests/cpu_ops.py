"""Oracle-backed stand-in for distributedes_b200.ops on CPU tensors.  TEST-ONLY: the CPU tests pass it as `kernels`, so
the host logic of engine.NESEngine, its closed-loop and host-stepped sources and the CMA-ES worker (sharding, the
collectives, ragged shards) runs under gloo without a GPU.  Every function has the name and arguments of its op
(test_cpu_ops.py checks it); the des_state counters live in a small tensor.  eval_workspace is deliberately absent:
without it the tape evaluation allocates no workspace."""
import numpy as np
import torch

from oracle import cma_oracle as cma
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po


def _gen(state, generation):
    """The generation word: the des_state counter when a state is given, else the explicit generation."""
    return int(state[0]) if state is not None else generation


def _stats(vec, d0):
    """The three parts of a [2 d0 + 1] vector: (mean, variance, count) of statistics, (sum, sum of squares, count) of
    totals.  None stays None."""
    if vec is None:
        return None
    a = vec.numpy()
    return a[:d0], a[d0:2 * d0], a[2 * d0]


def _out(res, out):
    """The ops' `out` convention: fill and return `out` when it is given, else return the new tensor."""
    if out is None:
        return res
    out.copy_(res.reshape(out.shape))
    return out


def _f32(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32))


def _rollout_out(fit, osum, osq, cnt, totals_out, out):
    if totals_out is not None:
        totals_out.copy_(torch.from_numpy(np.concatenate([osum, osq, [cnt]])))
    return _out(_f32(fit), out)


# ---- NES on the tape -------------------------------------------------------------------------------------------------
def param_count(d0, H, A):
    return orc.param_count(d0, H, A)


def new_state(device, generation=0):
    return torch.tensor([generation, 0, 1.0, 1.0], dtype=torch.float64)     # generation, adam_t, beta1_t, beta2_t


def state_advance(state, beta1=0.9, beta2=0.999):
    state[0] += 1
    state[1] += 1
    state[2] *= beta1
    state[3] *= beta2


def rank_workspace(n_local, device, N):
    return torch.empty(0)


def grad_workspace(n_local, P, device):
    return torch.empty(0)


def nes_eval(theta, obs, target, *, hidden, sigma, clip, seed, generation=0, state=None, member_offset=0, n_local,
             precision='fp32', out=None, workspace=None):
    f = orc.evaluate_population(theta.numpy(), obs.numpy(), target.numpy(), sigma, clip, seed, _gen(state, generation),
                                member_offset, n_local, obs.shape[1], hidden, target.shape[1])
    return _out(_f32(f), out)


def nes_eval_mirrored(theta, obs, target, *, hidden, sigma, clip, seed, generation=0, state=None, member_offset=0,
                      n_local, precision='fp32', out=None, workspace=None):
    f = mo.evaluate_population(theta.numpy(), obs.numpy(), target.numpy(), sigma, clip, seed, _gen(state, generation),
                               member_offset, n_local, obs.shape[1], hidden, target.shape[1])
    return _out(_f32(f), out)


def centered_rank(fitness_all, member_offset=0, n_local=None, *, workspace=None, return_ranks=False, out=None):
    return _out(_f32(orc.fitness_shift(fitness_all.numpy())[member_offset:member_offset + n_local]), out)


def nes_grad_partial(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None, out=None):
    s = shaped_local.numpy().astype(np.float64)
    part = s @ orc.noise(seed, _gen(state, generation), member_offset, s.size, P) if s.size else np.zeros(P)
    return _out(_f32(part), out)


def nes_grad_partial_mirrored(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None,
                              out=None):
    assert member_offset % 2 == 0 and shaped_local.numel() % 2 == 0, 'a mirrored shard holds whole pairs'
    s = shaped_local.numpy().astype(np.float64)
    c = s[0::2] - s[1::2]
    part = c @ orc.noise(seed, _gen(state, generation), member_offset // 2, c.size, P) if c.size else np.zeros(P)
    return _out(_f32(part), out)


def nes_apply(theta, adam_m, adam_v, partial_sum, N, state, *, sigma, learning_rate, weight_decay=0.005, beta1=0.9,
              beta2=0.999, epsilon=1e-8, update_out=None, grad_out=None):
    opt = orc.Adam(beta1, beta2, epsilon)
    opt.m, opt.v = adam_m.numpy().copy(), adam_v.numpy().copy()
    opt.beta1_t, opt.beta2_t = float(state[2]), float(state[3])
    g = partial_sum.numpy().astype(np.float64) / N / sigma
    th, upd = orc.nes_update(theta.numpy(), g, opt, weight_decay, learning_rate)
    theta.copy_(torch.from_numpy(th))
    adam_m.copy_(torch.from_numpy(np.asarray(opt.m)))
    adam_v.copy_(torch.from_numpy(np.asarray(opt.v)))
    if update_out is not None:
        update_out.copy_(torch.from_numpy(upd))


# ---- observation statistics ------------------------------------------------------------------------------------------
def _obs_stats(stats, d0):
    st = orc.ObsStats(d0)
    m, v, n = _stats(stats, d0)
    st.m, st.v, st.n = m.copy(), v.copy(), np.float32(n)
    return st


def obs_normalize(obs, stats, out=None):
    st = _obs_stats(stats, obs.shape[1])
    return _out(torch.from_numpy(np.stack([st.normalize(o) for o in obs.numpy()])), out)


def obs_stats_merge(stats, obs, n_feed):
    st = _obs_stats(stats, obs.shape[1])
    st.merge_tape(obs.numpy(), n_feed)
    stats.copy_(_f32(np.concatenate([st.m, st.v, [st.n]])))
    return stats


def obs_stats_merge_totals(stats, totals, state_dim):
    m, v, n = po.merge_totals(_stats(stats, state_dim), *_stats(totals, state_dim))
    stats.copy_(_f32(np.concatenate([m, v, [n]])))
    return stats


def obs_parts_reduce(parts, state_dim, out=None):
    tot = np.zeros(2 * state_dim + 1)
    for row in parts.numpy().reshape(-1, 2 * state_dim + 1):
        tot += row
    return _out(torch.from_numpy(tot), out)


# ---- closed-loop Pendulum rollouts on the device ---------------------------------------------------------------------
def rollout_eval(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                 generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None, totals_out=None,
                 workspace=None, out=None, episodes_out=None):
    gen, stats = _gen(state, generation), _stats(obs_stats, 3)
    if noiseless:
        ret = po.test_returns(theta.numpy(), hidden, seed, gen, repetitions, stats, horizon, clip)
        if episodes_out is not None:
            episodes_out.copy_(_f32(ret))
        return None
    fit, (osum, osq, cnt) = po.closed_fitness(theta.numpy(), hidden, sigma, seed, gen, member_offset, n_local,
                                              repetitions, stats, horizon, clip)
    return _rollout_out(fit, osum, osq, cnt, totals_out, out)


def rollout_eval_mirrored(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                          generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None,
                          totals_out=None, workspace=None, out=None, episodes_out=None):
    assert not noiseless and member_offset % 2 == 0 and n_local % 2 == 0
    fit, (osum, osq, cnt) = mo.closed_fitness(theta.numpy(), hidden, sigma, seed, _gen(state, generation), member_offset,
                                              n_local, repetitions, _stats(obs_stats, 3), horizon, clip)
    return _rollout_out(fit, osum, osq, cnt, totals_out, out)


def rollout_eval_solutions(solutions, *, env=0, hidden, horizon=200, repetitions=10, clip, action_noise_std=0.0, seed,
                           generation=0, member_offset=0, obs_stats=None, totals_out=None, workspace=None, out=None,
                           episodes_out=None):
    n = solutions.shape[0]
    ret, osum, osq, cnt = po.rollouts(solutions.numpy(), hidden, seed, generation,
                                      np.arange(member_offset, member_offset + n), repetitions, _stats(obs_stats, 3),
                                      horizon, clip, action_noise_std)
    return _rollout_out(ret.mean(1), osum, osq, cnt, totals_out, out)


# ---- host-stepped environments ---------------------------------------------------------------------------------------
def nes_perturb(theta, n_members, sigma, seed, generation, member_offset=0, out=None):
    P = theta.numel()
    eps = orc.noise(seed, generation, member_offset, n_members, P)
    return _out(_f32(orc.perturb(theta.numpy(), sigma, eps)).reshape(n_members, P), out)


def nes_perturb_mirrored(theta, n_members, sigma, seed, generation, member_offset=0, out=None):
    P = theta.numel()
    eps = mo.noise_mirrored(seed, generation, member_offset, n_members, P)
    return _out(_f32(orc.perturb(theta.numpy(), sigma, eps)).reshape(n_members, P), out)


def policy_act(rows, obs, alive, *, state_dim, hidden, action_dim, repetitions, clip, action_noise_std=0.0, seed,
               generation, member_offset=0, t, obs_stats=None, stat_part=None, out=None):
    n, d0, reps = rows.shape[0], state_dim, repetitions
    o = obs.numpy().reshape(n, reps, d0)
    al = alive.numpy().reshape(n, reps).astype(bool)
    if stat_part is not None:
        po.accumulate_stats(stat_part.numpy().reshape(n, 2 * d0 + 1), o, al)
    act = po.policy_actions(rows.numpy(), o, al, d0, hidden, action_dim, clip, _stats(obs_stats, d0), action_noise_std,
                            seed, generation, member_offset, t)
    return _out(_f32(act).reshape(n, reps, action_dim), out)


# ---- CMA-ES ----------------------------------------------------------------------------------------------------------
def noise_fill(n_members, P, seed, generation, member_offset=0, stream_tag=0, device='cpu'):
    return _f32(orc.noise(seed, generation, member_offset, n_members, P, stream=stream_tag))


def pop_eval(solutions, obs, target, *, hidden, clip, out=None):
    d0, A = obs.shape[1], target.shape[1]
    f = [orc.tape_fitness(orc.forward(s, obs.numpy(), d0, hidden, A), target.numpy(), clip) for s in solutions.numpy()]
    return _out(torch.tensor(f, dtype=torch.float32), out)


def cma_rank_mu(Y, w, out=None):
    return _out(_f32(cma.rank_mu_delta(Y.numpy().astype(np.float64), w.numpy().astype(np.float64))), out)


def cma_cov_apply(Cmat, dC, pc, *, decay, c1, cmu):
    p = pc.numpy().astype(np.float64)
    new = decay * Cmat.numpy().astype(np.float64) + c1 * np.outer(p, p) + cmu * dC.numpy().astype(np.float64)
    Cmat.copy_(_f32(new))
    return Cmat


# the "packed" payload of the stand-ins is the flattened full matrix: only these functions read it
def cma_packed_elems(n):
    return n * n


def cma_rank_mu_packed(Y, w, out=None):
    return _out(cma_rank_mu(Y, w).reshape(-1), out)


def cma_cov_apply_packed(Cmat, tiles, pc, *, decay, c1, cmu):
    n = Cmat.shape[0]
    return cma_cov_apply(Cmat, tiles.reshape(n, n), pc, decay=decay, c1=c1, cmu=cmu)
