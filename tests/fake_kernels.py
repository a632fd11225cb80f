"""Oracle-backed stand-in for distributedes_b200.ops on CPU tensors.  TEST-ONLY: lets the world_size>1 host
logic of engine.NESEngine (sharding, the two all-reduces, ragged shards) run under gloo without a GPU.  It has
the same function names/arguments as the ops module and keeps the des_state counters in a small tensor."""
import numpy as np
import torch

from oracle import nes_oracle as orc


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
    gen = int(state[0]) if state is not None else generation
    T, d0 = obs.shape
    A = target.shape[1]
    f = orc.evaluate_population(theta.numpy(), obs.numpy(), target.numpy(), sigma, clip, seed, gen, member_offset,
                                n_local, d0, hidden, A)
    res = torch.from_numpy(f.astype(np.float32))
    if out is None:
        return res
    out.copy_(res)
    return out


def centered_rank(fitness_all, member_offset=0, n_local=None, *, workspace=None, return_ranks=False, out=None):
    s = orc.fitness_shift(fitness_all.numpy())[member_offset:member_offset + n_local].astype(np.float32)
    out.copy_(torch.from_numpy(s))
    return out


def nes_grad_partial(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None, out=None):
    gen = int(state[0]) if state is not None else generation
    n = shaped_local.numel()
    part = shaped_local.numpy().astype(np.float64) @ orc.noise(seed, gen, member_offset, n, P) if n else np.zeros(P)
    out.copy_(torch.from_numpy(part.astype(np.float32)))
    return out


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


def _unpack(stats, d0):
    st = orc.ObsStats(d0)
    a = stats.numpy()
    st.m, st.v, st.n = a[:d0].copy(), a[d0:2 * d0].copy(), np.float32(a[2 * d0])
    return st


def obs_normalize(obs, stats, out=None):
    d0 = obs.shape[1]
    st = _unpack(stats, d0)
    res = torch.from_numpy(np.stack([st.normalize(o) for o in obs.numpy()]))
    if out is None:
        return res
    out.copy_(res)
    return out


def obs_stats_merge(stats, obs, n_feed):
    d0 = obs.shape[1]
    st = _unpack(stats, d0)
    st.merge_tape(obs.numpy(), n_feed)
    stats.copy_(torch.from_numpy(np.concatenate([st.m, st.v, [st.n]]).astype(np.float32)))
    return stats


def rollout_eval(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                 generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None, totals_out=None,
                 workspace=None, out=None, episodes_out=None):
    from oracle import pendulum_oracle as po
    gen = int(state[0]) if state is not None else generation
    stats = None
    if obs_stats is not None:
        a = obs_stats.numpy()
        stats = (a[:3], a[3:6], a[6])
    if noiseless:
        ret = po.test_returns(theta.numpy(), hidden, seed, gen, repetitions, stats, horizon, clip)
        if episodes_out is not None:
            episodes_out.copy_(torch.from_numpy(ret.astype(np.float32)))
        return None
    fit, (osum, osq, cnt) = po.closed_fitness(theta.numpy(), hidden, sigma, seed, gen, member_offset, n_local,
                                              repetitions, stats, horizon, clip)
    out.copy_(torch.from_numpy(fit.astype(np.float32)))
    if totals_out is not None:
        totals_out.copy_(torch.from_numpy(np.concatenate([osum, osq, [cnt]])))
    return out


def obs_stats_merge_totals(stats, totals, state_dim):
    from oracle import pendulum_oracle as po
    a, t = stats.numpy(), totals.numpy()
    d0 = state_dim
    m, v, n = po.merge_totals((a[:d0], a[d0:2 * d0], a[2 * d0]), t[:d0], t[d0:2 * d0], t[2 * d0])
    stats.copy_(torch.from_numpy(np.concatenate([m, v, [n]]).astype(np.float32)))
    return stats


# ---- CMA (for cma_es.CMAEvolutionStrategy under gloo) ------------------------------------------------------------------
def noise_fill(n_members, P, seed, generation, member_offset=0, stream_tag=0, device='cpu'):
    return torch.from_numpy(orc.noise(seed, generation, member_offset, n_members, P, stream=stream_tag).astype(np.float32))


def cma_rank_mu(Y, w, out=None):
    from oracle import cma_oracle as cma
    res = torch.from_numpy(cma.rank_mu_delta(Y.numpy().astype(np.float64), w.numpy().astype(np.float64)).astype(np.float32))
    if out is None:
        return res
    out.copy_(res)
    return out


def cma_cov_apply(Cmat, dC, pc, *, decay, c1, cmu):
    p = pc.numpy().astype(np.float64)
    new = decay * Cmat.numpy().astype(np.float64) + c1 * np.outer(p, p) + cmu * dC.numpy().astype(np.float64)
    Cmat.copy_(torch.from_numpy(new.astype(np.float32)))
    return Cmat


# the "packed" payload of the stand-ins is the flattened full matrix: only these functions read it
def cma_packed_elems(n):
    return n * n


def cma_rank_mu_packed(Y, w, out=None):
    res = cma_rank_mu(Y, w).reshape(-1)
    if out is None:
        return res
    out.copy_(res)
    return out


def cma_cov_apply_packed(Cmat, tiles, pc, *, decay, c1, cmu):
    n = Cmat.shape[0]
    return cma_cov_apply(Cmat, tiles.reshape(n, n), pc, decay=decay, c1=c1, cmu=cmu)
