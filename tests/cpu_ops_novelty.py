"""Oracle-backed stand-in for novelty search's ops (ops.rollout_eval_bc, ops.novelty, ops.ns_shape,
ops.ns_shape_workspace), on CPU tensors.  TEST-ONLY: the closed-loop evaluation is pendulum_oracle's episode loop with the
behaviour of oracle/novelty_oracle.py, the novelty its fp32-faithful restatement and the shaping its blend.  Combined
with cpu_ops it stands in for the kernels novelty.py calls.  Every call is appended to CALLS."""
import numpy as np
import torch

import cpu_ops
from oracle import nes_oracle as orc
from oracle import novelty_oracle as no
from oracle import pendulum_oracle as po

CALLS = []


def rollout_eval_bc(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                    generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None, totals_out=None,
                    workspace=None, out=None, episodes_out=None, bc_out):
    gen, stats = cpu_ops._gen(state, generation), cpu_ops._stats(obs_stats, 3)
    CALLS.append(dict(op='rollout_eval_bc', generation=gen, noiseless=noiseless, seed=seed, n_local=n_local))
    th = theta.numpy()
    if noiseless:
        rows, members = th.reshape(1, -1), [po.TEST_MEMBER]
    else:
        rows = orc.perturb(th, sigma, orc.noise(seed, gen, member_offset, n_local, th.size))
        members = np.arange(member_offset, member_offset + n_local)
    ret, (osum, osq, cnt), bc = no.closed_episodes(rows, hidden, seed, gen, members, repetitions, stats, horizon, clip,
                                                   action_noise_std)
    bc_out.copy_(torch.from_numpy(bc).reshape(bc_out.shape))
    if episodes_out is not None:
        episodes_out.copy_(cpu_ops._f32(ret).reshape(episodes_out.shape))
    return cpu_ops._rollout_out(ret.mean(1), osum, osq, cnt, totals_out, out)


def novelty(queries, archive, k, *, out=None):
    CALLS.append(dict(op='novelty', queries=queries.clone(), archive=archive.clone(), k=k))
    return cpu_ops._out(torch.from_numpy(no.novelty_fp32(queries.numpy(), archive.numpy(), k)), out)


def ns_shape_workspace(N, device):
    return torch.empty(0)


def ns_shape(fitness, novelty_, reward_weight, *, workspace=None, out=None):
    CALLS.append(dict(op='ns_shape', reward_weight=reward_weight))
    return cpu_ops._out(torch.from_numpy(no.blend(fitness.numpy(), novelty_.numpy(), reward_weight)), out)
