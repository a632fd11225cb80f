"""Oracle-backed stand-in for the genetic algorithm's novelty-search ops (ops.rollout_eval_ga_bc, ops.ns_ga_order,
ops.ns_ga_order_workspace), on CPU tensors.  TEST-ONLY: the closed-loop evaluation is pendulum_oracle's episode loop over
ga_oracle's member rows with the behaviour of oracle/novelty_oracle.py, and the order is tests/ga_novelty_oracle.py's.
Combined with cpu_ops, cpu_ops_ga and cpu_ops_novelty it stands in for the kernels novelty.train_ga calls.  Every call is
appended to CALLS."""
import numpy as np
import torch

import cpu_ops
import ga_novelty_oracle as gno
from oracle import ga_oracle as ga
from oracle import novelty_oracle as no

CALLS = []


def rollout_eval_ga_bc(parents, n_elites, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip,
                       action_noise_std=0.0, seed, generation=0, state=None, member_offset=0, n_local, obs_stats=None,
                       totals_out=None, workspace=None, out=None, episodes_out=None, bc_out):
    gen, stats = cpu_ops._gen(state, generation), cpu_ops._stats(obs_stats, 3)
    CALLS.append(dict(op='rollout_eval_ga_bc', n_parents=parents.shape[0], n_elites=n_elites, sigma=sigma, seed=seed,
                      generation=gen, member_offset=member_offset, n_local=n_local))
    members = np.arange(member_offset, member_offset + n_local)
    rows = ga.member_rows(parents.numpy(), n_elites, sigma, seed, gen, members)
    ret, (osum, osq, cnt), bc = no.closed_episodes(rows, hidden, seed, gen, members, repetitions, stats, horizon, clip,
                                                   action_noise_std)
    bc_out.copy_(torch.from_numpy(bc).reshape(bc_out.shape))
    if episodes_out is not None:
        episodes_out.copy_(cpu_ops._f32(ret).reshape(episodes_out.shape))
    return cpu_ops._rollout_out(ret.mean(1), osum, osq, cnt, totals_out, out)


def ns_ga_order_workspace(N, device):
    return torch.empty(0)


def ns_ga_order(fitness, novelty_, reward_weight, truncation, *, workspace=None, out=None):
    CALLS.append(dict(op='ns_ga_order', fitness=fitness.clone(), novelty=novelty_.clone(), reward_weight=reward_weight,
                      truncation=truncation))
    order = gno.ns_ga_order(fitness.numpy(), novelty_.numpy(), reward_weight, truncation).astype(np.int32)
    return cpu_ops._out(torch.from_numpy(order), out)
