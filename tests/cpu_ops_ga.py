"""Oracle-backed stand-in for the genetic algorithm's ops (ops.ga_rows, ops.rollout_eval_ga, ops.ga_order,
ops.ga_order_workspace), on CPU tensors.  TEST-ONLY: the rows are oracle/ga_oracle.py's member_rows, the closed-loop
evaluation is cpu_ops.rollout_eval_solutions of those rows at the same member offset, and the order is ga_oracle.order.
Combined with cpu_ops it stands in for the kernels genetic.py calls.  Every call is appended to CALLS."""
import numpy as np
import torch

import cpu_ops
from oracle import ga_oracle as ga

CALLS = []


def ga_rows(parents, n_elites, *, sigma, seed, generation, member_offset=0, n_local=None, members=None, out=None):
    m = members.numpy().astype(np.int64) if members is not None else np.arange(member_offset, member_offset + n_local)
    CALLS.append(dict(op='ga_rows', n_parents=parents.shape[0], n_elites=n_elites, sigma=sigma, seed=seed,
                      generation=generation, members=m.copy(), parents=parents.clone()))
    assert out is None or out.data_ptr() != parents.data_ptr(), 'the table is double-buffered'
    rows = torch.from_numpy(ga.member_rows(parents.numpy(), n_elites, sigma, seed, generation, m))
    return cpu_ops._out(rows, out)


def rollout_eval_ga(parents, n_elites, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0,
                    seed, generation=0, state=None, member_offset=0, n_local, obs_stats=None, totals_out=None,
                    workspace=None, out=None, episodes_out=None):
    gen = cpu_ops._gen(state, generation)
    CALLS.append(dict(op='rollout_eval_ga', n_parents=parents.shape[0], n_elites=n_elites, sigma=sigma, seed=seed,
                      generation=gen, member_offset=member_offset, n_local=n_local))
    rows = torch.from_numpy(ga.member_rows(parents.numpy(), n_elites, sigma, seed, gen,
                                           np.arange(member_offset, member_offset + n_local)))
    return cpu_ops.rollout_eval_solutions(rows, env=env, hidden=hidden, horizon=horizon, repetitions=repetitions,
                                          clip=clip, action_noise_std=action_noise_std, seed=seed, generation=gen,
                                          member_offset=member_offset, obs_stats=obs_stats, totals_out=totals_out,
                                          workspace=workspace, out=out, episodes_out=episodes_out)


def ga_order_workspace(N, device):
    return torch.empty(0)


def ga_order(fitness, truncation, *, workspace=None, out=None):
    CALLS.append(dict(op='ga_order', fitness=fitness.clone(), truncation=truncation))
    return cpu_ops._out(torch.from_numpy(ga.order(fitness.numpy(), truncation).astype(np.int32)), out)
