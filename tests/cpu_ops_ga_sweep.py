"""Oracle-backed stand-in for distributedes_b200.ops_runs with the genetic-algorithm sweep ops, on CPU tensors.  TEST-ONLY:
the ops of cpu_ops_cma_sweep, plus the four ops of ops_ga_sweep, each the single-run stand-in of cpu_ops_ga applied run by
run with run r's seed, sigma and action noise (its row of the sweep table) and its counts (its row of the count table,
clamped as the kernels clamp them) at member_offset 0, which is the contract the library's entry points keep.  The
count table is the library's own: ops_ga_sweep.ga_table builds it without a library call."""
import numpy as np
import torch

import cpu_ops_ga as g
from cpu_ops_cma_sweep import (centered_rank_runs, cma_cov_apply_runs, cma_rank_mu_runs, hp_rows,  # noqa: F401
                               nes_perturb_sweep, noise_fill_sweep, obs_parts_reduce_runs, obs_stats_merge_totals_runs,
                               param_count, policy_act_sweep, rollout_eval_solutions_sweep, rollout_eval_sweep, run_table)
from distributedes_b200.ops_ga_sweep import ga_table  # noqa: F401


def _counts(ga, r, rows):
    """(n_parents, n_elites, truncation) of run r, clamped to the buffer as the kernels clamp them."""
    T, E, Tr = (int(x) for x in ga[r, :3])
    T = min(max(T, 1), rows)
    return T, min(max(E, 0), T), min(max(Tr, 1), rows)


def rollout_eval_ga_sweep(parents, ga, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                          run_size, obs_stats=None, totals_out=None, workspace=None, out=None, episodes_out=None):
    R, rows, N = parents.shape[0], parents.shape[1], int(run_size)
    out = torch.empty((R, N)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        T, E, _ = _counts(ga, r, rows)
        g.rollout_eval_ga(parents[r, :T], E, hidden=hidden, horizon=horizon, repetitions=repetitions, sigma=h.sigma,
                          clip=clip, action_noise_std=h.action_noise_std, seed=h.seed, generation=generation, state=state,
                          member_offset=0, n_local=N, obs_stats=None if obs_stats is None else obs_stats[r],
                          totals_out=None if totals_out is None else totals_out[r], out=out[r],
                          episodes_out=None if episodes_out is None else episodes_out[r])
    return out


def ga_rows_sweep(parents, ga, hp, *, generation, run_size, members=None, out=None):
    R, rows, P = parents.shape
    N = int(run_size)
    if out is None:
        out = torch.empty((R, rows, P) if members is not None else (R * N, P))
    for r, h in enumerate(hp_rows(hp)):
        T, E, _ = _counts(ga, r, rows)
        if members is None:
            out[r * N:(r + 1) * N] = g.ga_rows(parents[r, :T], E, sigma=h.sigma, seed=h.seed, generation=generation,
                                                member_offset=0, n_local=N)
        else:
            keep = np.flatnonzero(members[r].numpy() >= 0)
            if len(keep):
                out[r, keep] = g.ga_rows(parents[r, :T], E, sigma=h.sigma, seed=h.seed, generation=generation,
                                         members=members[r, keep].contiguous())
    return out


def ga_order_runs_workspace(n_runs, run_size, device):
    return torch.empty(0)


def ga_order_runs(fitness, ga, table_rows, *, workspace=None, out=None):
    R, rows = fitness.shape[0], int(table_rows)
    out = torch.empty((R, rows), dtype=torch.int32) if out is None else out
    for r in range(R):
        _, _, Tr = _counts(ga, r, rows)
        out[r] = -1
        out[r, :Tr] = g.ga_order(fitness[r].contiguous(), Tr)
    return out
