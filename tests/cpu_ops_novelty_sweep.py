"""Oracle-backed stand-in for distributedes_b200.ops_runs with the novelty-search sweep ops, on CPU tensors.  TEST-ONLY:
the ops of cpu_ops_host_sweep and cpu_ops_sweep, plus the five ops of ops_novelty_sweep, each the single-run stand-in of
cpu_ops_novelty applied run by run with run r's seed, sigma and action noise (its row of the sweep table) at member_offset
0, its archive and its row of the weight table, which is the contract the library's entry points keep.  The weight
table is the library's own: ops_novelty_sweep.ns_weight_table builds it without a library call, and the blend reads its
two fp32 columns as des_ns_shape_runs does."""
import numpy as np
import torch

import cpu_ops
import cpu_ops_novelty as one
from cpu_ops_host_sweep import (centered_rank_runs, grad_runs_workspace, hp_rows, nes_apply_sweep,  # noqa: F401
                                nes_grad_partial_sweep, nes_perturb_sweep, new_state, obs_parts_reduce_runs,
                                obs_stats_merge_totals_runs, param_count, policy_act_sweep, rank_runs_workspace,
                                run_table, state_advance)
from cpu_ops_sweep import rollout_eval_sweep  # noqa: F401
from distributedes_b200.ops_novelty_sweep import ns_weight_table  # noqa: F401
from oracle import nes_oracle as orc
from oracle import novelty_oracle as no


def rollout_eval_bc_sweep(theta, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                          run_size, noiseless=False, obs_stats=None, totals_out=None, workspace=None, out=None,
                          episodes_out=None, bc_out):
    R, N = theta.shape[0], int(run_size)
    out = torch.empty((R, N)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        one.rollout_eval_bc(theta[r], hidden=hidden, horizon=horizon, repetitions=repetitions, sigma=h.sigma, clip=clip,
                            action_noise_std=h.action_noise_std, seed=h.seed, generation=generation, state=state,
                            member_offset=0, n_local=N, noiseless=noiseless,
                            obs_stats=None if obs_stats is None else obs_stats[r],
                            totals_out=None if totals_out is None else totals_out[r], out=out[r],
                            episodes_out=None if episodes_out is None else episodes_out[r], bc_out=bc_out[r])
    return out


def novelty_runs(queries, archive, k, *, size, out=None):
    out = torch.empty(queries.shape[:2]) if out is None else out
    for r in range(queries.shape[0]):
        one.novelty(queries[r], archive[r, :int(size)], k, out=out[r])
    return out


def ns_shape_runs_workspace(n_runs, run_size, device):
    return torch.empty(0)


def ns_shape_runs(fitness, novelty_, weights, *, workspace=None, out=None):
    out = torch.empty_like(fitness) if out is None else out
    for r in range(fitness.shape[0]):
        w, w1 = (np.float32(x) for x in weights[r].numpy())
        s_f = orc.fitness_shift(fitness[r].numpy()).astype(np.float32)
        s_n = orc.fitness_shift(novelty_[r].numpy()).astype(np.float32)
        cpu_ops._out(torch.from_numpy(no.fmaf32(w, s_f, (w1 * s_n).astype(np.float32))), out[r])
    return out
