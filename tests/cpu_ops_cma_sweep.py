"""Oracle-backed stand-in for distributedes_b200.ops_runs with the CMA-ES sweep ops, on CPU tensors.  TEST-ONLY: the ops of
cpu_ops_host_sweep, plus rollout_eval_sweep of cpu_ops_sweep and the four ops of ops_cma_sweep, each the single-run
stand-in of cpu_ops applied run by run (with run r's seed and action noise at member_offset 0 where the op reads the
table), which is the contract the library's entry points keep."""
import torch

import cpu_ops as k
from cpu_ops_host_sweep import (centered_rank_runs, hp_rows, nes_perturb_sweep, obs_parts_reduce_runs,  # noqa: F401
                                obs_stats_merge_totals_runs, param_count, policy_act_sweep, run_table)
from cpu_ops_sweep import rollout_eval_sweep  # noqa: F401


def noise_fill_sweep(hp, run_size, P, generation, stream_tag=1, out=None):
    rows = [k.noise_fill(int(run_size), int(P), h.seed, generation, 0, stream_tag) for h in hp_rows(hp)]
    res = torch.cat(rows) if rows else torch.empty((0, int(P)))
    return res if out is None else out.copy_(res)


def rollout_eval_solutions_sweep(rows, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, run_size,
                                 obs_stats=None, totals_out=None, workspace=None, out=None, episodes_out=None):
    N = int(run_size)
    R = rows.shape[0] // N
    out = torch.empty((R, N)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        k.rollout_eval_solutions(rows[r * N:(r + 1) * N], hidden=hidden, horizon=horizon, repetitions=repetitions,
                                 clip=clip, action_noise_std=h.action_noise_std, seed=h.seed, generation=generation,
                                 member_offset=0, obs_stats=None if obs_stats is None else obs_stats[r],
                                 totals_out=None if totals_out is None else totals_out[r], out=out[r])
    return out


def cma_rank_mu_runs(Y, w, out=None, workspace=None):
    R, n = Y.shape[0], Y.shape[2]
    out = torch.empty((R, n, n)) if out is None else out
    for r in range(R):
        k.cma_rank_mu(Y[r], w[r], out=out[r])
    return out


def cma_cov_apply_runs(Cmat, dC, pc, decay, *, c1, cmu):
    for r in range(Cmat.shape[0]):
        k.cma_cov_apply(Cmat[r], dC[r], pc[r], decay=float(decay[r]), c1=c1, cmu=cmu)
    return Cmat
