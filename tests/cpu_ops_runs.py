"""Oracle-backed stand-in for distributedes_b200.ops_runs on CPU tensors.  TEST-ONLY: every run-batched op is the
single-population stand-in of cpu_ops applied run by run, at member_offset r * run_size, which is the contract the
library's *_runs entry points keep."""
import torch

import cpu_ops as k
from cpu_ops import new_state, param_count, state_advance  # noqa: F401


def rank_runs_workspace(n_runs, run_size, device):
    return torch.empty(0)


def grad_runs_workspace(n_runs, run_size, P, device):
    return torch.empty(0)


def rollout_eval_runs(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                      generation=0, state=None, run_size, noiseless=False, obs_stats=None, totals_out=None,
                      workspace=None, out=None, episodes_out=None):
    R, N = theta.shape[0], int(run_size)
    out = torch.empty((R, N)) if out is None else out
    for r in range(R):
        kw = dict(hidden=hidden, horizon=horizon, repetitions=repetitions, sigma=sigma, clip=clip,
                  action_noise_std=action_noise_std, seed=seed, generation=generation, state=state,
                  member_offset=r * N, n_local=N, noiseless=noiseless,
                  obs_stats=None if obs_stats is None else obs_stats[r],
                  totals_out=None if totals_out is None else totals_out[r])
        if noiseless:
            k.rollout_eval(theta[r], episodes_out=episodes_out.reshape(R, -1)[r], **kw)
        else:
            k.rollout_eval(theta[r], out=out[r], **kw)
    return out


def centered_rank_runs(fitness, *, workspace=None, return_ranks=False, out=None):
    out = torch.empty_like(fitness) if out is None else out
    for r in range(fitness.shape[0]):
        k.centered_rank(fitness[r], 0, fitness.shape[1], out=out[r])
    return out


def nes_grad_partial_runs(shaped, P, *, seed, generation=0, state=None, workspace=None, out=None):
    R, N = shaped.shape
    out = torch.empty((R, P)) if out is None else out
    for r in range(R):
        k.nes_grad_partial(shaped[r], P, seed=seed, generation=generation, state=state, member_offset=r * N, out=out[r])
    return out


def nes_apply_runs(theta, adam_m, adam_v, partial_sum, N, state, *, sigma, learning_rate, weight_decay=0.005,
                   beta1=0.9, beta2=0.999, epsilon=1e-8, update_out=None, grad_out=None):
    for r in range(theta.shape[0]):
        k.nes_apply(theta[r], adam_m[r], adam_v[r], partial_sum[r], N, state, sigma=sigma, learning_rate=learning_rate,
                    weight_decay=weight_decay, beta1=beta1, beta2=beta2, epsilon=epsilon,
                    update_out=None if update_out is None else update_out[r])


def obs_stats_merge_totals_runs(stats, totals, state_dim):
    for r in range(stats.shape[0]):
        k.obs_stats_merge_totals(stats[r], totals[r], state_dim)
    return stats
