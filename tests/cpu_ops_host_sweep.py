"""Oracle-backed stand-in for distributedes_b200.ops_runs with the sweep ops of host-stepped environments, on CPU tensors.
TEST-ONLY: the ops of cpu_ops_sweep, plus nes_perturb_sweep, policy_act_sweep and obs_parts_reduce_runs, each the
single-population stand-in of cpu_ops applied run by run with run r's seed, sigma and action noise at member_offset 0,
which is the contract the library's entry points keep."""
import torch

import cpu_ops as k
from cpu_ops_sweep import (centered_rank_runs, grad_runs_workspace, hp_rows, nes_apply_sweep,  # noqa: F401
                           nes_grad_partial_sweep, new_state, obs_stats_merge_totals_runs, param_count,
                           rank_runs_workspace, run_table, state_advance)


def nes_perturb_sweep(theta, hp, run_size, generation, out=None):
    R, P, N = theta.shape[0], theta.shape[1], int(run_size)
    out = torch.empty((R * N, P)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        k.nes_perturb(theta[r], N, h.sigma, h.seed, generation, 0, out=out[r * N:(r + 1) * N])
    return out


def policy_act_sweep(rows, obs, alive, hp, *, state_dim, hidden, action_dim, repetitions, clip, generation, run_size, t,
                     obs_stats=None, stat_part=None, out=None):
    N, reps = int(run_size), int(repetitions)
    out = torch.empty((rows.shape[0], reps, action_dim)) if out is None else out
    obs, alive, acts = (x.reshape(rows.shape[0], -1) for x in (obs, alive, out))
    for r, h in enumerate(hp_rows(hp)):
        s = slice(r * N, (r + 1) * N)
        k.policy_act(rows[s], obs[s], alive[s], state_dim=state_dim, hidden=hidden, action_dim=action_dim,
                     repetitions=reps, clip=clip, action_noise_std=h.action_noise_std, seed=h.seed, generation=generation,
                     member_offset=0, t=t, obs_stats=None if obs_stats is None else obs_stats[r],
                     stat_part=None if stat_part is None else stat_part[s], out=acts[s])
    return out


def obs_parts_reduce_runs(parts, state_dim, run_size, out=None):
    w, N = 2 * int(state_dim) + 1, int(run_size)
    R = parts.numel() // (w * N)
    out = torch.empty((R, w), dtype=torch.float64) if out is None else out
    for r in range(R):
        k.obs_parts_reduce(parts.reshape(R * N, w)[r * N:(r + 1) * N], state_dim, out=out[r])
    return out
