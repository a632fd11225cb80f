"""Oracle-backed stand-in for distributedes_b200.ops_runs with its sweep ops, on CPU tensors.  TEST-ONLY: the ops of
cpu_ops_runs, plus the three sweep ops, each the single-population stand-in of cpu_ops applied run by run with run r's
row of the table (its seed, sigma, learning rate, weight decay and action noise) at member_offset 0, which is the
contract the library's *_sweep entry points keep.  The table is the library's own: ops_sweep.run_table builds it without
a library call, and each row is read back through the ctypes mirror of des_run_hp."""
import torch

import cpu_ops as k
from cpu_ops_runs import (centered_rank_runs, grad_runs_workspace, nes_apply_runs, nes_grad_partial_runs,  # noqa: F401
                          new_state, obs_stats_merge_totals_runs, param_count, rank_runs_workspace, rollout_eval_runs,
                          state_advance)
from distributedes_b200._lib import RunHp
from distributedes_b200.ops_sweep import run_table  # noqa: F401


def hp_rows(hp):
    """The des_run_hp of every row of a uint8 [R, 40] table."""
    return [RunHp.from_buffer_copy(bytes(row.tolist())) for row in hp]


def rollout_eval_sweep(theta, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                       run_size, noiseless=False, obs_stats=None, totals_out=None, workspace=None, out=None,
                       episodes_out=None):
    R, N = theta.shape[0], int(run_size)
    out = torch.empty((R, N)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        kw = dict(hidden=hidden, horizon=horizon, repetitions=repetitions, sigma=h.sigma, clip=clip,
                  action_noise_std=h.action_noise_std, seed=h.seed, generation=generation, state=state, member_offset=0,
                  n_local=N, noiseless=noiseless, obs_stats=None if obs_stats is None else obs_stats[r],
                  totals_out=None if totals_out is None else totals_out[r])
        if noiseless:
            k.rollout_eval(theta[r], episodes_out=episodes_out.reshape(R, -1)[r], **kw)
        else:
            k.rollout_eval(theta[r], out=out[r], **kw)
    return out


def nes_grad_partial_sweep(shaped, P, hp, *, generation=0, state=None, workspace=None, out=None):
    out = torch.empty((shaped.shape[0], P)) if out is None else out
    for r, h in enumerate(hp_rows(hp)):
        k.nes_grad_partial(shaped[r], P, seed=h.seed, generation=generation, state=state, member_offset=0, out=out[r])
    return out


def nes_apply_sweep(theta, adam_m, adam_v, partial_sum, N, state, hp, *, beta1=0.9, beta2=0.999, epsilon=1e-8,
                    update_out=None, grad_out=None):
    for r, h in enumerate(hp_rows(hp)):
        k.nes_apply(theta[r], adam_m[r], adam_v[r], partial_sum[r], N, state, sigma=h.sigma,
                    learning_rate=h.learning_rate, weight_decay=h.weight_decay, beta1=beta1, beta2=beta2,
                    epsilon=epsilon, update_out=None if update_out is None else update_out[r])
