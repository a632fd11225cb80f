"""Torch-tensor front ends for the recordings of closed-loop episodes (include/des_b200.h, "recorded episodes"):
des_rollout_record and des_rollout_record_solutions, launched through ops._rollout, the launcher of the evaluations they
record, so every tensor is checked in ops._ptr.  ops re-exports both."""
from __future__ import annotations

from .ops import _rollout, _rows


def rollout_record(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                   generation=0, state=None, member_offset=0, n_local, noiseless=False, mirrored=False, obs_stats=None,
                   totals_out=None, workspace=None, out=None, episodes_out=None, states_out=None, obs_out=None,
                   actions_out=None, rewards_out=None):
    """rollout_eval (rollout_eval_mirrored when `mirrored`) with the same outputs, bit for bit, that also records every
    step of every episode (des_rollout_record): states_out fp64 [n_local, repetitions, horizon, 2] (th, thdot before the
    step), obs_out fp32 [.., d0] (the raw observation), actions_out fp32 [.., A] (after noise and the clip, before the
    environment's clamp) and rewards_out fp64 [n_local, repetitions, horizon].  Each is optional."""
    return _rollout('des_rollout_record', theta, 'theta', (sigma, state, noiseless), env, hidden, horizon, repetitions,
                    clip, action_noise_std, seed, generation, member_offset, n_local, obs_stats, totals_out, workspace,
                    out, episodes_out, (mirrored, states_out, obs_out, actions_out, rewards_out))


def rollout_record_solutions(solutions, *, env=0, hidden, horizon=200, repetitions=10, clip, action_noise_std=0.0, seed,
                             generation=0, member_offset=0, obs_stats=None, totals_out=None, workspace=None, out=None,
                             episodes_out=None, states_out=None, obs_out=None, actions_out=None, rewards_out=None):
    """rollout_eval_solutions with the same outputs, bit for bit, and the trajectories of rollout_record
    (des_rollout_record_solutions)."""
    return _rollout('des_rollout_record_solutions', solutions, 'solutions', None, env, hidden, horizon, repetitions, clip,
                    action_noise_std, seed, generation, member_offset, _rows(solutions, 'solutions'), obs_stats,
                    totals_out, workspace, out, episodes_out, (False, states_out, obs_out, actions_out, rewards_out))
