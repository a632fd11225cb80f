"""Torch-tensor front ends for the run-batched entry points (include/des_b200.h, "batches of independent runs"): R
independent NES runs of N members each, one row per run in every per-run tensor.  Run r's member i is the global member
r*N + i, so run 0 is the population the ops of distributedes_b200.ops evaluate alone.  Each op equals, run by run, the op
of ops.py it is named after; the checks are those of ops._ptr.

param_count, new_state and state_advance are ops.py's, re-exported so that this module is the whole set of device ops
engine.RolloutRunsEngine calls (and a test stand-in can replace all of them at once).
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import Dims, Opt
from .ops import F32, F64, I32, STATE_BYTES, U8, _env_dims, _launch, _mlp, _ptr, _rows, _ws
from .ops import new_state, param_count, state_advance  # noqa: F401  (see the module docstring)


def _runs(t, name):
    """(R, N) of a 2-D per-run tensor t[R, N]."""
    return _rows(t, name), t.shape[1]


def rollout_eval_runs(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                      generation=0, state=None, run_size, noiseless=False, obs_stats=None, totals_out=None,
                      workspace=None, out=None, episodes_out=None):
    """Closed-loop fitness[R, run_size] of R runs from theta[R, P]: run r is ops.rollout_eval(theta[r],
    obs_stats=obs_stats[r], member_offset=r*run_size, n_local=run_size).  obs_stats and totals_out are [R, 2*d0+1];
    episodes_out [R, run_size, repetitions].  noiseless needs run_size 1: run r's test episodes."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    R, N, reps, w, dev = _rows(theta, 'theta'), int(run_size), int(repetitions), 2 * d0 + 1, theta.device
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(R * N, 1) * w, dtype=F64, device=dev)
    _launch('des_rollout_eval_runs', theta, 'theta', _ptr(out, 'out', F32, R * N, dev),
            _ptr(episodes_out, 'episodes_out', F32, R * N * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, R * w, dev, True), _ptr(theta, 'theta', F32, R * P, need=mlp + ' R x P ='),
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), int(env), Dims(d0, hidden, A, horizon), reps,
            float(sigma), float(clip), float(action_noise_std), int(seed), int(generation),
            _ptr(state, 'state', U8, STATE_BYTES, dev, True), R, N, 1 if noiseless else 0, *_ws(workspace, dev))
    return out


def obs_stats_merge_totals_runs(stats, totals, state_dim):
    """ops.obs_stats_merge_totals of every run: row r of totals[R, 2*d0+1] into row r of stats[R, 2*d0+1], in place."""
    R, w = _rows(stats, 'stats'), 2 * int(state_dim) + 1
    _launch('des_obs_stats_merge_totals_runs', stats, 'stats', _ptr(stats, 'stats', F32, R * w),
            _ptr(totals, 'totals', F64, R * w, stats.device), int(state_dim), R)
    return stats


def rank_runs_workspace(n_runs, run_size, device):
    nbytes = _lib.load().des_rank_runs_workspace_bytes(int(n_runs), int(run_size))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def centered_rank_runs(fitness, *, workspace=None, return_ranks=False, out=None):
    """ops.centered_rank within each run: shaped[R, N] of fitness[R, N]."""
    pf = _ptr(fitness, 'fitness', F32)
    (R, N), dev = _runs(fitness, 'fitness'), fitness.device
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    ranks = torch.empty((R, N), dtype=I32, device=dev) if return_ranks else None
    if workspace is None:
        workspace = rank_runs_workspace(R, N, dev)
    _launch('des_centered_rank_runs', fitness, 'fitness', _ptr(out, 'out', F32, R * N, dev),
            _ptr(ranks, 'ranks', I32, R * N, dev, True), pf, R, N, *_ws(workspace, dev))
    return (out, ranks) if return_ranks else out


def grad_runs_workspace(n_runs, run_size, P, device):
    nbytes = _lib.load().des_grad_runs_workspace_bytes(int(n_runs), int(run_size), int(P))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def nes_grad_partial_runs(shaped, P, *, seed, generation=0, state=None, workspace=None, out=None):
    """partial[R, P]: run r is ops.nes_grad_partial(shaped[r], P, member_offset=r*N) for shaped[R, N]."""
    ps = _ptr(shaped, 'shaped', F32)
    (R, N), dev = _runs(shaped, 'shaped'), shaped.device
    if out is None:
        out = torch.empty((R, P), dtype=F32, device=dev)
    if workspace is None:
        workspace = grad_runs_workspace(R, N, P, dev)
    _launch('des_nes_grad_partial_runs', shaped, 'shaped', _ptr(out, 'out', F32, R * P, dev), ps, R, N, P, seed,
            generation, _ptr(state, 'state', U8, STATE_BYTES, dev, True), *_ws(workspace, dev))
    return out


def nes_apply_runs(theta, adam_m, adam_v, partial_sum, N, state, *, sigma, learning_rate, weight_decay=0.005,
                   beta1=0.9, beta2=0.999, epsilon=1e-8, update_out=None, grad_out=None):
    """ops.nes_apply of every run, in place on theta[R, P] and the fp64 Adam moments adam_m / adam_v [R, P]; N is the run
    size.  Adam's t and beta^t in `state` are shared: advance them once per generation."""
    pt = _ptr(theta, 'theta', F32)
    (R, P), dev = _runs(theta, 'theta'), theta.device
    _launch('des_nes_apply_runs', theta, 'theta', pt, _ptr(adam_m, 'adam_m', F64, R * P, dev),
            _ptr(adam_v, 'adam_v', F64, R * P, dev), _ptr(update_out, 'update_out', F32, R * P, dev, True),
            _ptr(grad_out, 'grad_out', F64, R * P, dev, True), _ptr(partial_sum, 'partial_sum', F32, R * P, dev), P, R,
            int(N), Opt(sigma, learning_rate, weight_decay, beta1, beta2, epsilon),
            _ptr(state, 'state', U8, STATE_BYTES, dev))

# The recordings of one population (RolloutRunsEngine.record_test_episodes records one run at a time): ops.py's.
from .ops import rollout_record, rollout_record_solutions  # noqa: E402,F401
# The sweep ops (seeds and NES hyper-parameters per run): defined in ops_sweep, listed here so that this module stays the
# whole set of device ops engine.RolloutRunsEngine and engine.HostEnvSweepEngine call.
from .ops_sweep import (nes_apply_sweep, nes_grad_partial_sweep, nes_perturb_sweep, obs_parts_reduce_runs,  # noqa: E402,F401
                        policy_act_sweep, rollout_eval_sweep, run_table)
# The CMA-ES sweep ops (cma_es.CMASweep, fitness.DeviceSweep): defined in ops_cma_sweep, on the same table.
from .ops_cma_sweep import (cma_cov_apply_runs, cma_rank_mu_runs, noise_fill_sweep,  # noqa: E402,F401
                            rollout_eval_solutions_sweep)
# The genetic-algorithm sweep ops (genetic.GASweep, fitness.DeviceSweep.ga_members): defined in ops_ga_sweep, on the same
# table and a count table of their own.
from .ops_ga_sweep import (ga_order_runs, ga_order_runs_workspace, ga_rows_sweep, ga_table,  # noqa: E402,F401
                           rollout_eval_ga_sweep)
# The novelty-search sweep ops (novelty.NoveltySweep): defined in ops_novelty_sweep, on the same table and a table of
# reward weights of their own.
from .ops_novelty_sweep import (novelty_runs, ns_shape_runs, ns_shape_runs_workspace,  # noqa: E402,F401
                                ns_weight_table, rollout_eval_bc_sweep)
