"""Torch-tensor front ends for the sweep entry points (include/des_b200.h, "sweeps"): a batch of R NES runs of N members
whose seed, sigma, learning rate, weight decay and action-noise std differ per run.  The per-run values travel in a
device table, `hp` (run_table), one 40-byte des_run_hp row per run.  Run r's member i is member i of a standalone
population under run r's seed, so each op equals, run by run, the op of ops.py it is named after with run r's seed and
hyper-parameters at member_offset 0.  The checks are those of ops._ptr; the table is checked like every other tensor.

ops_runs re-exports these ops, so that it stays the one module of device ops engine.RolloutRunsEngine and
engine.HostEnvSweepEngine call.  Ranking and the statistics merge need no table: ops_runs.centered_rank_runs and
ops_runs.obs_stats_merge_totals_runs.  On host-stepped environments the rows of every run come from nes_perturb_sweep, each
environment step of every run is one policy_act_sweep, and obs_parts_reduce_runs sums each run's observation rows
(defined in ops_host_sweep, listed here).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ._lib import Dims, RunHp
from .ops import F32, F64, STATE_BYTES, U8, _env_dims, _launch, _mlp, _ptr, _rows, _ws

HP_BYTES = C.sizeof(RunHp)               # 40
_HP_DTYPE = np.dtype({'names': [n for n, _ in RunHp._fields_],
                      'formats': ['<u8', '<f8', '<f8', '<f8', '<f8'],
                      'offsets': [getattr(RunHp, n).offset for n, _ in RunHp._fields_], 'itemsize': HP_BYTES})


def per_run(value, runs, name):
    """A length-`runs` list of `value`: a scalar is repeated, a sequence (list, tuple, array) must have `runs` entries."""
    if np.ndim(value) == 0:
        return [value] * runs
    vals = value.tolist() if hasattr(value, 'tolist') else list(value)
    if len(vals) != runs:
        raise ValueError('%s has %d entries; a sweep of %d runs needs one per run (or a scalar)' % (name, len(vals), runs))
    return vals


def run_table(seeds, sigma, learning_rate, weight_decay, action_noise_std, device, runs=None):
    """The table of a sweep: uint8 [R, 40] on `device`, row r the des_run_hp of run r.  Each argument is a scalar or a
    sequence of R entries; R is `runs`, else the length of the first sequence (1 when every argument is a scalar)."""
    cols = dict(seeds=seeds, sigma=sigma, learning_rate=learning_rate, weight_decay=weight_decay,
                action_noise_std=action_noise_std)
    if runs is None:
        runs = next((np.size(v) for v in cols.values() if np.ndim(v) > 0), 1)
    R = int(runs)
    cols = {n: per_run(v, R, n) for n, v in cols.items()}
    t = np.zeros(R, dtype=_HP_DTYPE)
    t['seed'] = [int(s) & 0xFFFFFFFFFFFFFFFF for s in cols['seeds']]       # a uint64_t, as the seed of the ops
    for n in ('sigma', 'learning_rate', 'weight_decay', 'action_noise_std'):
        t[n] = [float(v) for v in cols[n]]
    return torch.from_numpy(t.view(np.uint8).reshape(R, HP_BYTES).copy()).to(device)


def _hp(hp, R, dev):
    return _ptr(hp, 'hp', U8, R * HP_BYTES, dev, need='needs one 40-byte row per run:')


def rollout_eval_sweep(theta, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                       run_size, noiseless=False, obs_stats=None, totals_out=None, workspace=None, out=None,
                       episodes_out=None):
    """Closed-loop fitness[R, run_size] of a sweep from theta[R, P]: run r is ops.rollout_eval(theta[r],
    obs_stats=obs_stats[r], seed, sigma and action_noise_std of hp row r, member_offset=0, n_local=run_size).  obs_stats
    and totals_out are [R, 2*d0+1]; episodes_out [R, run_size, repetitions].  noiseless needs run_size 1: run r's test
    episodes under its own seed."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    R, N, reps, w, dev = _rows(theta, 'theta'), int(run_size), int(repetitions), 2 * d0 + 1, theta.device
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(R * N, 1) * w, dtype=F64, device=dev)
    _launch('des_rollout_eval_sweep', theta, 'theta', _ptr(out, 'out', F32, R * N, dev),
            _ptr(episodes_out, 'episodes_out', F32, R * N * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, R * w, dev, True), _ptr(theta, 'theta', F32, R * P, need=mlp + ' R x P ='),
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), int(env), Dims(d0, hidden, A, horizon), reps,
            float(clip), _hp(hp, R, dev), int(generation), _ptr(state, 'state', U8, STATE_BYTES, dev, True), R, N,
            1 if noiseless else 0, *_ws(workspace, dev))
    return out


def nes_grad_partial_sweep(shaped, P, hp, *, generation=0, state=None, workspace=None, out=None):
    """partial[R, P]: run r is ops.nes_grad_partial(shaped[r], P, seed=hp row r's seed, member_offset=0) for
    shaped[R, N].  The workspace is ops_runs.grad_runs_workspace's."""
    from .ops_runs import grad_runs_workspace        # ops_runs imports this module
    ps = _ptr(shaped, 'shaped', F32)
    R, N, dev = _rows(shaped, 'shaped'), shaped.shape[1], shaped.device
    if out is None:
        out = torch.empty((R, P), dtype=F32, device=dev)
    if workspace is None:
        workspace = grad_runs_workspace(R, N, P, dev)
    _launch('des_nes_grad_partial_sweep', shaped, 'shaped', _ptr(out, 'out', F32, R * P, dev), ps, R, N, P,
            _hp(hp, R, dev), generation, _ptr(state, 'state', U8, STATE_BYTES, dev, True), *_ws(workspace, dev))
    return out


def nes_apply_sweep(theta, adam_m, adam_v, partial_sum, N, state, hp, *, beta1=0.9, beta2=0.999, epsilon=1e-8,
                    update_out=None, grad_out=None):
    """ops.nes_apply of every run with hp row r's sigma, learning rate and weight decay, in place on theta[R, P] and the
    fp64 Adam moments adam_m / adam_v [R, P]; N is the run size.  beta1, beta2, epsilon and Adam's t and beta^t in
    `state` are shared: advance them once per generation."""
    pt = _ptr(theta, 'theta', F32)
    R, P, dev = _rows(theta, 'theta'), theta.shape[1], theta.device
    _launch('des_nes_apply_sweep', theta, 'theta', pt, _ptr(adam_m, 'adam_m', F64, R * P, dev),
            _ptr(adam_v, 'adam_v', F64, R * P, dev), _ptr(update_out, 'update_out', F32, R * P, dev, True),
            _ptr(grad_out, 'grad_out', F64, R * P, dev, True), _ptr(partial_sum, 'partial_sum', F32, R * P, dev), P, R,
            int(N), _hp(hp, R, dev), float(beta1), float(beta2), float(epsilon),
            _ptr(state, 'state', U8, STATE_BYTES, dev))


# The sweep ops of host-stepped environments (engine.HostEnvSweepEngine) live in ops_host_sweep, on the same table.
from .ops_host_sweep import nes_perturb_sweep, obs_parts_reduce_runs, policy_act_sweep  # noqa: E402,F401
