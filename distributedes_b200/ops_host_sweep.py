"""Torch-tensor front ends for the sweep entry points of host-stepped environments (include/des_b200.h, "sweeps on
host-stepped environments"): the weight rows of every run, the policy step of every run and each run's observation totals,
one launch each.  Run r's member i is row r * run_size + i and member i of a standalone population under the seed of its
row of the sweep table `hp` (ops_sweep.run_table), so each op equals, run by run, the op of ops.py it is named after at
member_offset 0.  The checks are those of ops._ptr.  ops_sweep and ops_runs list these ops.
"""
from __future__ import annotations

import torch

from ._lib import Dims
from .ops import F32, F64, U8, _launch, _mlp, _ptr, _rows

def nes_perturb_sweep(theta, hp, run_size, generation, out=None):
    """rows[R * run_size, P] from theta[R, P]: run r's rows are ops.nes_perturb(theta[r], run_size, sigma and seed of hp
    row r, generation, member_offset=0)."""
    from .ops_sweep import _hp           # ops_sweep imports this module
    pt = _ptr(theta, 'theta', F32)
    R, P, N, dev = _rows(theta, 'theta'), theta.shape[1], int(run_size), theta.device
    if out is None:
        out = torch.empty((R * N, P), dtype=F32, device=dev)
    _launch('des_nes_perturb_sweep', theta, 'theta', _ptr(out, 'out', F32, R * N * P, dev), pt, R, N, P, _hp(hp, R, dev),
            int(generation))
    return out


def policy_act_sweep(rows, obs, alive, hp, *, state_dim, hidden, action_dim, repetitions, clip, generation, run_size, t,
                     obs_stats=None, stat_part=None, out=None):
    """One environment step of every run of a sweep: run r's actions are ops.policy_act of its run_size rows of
    rows[R * run_size, P] (and of obs, alive, stat_part, out) with obs_stats[r] and the seed and action noise of hp row
    r, member_offset=0.  obs_stats is [R, 2*d0+1]; run_size 1 steps every run's test episodes."""
    from .ops_sweep import _hp           # ops_sweep imports this module
    N, dev = int(run_size), rows.device
    n = _rows(rows, 'rows')
    R = n // N if N > 0 else 0
    if N <= 0 or R * N != n:
        raise RuntimeError('rows has %d rows, not a whole number of runs of run_size %d' % (n, N))
    d0, A, reps = int(state_dim), int(action_dim), int(repetitions)
    P, mlp = _mlp(d0, int(hidden), A)
    w = 2 * d0 + 1
    if out is None:
        out = torch.empty((n, reps, A), dtype=F32, device=dev)
    _launch('des_policy_act_sweep', rows, 'rows', _ptr(out, 'out', F32, n * reps * A, dev),
            _ptr(stat_part, 'stat_part', F64, n * w, dev, True), _ptr(rows, 'rows', F32, n * P, need=mlp + ' n x P ='),
            P, _ptr(obs, 'obs', F32, n * reps * d0, dev), _ptr(alive, 'alive', U8, n * reps, dev),
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), Dims(d0, int(hidden), A, 0), reps, float(clip),
            _hp(hp, R, dev), int(generation), R, N, int(t))
    return out


def obs_parts_reduce_runs(parts, state_dim, run_size, out=None):
    """totals[R, 2*d0+1] fp64: row r is ops.obs_parts_reduce of run r's run_size rows of parts[R * run_size, 2*d0+1]."""
    w, N, pp = 2 * int(state_dim) + 1, int(run_size), _ptr(parts, 'parts', F64)
    R = parts.numel() // (w * N) if N > 0 else 0
    if N <= 0 or parts.numel() != R * N * w:
        raise RuntimeError('parts has %d entries, not a whole number of runs of %d rows of 2*d0+1 = %d'
                           % (parts.numel(), N, w))
    if out is None:
        out = torch.empty((R, w), dtype=F64, device=parts.device)
    _launch('des_obs_parts_reduce_runs', parts, 'parts', _ptr(out, 'out', F64, R * w, parts.device), pp, R, N,
            int(state_dim))
    return out
