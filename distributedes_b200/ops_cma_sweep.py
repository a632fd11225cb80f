"""Torch-tensor front ends for the CMA-ES sweep entry points (include/des_b200.h, "CMA-ES sweeps"): the normals z of every
run, the closed-loop evaluation of every run's solutions, and the rank-mu partial and covariance update of every run, one
launch each (the rank-mu partial once per run from n = 2048, on the tensor cores).  Run r's member i is row
r * run_size + i and member i of a standalone population under the seed of its row of the sweep table `hp`
(ops_sweep.run_table), so each op equals, run by run, the op of ops.py it is named after at member_offset 0.  The checks
are those of ops._ptr.  cma_es.CMASweep and fitness.DeviceSweep call these through ops_runs.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import Dims
from .ops import F32, F64, _env_dims, _launch, _mlp, _ptr, _rows, _ws
from .ops_sweep import _hp

_RANK_MU_WS = {}      # (device, R, lambda, n) -> workspace tensor of des_cma_rank_mu_runs (tensor-core shapes only)


def noise_fill_sweep(hp, run_size, P, generation, stream_tag=1, out=None):
    """z[R * run_size, P] fp32: run r's rows are ops.noise_fill(run_size, P, seed of hp row r, generation,
    member_offset=0, stream_tag).  CMA-ES's z of every run (stream 1)."""
    R, N, dev = _rows(hp, 'hp'), int(run_size), hp.device
    if out is None:
        out = torch.empty((R * N, int(P)), dtype=F32, device=dev)
    _launch('des_noise_fill_sweep', hp, 'hp', _ptr(out, 'out', F32, R * N * int(P), dev), R, N, int(P), _hp(hp, R, dev),
            int(generation), int(stream_tag))
    return out


def rollout_eval_solutions_sweep(rows, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, run_size,
                                 obs_stats=None, totals_out=None, workspace=None, out=None, episodes_out=None):
    """Closed-loop fitness[R, run_size] of every run's solutions rows[R * run_size, P]: run r is
    ops.rollout_eval_solutions(its run_size rows, obs_stats=obs_stats[r], seed and action_noise_std of hp row r,
    member_offset=0).  obs_stats and totals_out are [R, 2*d0+1]; episodes_out [R, run_size, repetitions]."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    n, N, reps, w, dev = _rows(rows, 'rows'), int(run_size), int(repetitions), 2 * d0 + 1, rows.device
    R = n // N if N > 0 else 0
    if N <= 0 or R * N != n:
        raise RuntimeError('rows has %d rows, not a whole number of runs of run_size %d' % (n, N))
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(n, 1) * w, dtype=F64, device=dev)
    _launch('des_rollout_eval_solutions_sweep', rows, 'rows', _ptr(out, 'out', F32, n, dev),
            _ptr(episodes_out, 'episodes_out', F32, n * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, R * w, dev, True), _ptr(rows, 'rows', F32, n * P, need=mlp + ' n x P ='),
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), int(env), Dims(d0, int(hidden), A, int(horizon)), reps,
            float(clip), _hp(hp, R, dev), int(generation), R, N, *_ws(workspace, dev))
    return out


def cma_rank_mu_runs_workspace(R, lam, n, device):
    """The workspace des_cma_rank_mu_runs needs (empty below n = 2048), cached per shape and device."""
    key = (str(device), int(R), int(lam), int(n))
    ws = _RANK_MU_WS.get(key)
    if ws is None:
        nbytes = int(_lib.load().des_cma_rank_mu_runs_workspace_bytes(int(R), int(lam), int(n)))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        if len(_RANK_MU_WS) > 8:
            _RANK_MU_WS.clear()
        _RANK_MU_WS[key] = ws
    return ws


def cma_rank_mu_runs(Y, w, out=None, workspace=None):
    """dC[R, n, n]: run r's is ops.cma_rank_mu(Y[r], w[r]) for Y[R, lambda, n] and w[R, lambda]."""
    if not isinstance(Y, torch.Tensor) or Y.dim() != 3:
        raise RuntimeError('Y must be a 3-D tensor [R, lambda, n], got shape %r' % (tuple(getattr(Y, 'shape', ())),))
    py = _ptr(Y, 'Y', F32)
    (R, lam, n), dev = Y.shape, Y.device
    if out is None:
        out = torch.empty((R, n, n), dtype=F32, device=dev)
    if workspace is None and dev.type == 'cuda':
        workspace = cma_rank_mu_runs_workspace(R, lam, n, dev)
    _launch('des_cma_rank_mu_runs', Y, 'Y', _ptr(out, 'out', F32, R * n * n, dev), py, _ptr(w, 'w', F32, R * lam, dev), R,
            lam, n, *_ws(workspace, dev))
    return out


def cma_cov_apply_runs(Cmat, dC, pc, decay, *, c1, cmu):
    """ops.cma_cov_apply of every run, in place on Cmat[R, n, n]: dC [R, n, n], pc [R, n] (or None), decay [R] fp64 on
    the device (one per run: hsig differs), c1 and cmu shared."""
    if not isinstance(Cmat, torch.Tensor) or Cmat.dim() != 3:
        raise RuntimeError('Cmat must be a 3-D tensor [R, n, n], got shape %r' % (tuple(getattr(Cmat, 'shape', ())),))
    pC = _ptr(Cmat, 'Cmat', F32)
    R, n, dev = Cmat.shape[0], Cmat.shape[1], Cmat.device
    if Cmat.shape[2] != n:
        raise RuntimeError('Cmat must be [R, n, n], got shape %r' % (tuple(Cmat.shape),))
    _launch('des_cma_cov_apply_runs', Cmat, 'Cmat', pC, _ptr(dC, 'dC', F32, R * n * n, dev),
            _ptr(pc, 'pc', F32, R * n, dev, True), _ptr(decay, 'decay', F64, R, dev), float(c1), float(cmu), R, n)
    return Cmat
