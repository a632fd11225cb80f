"""Torch-tensor front ends for the novelty-search sweep entry points (include/des_b200.h, "novelty-search sweeps"): R
runs of N members whose seeds and NES hyper-parameters are rows of the sweep table `hp` (ops_sweep.run_table), each run
with its own archive and reward weight.  The weights travel in a second device table, `weights` (ns_weight_table: fp32
[R, 2], row r = (fp32(w_r), fp32(1 - w_r))).  Each op equals, run by run, the op of ops_novelty it is named after; the
checks are those of ops._ptr.  novelty.NoveltySweep calls these through ops_runs, which re-exports them."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import Dims
from .ops import F32, F64, STATE_BYTES, U8, _env_dims, _launch, _mlp, _ptr, _rows, _ws
from .ops_sweep import _hp


def rollout_eval_bc_sweep(theta, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                          run_size, noiseless=False, obs_stats=None, totals_out=None, workspace=None, out=None,
                          episodes_out=None, bc_out):
    """ops_sweep.rollout_eval_sweep, bit for bit, that also writes bc_out[R, run_size, d0]: run r's rows are
    ops_novelty.rollout_eval_bc(theta[r], obs_stats=obs_stats[r], seed, sigma and action_noise_std of hp row r,
    member_offset=0, n_local=run_size) (des_rollout_eval_bc_sweep).  noiseless needs run_size 1: run r's test episodes."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    R, N, reps, w, dev = _rows(theta, 'theta'), int(run_size), int(repetitions), 2 * d0 + 1, theta.device
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(R * N, 1) * w, dtype=F64, device=dev)
    _launch('des_rollout_eval_bc_sweep', theta, 'theta', _ptr(out, 'out', F32, R * N, dev),
            _ptr(episodes_out, 'episodes_out', F32, R * N * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, R * w, dev, True), _ptr(theta, 'theta', F32, R * P, need=mlp + ' R x P ='),
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), int(env), Dims(d0, hidden, A, horizon), reps,
            float(clip), _hp(hp, R, dev), int(generation), _ptr(state, 'state', U8, STATE_BYTES, dev, True), R, N,
            1 if noiseless else 0, _ptr(bc_out, 'bc_out', F32, R * N * d0, dev), *_ws(workspace, dev))
    return out


def novelty_runs(queries, archive, k, *, size, out=None):
    """novelty[R, n] fp32 of queries[R, n, d] against the first `size` rows of each run's archive[R, capacity, d]: run r's
    row is ops_novelty.novelty(queries[r], archive[r, :size], k) (des_novelty_runs).  Rows at `size` and above are not
    read."""
    for t, name in ((queries, 'queries'), (archive, 'archive')):
        if not isinstance(t, torch.Tensor) or t.dim() != 3:
            raise RuntimeError('%s must be a 3-D tensor [R, rows, d], got shape %r'
                               % (name, tuple(getattr(t, 'shape', ()))))
    R, n, d = (int(x) for x in queries.shape)
    capacity, dev = int(archive.shape[1]), archive.device
    pa = _ptr(archive, 'archive', F32)
    if tuple(archive.shape[::2]) != (R, d):
        raise RuntimeError('archive is [%d, %d, %d]; the queries [%d, %d, %d] need [%d, capacity, %d]'
                           % (*archive.shape, R, n, d, R, d))
    if out is None:
        out = torch.empty((R, n), dtype=F32, device=dev)
    _launch('des_novelty_runs', archive, 'archive', _ptr(out, 'out', F32, R * n, dev),
            _ptr(queries, 'queries', F32, R * n * d, dev), R, n, pa, capacity, int(size), d, int(k))
    return out


def ns_weight_table(weights, device):
    """The reward-weight table of a sweep: fp32 [R, 2] on `device`, row r = (fp32(w_r), fp32(1 - w_r)) with 1 - w_r
    computed in fp64, as des_ns_shape converts its weight.  The library cannot read it, so the weights are checked here:
    each in [0, 1], or ValueError."""
    t = np.zeros((len(weights), 2), dtype=np.float32)
    for r, w in enumerate(weights):
        w = float(w)
        if not 0.0 <= w <= 1.0:
            raise ValueError('ns_weight_table: run %d has reward weight %r, not in [0, 1]' % (r, w))
        t[r] = (np.float32(w), np.float32(1.0 - w))
    return torch.from_numpy(t).to(device)


def ns_shape_runs_workspace(n_runs, run_size, device):
    nbytes = _lib.load().des_ns_shape_runs_workspace_bytes(int(n_runs), int(run_size))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def ns_shape_runs(fitness, novelty_, weights, *, workspace=None, out=None):
    """shaped[R, N]: run r's row is ops_novelty.ns_shape(fitness[r], novelty_[r], w_r), w_r row r of the weight table
    `weights` (ns_weight_table); at w_r = 1 it is ops_runs.centered_rank_runs' row r, bit for bit (des_ns_shape_runs)."""
    pf = _ptr(fitness, 'fitness', F32)
    R, dev = _rows(fitness, 'fitness'), fitness.device
    N = int(fitness.shape[1])
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if workspace is None:
        workspace = ns_shape_runs_workspace(R, N, dev)
    _launch('des_ns_shape_runs', fitness, 'fitness', _ptr(out, 'out', F32, R * N, dev), pf,
            _ptr(novelty_, 'novelty', F32, R * N, dev), R, N,
            _ptr(weights, 'weights', F32, 2 * R, dev, need='needs one row (w, 1 - w) per run:'), *_ws(workspace, dev))
    return out
