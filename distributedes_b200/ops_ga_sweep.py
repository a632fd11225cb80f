"""Torch-tensor front ends for the genetic-algorithm sweep entry points (include/des_b200.h, "genetic-algorithm sweeps"):
R runs of N members whose seed, mutation power and action noise are rows of the sweep table `hp` (ops_sweep.run_table)
and whose parents tables share one buffer parents[R, table_rows, P].  Each run's current n_parents and n_elites, and its
truncation, are rows of a second device table, `ga` (ga_table: int32 [R, 4], one 16-byte des_ga_run row per run).  Run
r's member i is member i of a standalone population under its own seed at member_offset 0, so each op equals, run by
run, the op of ops_ga it is named after.  The checks are those of ops._ptr.  genetic.GASweep and fitness.DeviceSweep
call these through ops_runs.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import Dims
from .ops import F32, F64, I32, STATE_BYTES, U8, _env_dims, _launch, _mlp, _ptr, _rows, _ws
from .ops_sweep import _hp

GA_COLS = 4                   # des_ga_run: n_parents, n_elites, truncation, pad (int32 each)


def ga_table(n_parents, n_elites, truncation, table_rows, device):
    """The count table of a GA sweep: int32 [R, 4] on `device`, row r the des_ga_run (n_parents[r], n_elites[r],
    truncation[r], 0).  The library cannot read it, so the counts are checked here: 1 <= n_parents <= table_rows,
    0 <= n_elites <= n_parents and 1 <= truncation <= table_rows, or ValueError."""
    rows = np.zeros((len(n_parents), GA_COLS), dtype=np.int32)
    for r, (T, E, Tr) in enumerate(zip(n_parents, n_elites, truncation)):
        T, E, Tr = int(T), int(E), int(Tr)
        if not 1 <= T <= table_rows:
            raise ValueError('ga_table: run %d has n_parents %d, not in [1, table_rows = %d]' % (r, T, table_rows))
        if not 0 <= E <= T:
            raise ValueError('ga_table: run %d has n_elites %d, not in [0, n_parents = %d]' % (r, E, T))
        if not 1 <= Tr <= table_rows:
            raise ValueError('ga_table: run %d has truncation %d, not in [1, table_rows = %d]' % (r, Tr, table_rows))
        rows[r, :3] = (T, E, Tr)
    return torch.from_numpy(rows).to(device)


def _tables(parents):
    """(R, table_rows, P) of the parents buffer [R, table_rows, P]."""
    if not isinstance(parents, torch.Tensor) or parents.dim() != 3:
        raise RuntimeError('parents must be a 3-D tensor [R, table_rows, P], got shape %r'
                           % (tuple(getattr(parents, 'shape', ())),))
    return tuple(int(x) for x in parents.shape)


def _ga(ga, R, dev):
    return _ptr(ga, 'ga', I32, R * GA_COLS, dev, need='needs one 16-byte row per run:')


def rollout_eval_ga_sweep(parents, ga, hp, *, env=0, hidden, horizon=200, repetitions=10, clip, generation=0, state=None,
                          run_size, obs_stats=None, totals_out=None, workspace=None, out=None, episodes_out=None):
    """Closed-loop fitness[R, run_size] of every run's generation: run r is ops.rollout_eval_ga(its table
    parents[r, :n_parents_r], n_elites_r, obs_stats=obs_stats[r], seed, sigma and action_noise_std of hp row r,
    member_offset=0, n_local=run_size).  obs_stats and totals_out are [R, 2*d0+1]; episodes_out [R, run_size,
    repetitions]."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    R, rows, _ = _tables(parents)
    N, reps, w, dev = int(run_size), int(repetitions), 2 * d0 + 1, parents.device
    if out is None:
        out = torch.empty((R, N), dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(R * N, 1) * w, dtype=F64, device=dev)
    _launch('des_rollout_eval_ga_sweep', parents, 'parents', _ptr(out, 'out', F32, R * N, dev),
            _ptr(episodes_out, 'episodes_out', F32, R * N * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, R * w, dev, True),
            _ptr(parents, 'parents', F32, R * rows * P, need=mlp + ' R x table_rows x P ='), _ga(ga, R, dev), rows,
            _ptr(obs_stats, 'obs_stats', F32, R * w, dev, True), int(env), Dims(d0, int(hidden), A, int(horizon)), reps,
            float(clip), _hp(hp, R, dev), int(generation), _ptr(state, 'state', U8, STATE_BYTES, dev, True), R, N,
            *_ws(workspace, dev))
    return out


def ga_rows_sweep(parents, ga, hp, *, generation, run_size, members=None, out=None):
    """Rows mode (members None): rows[R * run_size, P], run r's rows ops.ga_rows(its table, n_elites_r, sigma and seed
    of hp row r, member_offset=0, n_local=run_size).  Gather mode: members int32 [R, table_rows] (-1: none), out
    [R, table_rows, P], row (r, k) the weights of member members[r, k] of run r; rows of -1 are not written.  `out` may
    not overlap `parents`."""
    R, rows, P = _tables(parents)
    N, dev = int(run_size), parents.device
    pm = _ptr(members, 'members', I32, R * rows, dev, True)
    n = R * rows if members is not None else R * N
    if out is None:
        out = torch.empty((R, rows, P) if members is not None else (R * N, P), dtype=F32, device=dev)
    _launch('des_ga_rows_sweep', parents, 'parents', _ptr(out, 'out', F32, n * P, dev), _ptr(parents, 'parents', F32),
            _ga(ga, R, dev), rows, P, _hp(hp, R, dev), int(generation), R, N, pm)
    return out


def ga_order_runs_workspace(n_runs, run_size, device):
    nbytes = _lib.load().des_ga_order_runs_workspace_bytes(int(n_runs), int(run_size))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def ga_order_runs(fitness, ga, table_rows, *, workspace=None, out=None):
    """order[R, table_rows] int32 of fitness[R, N]: run r's first truncation_r entries are ops.ga_order(fitness[r],
    truncation_r), the rest -1."""
    pf = _ptr(fitness, 'fitness', F32)
    R, dev = _rows(fitness, 'fitness'), fitness.device
    N, rows = fitness.shape[1], int(table_rows)
    if out is None:
        out = torch.empty((R, max(rows, 0)), dtype=I32, device=dev)
    if workspace is None:
        workspace = ga_order_runs_workspace(R, N, dev)
    _launch('des_ga_order_runs', fitness, 'fitness', _ptr(out, 'out', I32, R * rows, dev), pf, _ga(ga, R, dev), rows, R, N,
            *_ws(workspace, dev))
    return out
