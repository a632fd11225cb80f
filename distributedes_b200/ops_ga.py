"""Torch-tensor front ends for the genetic algorithm's entry points (include/des_b200.h, "genetic algorithm"):
des_ga_rows, des_rollout_eval_ga and des_ga_order.  Every tensor is checked in ops._ptr.  ops re-exports all three."""
from __future__ import annotations

import torch

from . import _lib
from .ops import F32, F64, I32, STATE_BYTES, U8, Dims, _env_dims, _launch, _mlp, _ptr, _rows, _ws


def _table(parents, n_elites):
    """(n_parents, P, n_elites) of a parents table [n_parents, P]."""
    return _rows(parents, 'parents'), (parents.shape[1] if parents.dim() == 2 else 0), int(n_elites)


def ga_rows(parents, n_elites, *, sigma, seed, generation, member_offset=0, n_local=None, members=None, out=None):
    """rows[n_local, P] of a generation whose table is parents[n_parents, P] with n_elites elites: row i is member
    members[i] (an int32 tensor on the device) or member_offset + i, an elite's parent row as it is or a parent row plus
    sigma*eps of the member (des_ga_rows).  With `members` n_local is its length.  `out` may not overlap `parents`."""
    n_parents, P, n_elites = _table(parents, n_elites)
    dev = parents.device
    pm = _ptr(members, 'members', I32, None, dev, True)
    if members is not None:
        n_local = members.numel()
    elif n_local is None:
        raise RuntimeError('ga_rows: give n_local or members')
    n_local = int(n_local)
    if out is None:
        out = torch.empty((n_local, P), dtype=F32, device=dev)
    _launch('des_ga_rows', parents, 'parents', _ptr(out, 'out', F32, n_local * P, dev), _ptr(parents, 'parents', F32),
            n_parents, n_elites, P, float(sigma), int(seed), int(generation), int(member_offset), n_local, pm)
    return out


def rollout_eval_ga(parents, n_elites, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0,
                    seed, generation=0, state=None, member_offset=0, n_local, obs_stats=None, totals_out=None,
                    workspace=None, out=None, episodes_out=None):
    """Closed-loop fitness of members [member_offset, member_offset + n_local) of the generation whose table is
    parents[n_parents, P] (des_rollout_eval_ga): rollout_eval_solutions of ga_rows' rows, bit for bit, with no rows in
    memory."""
    return _rollout_ga('des_rollout_eval_ga', parents, n_elites, env, hidden, horizon, repetitions, sigma, clip,
                       action_noise_std, seed, generation, state, member_offset, n_local, obs_stats, totals_out,
                       workspace, out, episodes_out)


def _rollout_ga(fn, parents, n_elites, env, hidden, horizon, repetitions, sigma, clip, action_noise_std, seed,
                generation, state, member_offset, n_local, obs_stats, totals_out, workspace, out, episodes_out,
                bc_out=None):
    """The launch of rollout_eval_ga, and with `bc_out` [n_local, d0] that of rollout_eval_ga_bc (ops_ga_novelty)."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    n_parents, _, n_elites = _table(parents, n_elites)
    n_local, reps, w, dev = int(n_local), int(repetitions), 2 * d0 + 1, parents.device
    if out is None:
        out = torch.empty(n_local, dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(n_local, 1) * w, dtype=F64, device=dev)
    bc = () if bc_out is None else (_ptr(bc_out, 'bc_out', F32, n_local * d0, dev),)
    _launch(fn, parents, 'parents', _ptr(out, 'out', F32, n_local, dev),
            _ptr(episodes_out, 'episodes_out', F32, n_local * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, w, dev, True),
            _ptr(parents, 'parents', F32, n_parents * P, need=mlp + ' n_parents x P ='), n_parents, n_elites,
            _ptr(obs_stats, 'obs_stats', F32, w, dev, True), int(env), Dims(d0, hidden, A, horizon), reps, float(sigma),
            float(clip), float(action_noise_std), int(seed), int(generation),
            _ptr(state, 'state', U8, STATE_BYTES, dev, True), int(member_offset), n_local, 0, *bc, *_ws(workspace, dev))
    return out


def ga_order_workspace(N, device):
    nbytes = _lib.load().des_ga_order_workspace_bytes(int(N))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def ga_order(fitness, truncation, *, workspace=None, out=None):
    """order[truncation] int32: the members of the `truncation` best fitness values, best first; ties to the lower
    index, NaN last, -0 == +0 (des_ga_order)."""
    pf = _ptr(fitness, 'fitness', F32)
    N, T, dev = fitness.numel(), int(truncation), fitness.device
    if out is None:
        out = torch.empty(max(T, 0), dtype=I32, device=dev)
    if workspace is None:
        workspace = ga_order_workspace(N, dev)
    _launch('des_ga_order', fitness, 'fitness', _ptr(out, 'out', I32, T, dev), pf, N, T, *_ws(workspace, dev))
    return out
