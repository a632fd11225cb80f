"""Torch-tensor front ends for novelty search's entry points (include/des_b200.h, "novelty search"): des_rollout_eval_bc,
des_novelty and des_ns_shape.  Every tensor is checked in ops._ptr.  ops re-exports all of them."""
from __future__ import annotations

import torch

from . import _lib
from .ops import F32, _launch, _ptr, _rollout, _ws


def rollout_eval_bc(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                    generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None, totals_out=None,
                    workspace=None, out=None, episodes_out=None, bc_out):
    """rollout_eval (members or noiseless test episodes), bit for bit, that also writes bc_out[n_local, d0]: each member's
    raw observation after the last step of its episodes, averaged over the repetitions (des_rollout_eval_bc)."""
    return _rollout('des_rollout_eval_bc', theta, 'theta', (sigma, state, noiseless), env, hidden, horizon, repetitions,
                    clip, action_noise_std, seed, generation, member_offset, n_local, obs_stats, totals_out, workspace,
                    out, episodes_out, bc_out=bc_out)


def novelty(queries, archive, k, *, out=None):
    """novelty[n] fp32 of queries[n, d] against archive[A, d]: the mean distance to the min(k, A) nearest archive rows,
    ordered by (squared distance, row) with NaN last (des_novelty)."""
    for t, name in ((queries, 'queries'), (archive, 'archive')):
        if not isinstance(t, torch.Tensor) or t.dim() != 2:
            raise RuntimeError('%s must be a 2-D tensor [rows, d], got shape %r' % (name, tuple(getattr(t, 'shape', ()))))
    n, d, A, dev = queries.shape[0], queries.shape[1], archive.shape[0], archive.device
    pa = _ptr(archive, 'archive', F32)
    if archive.shape[1] != d:
        raise RuntimeError('archive rows have %d entries, the queries %d' % (archive.shape[1], d))
    if out is None:
        out = torch.empty(n, dtype=F32, device=dev)
    _launch('des_novelty', archive, 'archive', _ptr(out, 'out', F32, n, dev), _ptr(queries, 'queries', F32, n * d, dev),
            n, pa, A, d, int(k))
    return out


def ns_shape_workspace(N, device):
    nbytes = _lib.load().des_ns_shape_workspace_bytes(int(N))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def ns_shape(fitness, novelty_, reward_weight, *, workspace=None, out=None):
    """shaped[N] = fmaf(w, centered_rank(fitness), fp32(1 - w) * centered_rank(novelty)) in fp32 (des_ns_shape); at w = 1
    it is centered_rank(fitness), bit for bit."""
    pf = _ptr(fitness, 'fitness', F32)
    N, dev = fitness.numel(), fitness.device
    if out is None:
        out = torch.empty(N, dtype=F32, device=dev)
    if workspace is None:
        workspace = ns_shape_workspace(N, dev)
    _launch('des_ns_shape', fitness, 'fitness', _ptr(out, 'out', F32, N, dev), pf,
            _ptr(novelty_, 'novelty', F32, N, dev), N, float(reward_weight), *_ws(workspace, dev))
    return out
