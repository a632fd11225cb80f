"""Torch-tensor front ends for the genetic algorithm's novelty search (include/des_b200.h, "novelty search for the genetic
algorithm"): des_rollout_eval_ga_bc and des_ns_ga_order.  Every tensor is checked in ops._ptr.  ops re-exports all of
them."""
from __future__ import annotations

import torch

from . import _lib
from .ops import F32, I32, _launch, _ptr, _ws
from .ops_ga import _rollout_ga


def rollout_eval_ga_bc(parents, n_elites, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip,
                       action_noise_std=0.0, seed, generation=0, state=None, member_offset=0, n_local, obs_stats=None,
                       totals_out=None, workspace=None, out=None, episodes_out=None, bc_out):
    """rollout_eval_ga, bit for bit, that also writes bc_out[n_local, d0]: each member's raw observation after the last
    step of its episodes, averaged over the repetitions (des_rollout_eval_ga_bc)."""
    _ptr(bc_out, 'bc_out', F32)          # required: None would launch without it
    return _rollout_ga('des_rollout_eval_ga_bc', parents, n_elites, env, hidden, horizon, repetitions, sigma, clip,
                       action_noise_std, seed, generation, state, member_offset, n_local, obs_stats, totals_out,
                       workspace, out, episodes_out, bc_out=bc_out)


def ns_ga_order_workspace(N, device):
    nbytes = _lib.load().des_ns_ga_order_workspace_bytes(int(N))
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def ns_ga_order(fitness, novelty_, reward_weight, truncation, *, workspace=None, out=None):
    """order[truncation] int32: the members of the `truncation` smallest keys fmaf(w, centered_rank(-fitness),
    fp32(1 - w) * centered_rank(-novelty)), ties to the lower index (des_ns_ga_order).  At w = 1 it is ga_order(fitness),
    bit for bit; at w = 0 the most novel come first."""
    pf = _ptr(fitness, 'fitness', F32)
    N, T, dev = fitness.numel(), int(truncation), fitness.device
    if out is None:
        out = torch.empty(max(T, 0), dtype=I32, device=dev)
    if workspace is None:
        workspace = ns_ga_order_workspace(N, dev)
    _launch('des_ns_ga_order', fitness, 'fitness', _ptr(out, 'out', I32, T, dev), pf,
            _ptr(novelty_, 'novelty', F32, N, dev), N, T, float(reward_weight), *_ws(workspace, dev))
    return out
