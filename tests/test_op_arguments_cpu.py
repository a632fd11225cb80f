"""The entry points of libdes_b200 see raw pointers, never allocation sizes: ops checks every tensor an op passes them
(dtype, contiguity, element count, device) before it enters the device, and only then rejects a CPU tensor.  So on the
CPU a valid call reaches that last check, and each broken argument is reported by name before it."""
import inspect
import re

import pytest
import torch

from distributedes_b200 import ops
from lib_fixture import lib  # noqa: F401

# ops that take no caller tensor
EXEMPT = {
    'param_count': 'integers in, an integer out',
    'new_state': 'allocates its own state tensor',
    'read_state': 'copies the state to the host; no pointer reaches the library',
    'noise_fill': 'allocates its own output',
    'rank_workspace': 'a size query and an allocation',
    'grad_workspace': 'a size query and an allocation',
    'eval_workspace': 'a size query and an allocation',
    'cma_packed_elems': 'integers in, an integer out',
}

# how an argument's element count is fixed
COUNT = 'count'         # by the other arguments: one entry short or long is an error
ROW = 'row'             # a table [n, P] whose row length P is fixed: one entry short or long per row
TAPE = 'tape'           # obs[T, d0] / target[T, A]: one row short or long is an error
MULTIPLE = 'multiple'   # a multiple of 2*d0+1: one entry short is an error
FREE = 'free'           # the argument fixes the op's shape itself
WORKSPACE = 'workspace'  # any dtype; the library judges its size

d0, H, A, T, N, REPS = 3, 16, 1, 8, 4, 2         # the tape and Pendulum-v0 (d0 = 3, A = 1) at H = 16
W = 2 * d0 + 1


def z(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype)


def _table():
    """op -> (its non-tensor arguments, {tensor argument: (tensor, kind)} with the anchor first) of one valid call."""
    P, K = ops.param_count(d0, H, A), ops.cma_packed_elems(6)
    state = (z(32, dtype=torch.uint8), COUNT)
    tape = dict(obs=(z(T, d0), TAPE), target=(z(T, A), TAPE))
    closed = dict(obs_stats=(z(W), COUNT), totals_out=(z(W, dtype=torch.float64), COUNT),
                  workspace=(z(N * W, dtype=torch.float64), WORKSPACE), out=(z(N), COUNT), episodes_out=(z(N, REPS), COUNT))
    noisy = dict(hidden=H, repetitions=REPS, sigma=0.1, clip=2.0, seed=0, n_local=N)
    perturb = (dict(n_members=N, sigma=0.1, seed=0, generation=0), dict(theta=(z(P), FREE), out=(z(N, P), COUNT)))
    nes_eval = (dict(hidden=H, sigma=0.1, clip=1.0, seed=0, n_local=N),
                dict(theta=(z(P), COUNT), **tape, state=state, out=(z(N), COUNT),
                     workspace=(z(16, dtype=torch.uint8), WORKSPACE)))
    grad = (dict(P=P, seed=0), dict(shaped_local=(z(N), FREE), state=state, out=(z(P), COUNT),
                                    workspace=(z(64, dtype=torch.uint8), WORKSPACE)))
    Y = dict(Y=(z(5, 6), FREE), w=(z(5), COUNT))
    cov = dict(decay=0.9, c1=0.1, cmu=0.1)
    return {
        'state_advance': ({}, dict(state=state)),
        'nes_perturb': perturb,
        'nes_perturb_mirrored': perturb,
        'obs_stats_merge': (dict(n_feed=1.0), dict(obs=(z(T, d0), FREE), stats=(z(W), COUNT))),
        'obs_normalize': ({}, dict(obs=(z(T, d0), FREE), stats=(z(W), COUNT), out=(z(T, d0), COUNT))),
        'rollout_eval': (noisy, dict(theta=(z(P), COUNT), state=state, **closed)),
        'rollout_eval_mirrored': (noisy, dict(theta=(z(P), COUNT), state=state, **closed)),
        'rollout_eval_solutions': (dict(hidden=H, repetitions=REPS, clip=2.0, seed=0),
                                   dict(solutions=(z(N, P), ROW), **closed)),
        'obs_stats_merge_totals': (dict(state_dim=d0), dict(stats=(z(W), COUNT),
                                                            totals=(z(W, dtype=torch.float64), COUNT))),
        'policy_act': (dict(state_dim=d0, hidden=H, action_dim=A, repetitions=REPS, clip=2.0, seed=0, generation=0, t=0),
                       dict(rows=(z(N, P), ROW), obs=(z(N, REPS, d0), COUNT), alive=(z(N, REPS, dtype=torch.uint8), COUNT),
                            obs_stats=(z(W), COUNT), stat_part=(z(N, W, dtype=torch.float64), COUNT),
                            out=(z(N, REPS, A), COUNT))),
        'obs_parts_reduce': (dict(state_dim=d0), dict(parts=(z(N, W, dtype=torch.float64), MULTIPLE),
                                                      out=(z(W, dtype=torch.float64), COUNT))),
        'nes_eval': nes_eval,
        'nes_eval_mirrored': nes_eval,
        'pop_eval': (dict(hidden=H, clip=1.0), dict(solutions=(z(N, P), ROW), **tape, out=(z(N), COUNT))),
        'centered_rank': (dict(member_offset=2, n_local=N),
                          dict(fitness_all=(z(8), FREE), workspace=(z(64, dtype=torch.uint8), WORKSPACE),
                               out=(z(N), COUNT))),
        'nes_grad_partial': grad,
        'nes_grad_partial_mirrored': grad,
        'nes_apply': (dict(N=8, sigma=0.1, learning_rate=0.1),
                      dict(theta=(z(P), FREE), adam_m=(z(P, dtype=torch.float64), COUNT),
                           adam_v=(z(P, dtype=torch.float64), COUNT), partial_sum=(z(P), COUNT), state=state,
                           update_out=(z(P), COUNT), grad_out=(z(P, dtype=torch.float64), COUNT))),
        'cma_rank_mu': ({}, dict(**Y, out=(z(6, 6), COUNT))),
        'cma_rank_mu_packed': ({}, dict(**Y, out=(z(K), COUNT))),
        'cma_cov_apply': (cov, dict(Cmat=(z(6, 6), ROW), dC=(z(6, 6), COUNT), pc=(z(6), COUNT))),
        'cma_cov_apply_packed': (cov, dict(Cmat=(z(6, 6), ROW), tiles=(z(K), COUNT), pc=(z(6), COUNT))),
    }


def _resized(t, kind, d):
    """t with d entries more (d = -1 or +1): on the flat count, per row, or by one tape row."""
    if kind == ROW:
        return z(t.shape[0], t.shape[1] + d, dtype=t.dtype)
    if kind == TAPE:
        return z(t.shape[0] + d, *t.shape[1:], dtype=t.dtype)
    return z(t.numel() + d, dtype=t.dtype)


def _variants(t, kind, anchor):
    if kind not in (FREE, WORKSPACE):
        yield 'one short', _resized(t, kind, -1)
    if kind in (COUNT, ROW, TAPE):
        yield 'one long', _resized(t, kind, +1)
    if kind != WORKSPACE:
        yield 'wrong dtype', t.to(torch.float64 if t.dtype == torch.float32 else torch.float32)
    if t.numel() >= 2:
        yield 'not contiguous', torch.stack([t, t], -1)[..., 0]
    if not anchor:
        yield 'on another device', torch.empty_like(t, device='meta')


def _call(name, scalars, tensors):
    getattr(ops, name)(**scalars, **{k: t for k, (t, _) in tensors.items()})


def test_every_op_taking_a_tensor_has_a_row(lib):  # noqa: F811
    public = {n for n, f in vars(ops).items()
              if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith('_')}
    table = _table()
    assert not set(table) & set(EXEMPT)
    assert set(table) | set(EXEMPT) == public


def test_a_valid_call_passes_every_check_and_stops_at_the_cpu_anchor(lib):  # noqa: F811
    for name, (scalars, tensors) in _table().items():
        with pytest.raises(RuntimeError, match='CPU tensor'):
            _call(name, scalars, tensors)


def test_each_broken_tensor_argument_is_named_before_the_device_is_entered(lib):  # noqa: F811
    missed = []
    for name, (scalars, tensors) in _table().items():
        for i, (arg, (t, kind)) in enumerate(tensors.items()):
            for what, bad in _variants(t, kind, anchor=i == 0):
                try:
                    _call(name, scalars, {**tensors, arg: (bad, kind)})
                    missed.append('%s(%s %s): no error' % (name, arg, what))
                except Exception as e:
                    if type(e) is not RuntimeError or 'CPU tensor' in str(e) or not re.search(r'\b%s\b' % arg, str(e)):
                        missed.append('%s(%s %s): %s: %s' % (name, arg, what, type(e).__name__, e))
    assert not missed, '\n'.join(missed)
