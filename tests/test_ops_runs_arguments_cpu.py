"""ops_runs checks every tensor a run-batched op passes to the library as ops does (dtype, contiguity, element count,
device) before it rejects a CPU tensor: on the CPU a valid call reaches that last check, and each broken argument is named
before it.  The variants are those of test_op_arguments_cpu."""
import inspect
import re

import pytest
import torch

from distributedes_b200 import ops, ops_runs
from lib_fixture import lib  # noqa: F401
from test_op_arguments_cpu import COUNT, FREE, ROW, WORKSPACE, _variants, z

EXEMPT = {
    'rank_runs_workspace': 'a size query and an allocation',
    'grad_runs_workspace': 'a size query and an allocation',
}

d0, H, A, R, N, REPS = 3, 16, 1, 3, 4, 2
W = 2 * d0 + 1


def _table():
    """op -> (its non-tensor arguments, {tensor argument: (tensor, kind)} with the anchor first) of one valid call."""
    P = ops.param_count(d0, H, A)
    state = (z(32, dtype=torch.uint8), COUNT)
    return {
        'rollout_eval_runs': (dict(hidden=H, repetitions=REPS, sigma=0.1, clip=2.0, seed=0, run_size=N),
                              dict(theta=(z(R, P), ROW), state=state, obs_stats=(z(R, W), COUNT),
                                   totals_out=(z(R, W, dtype=torch.float64), COUNT),
                                   workspace=(z(R * N * W, dtype=torch.float64), WORKSPACE), out=(z(R, N), COUNT),
                                   episodes_out=(z(R, N, REPS), COUNT))),
        'obs_stats_merge_totals_runs': (dict(state_dim=d0), dict(stats=(z(R, W), ROW),
                                                                 totals=(z(R, W, dtype=torch.float64), COUNT))),
        'centered_rank_runs': ({}, dict(fitness=(z(R, N), FREE), workspace=(z(64, dtype=torch.uint8), WORKSPACE),
                                        out=(z(R, N), COUNT))),
        'nes_grad_partial_runs': (dict(P=P, seed=0), dict(shaped=(z(R, N), FREE), state=state, out=(z(R, P), COUNT),
                                                          workspace=(z(64, dtype=torch.uint8), WORKSPACE))),
        'nes_apply_runs': (dict(N=N, sigma=0.1, learning_rate=0.1),
                           dict(theta=(z(R, P), FREE), adam_m=(z(R, P, dtype=torch.float64), COUNT),
                                adam_v=(z(R, P, dtype=torch.float64), COUNT), partial_sum=(z(R, P), COUNT), state=state,
                                update_out=(z(R, P), COUNT), grad_out=(z(R, P, dtype=torch.float64), COUNT))),
    }


def _call(name, scalars, tensors):
    getattr(ops_runs, name)(**scalars, **{k: t for k, (t, _) in tensors.items()})


def test_every_run_op_taking_a_tensor_has_a_row(lib):  # noqa: F811
    public = {n for n, f in vars(ops_runs).items()
              if inspect.isfunction(f) and f.__module__ == ops_runs.__name__ and not n.startswith('_')}
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
