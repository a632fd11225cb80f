"""ops_sweep checks every tensor a sweep op passes to the library as ops does (dtype, contiguity, element count, device)
before it rejects a CPU tensor, the table `hp` included: on the CPU a valid call reaches that last check, and each broken
argument (a table of the wrong dtype, length or device among them) is named before it.  The variants are those of
test_op_arguments_cpu.  ops_runs re-exports the sweep ops: the engine's one module of device ops."""
import inspect
import re

import pytest
import torch

from distributedes_b200 import ops, ops_runs, ops_sweep
from lib_fixture import lib  # noqa: F401
from test_op_arguments_cpu import COUNT, FREE, ROW, WORKSPACE, _variants, z

EXEMPT = {
    'run_table': 'builds the table from Python values',
    'per_run': 'a host helper: one value per run',
}

d0, H, A, R, N, REPS = 3, 16, 1, 3, 4, 2
W = 2 * d0 + 1


def _table():
    """op -> (its non-tensor arguments, {tensor argument: (tensor, kind)} with the anchor first) of one valid call."""
    P = ops.param_count(d0, H, A)
    state = (z(32, dtype=torch.uint8), COUNT)
    hp = (z(R, 40, dtype=torch.uint8), COUNT)
    return {
        'rollout_eval_sweep': (dict(hidden=H, repetitions=REPS, clip=2.0, run_size=N),
                               dict(theta=(z(R, P), ROW), hp=hp, state=state, obs_stats=(z(R, W), COUNT),
                                    totals_out=(z(R, W, dtype=torch.float64), COUNT),
                                    workspace=(z(R * N * W, dtype=torch.float64), WORKSPACE), out=(z(R, N), COUNT),
                                    episodes_out=(z(R, N, REPS), COUNT))),
        'nes_grad_partial_sweep': (dict(P=P), dict(shaped=(z(R, N), FREE), hp=hp, state=state, out=(z(R, P), COUNT),
                                                   workspace=(z(64, dtype=torch.uint8), WORKSPACE))),
        'nes_apply_sweep': (dict(N=N), dict(theta=(z(R, P), FREE), adam_m=(z(R, P, dtype=torch.float64), COUNT),
                                            adam_v=(z(R, P, dtype=torch.float64), COUNT), partial_sum=(z(R, P), COUNT),
                                            state=state, hp=hp, update_out=(z(R, P), COUNT),
                                            grad_out=(z(R, P, dtype=torch.float64), COUNT))),
    }


def _call(name, scalars, tensors):
    getattr(ops_sweep, name)(**scalars, **{k: t for k, (t, _) in tensors.items()})


def test_every_sweep_op_taking_a_tensor_has_a_row_and_ops_runs_lists_it(lib):  # noqa: F811
    public = {n for n, f in vars(ops_sweep).items()
              if inspect.isfunction(f) and f.__module__ == ops_sweep.__name__ and not n.startswith('_')}
    table = _table()
    assert not set(table) & set(EXEMPT)
    assert set(table) | set(EXEMPT) == public
    for name in list(table) + ['run_table']:
        assert getattr(ops_runs, name) is getattr(ops_sweep, name), name


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


@pytest.mark.parametrize('bad,match', [
    (z(R, 40, dtype=torch.float32), r'hp must be torch\.uint8'),
    (z(R + 1, 40, dtype=torch.uint8), r'hp has 160 entries, needs one 40-byte row per run: 120'),
    (z(R, 39, dtype=torch.uint8), r'hp has 117 entries'),
    (torch.empty(R, 40, dtype=torch.uint8, device='meta'), r'hp is on meta'),
])
def test_a_table_of_the_wrong_dtype_length_or_device_is_refused(lib, bad, match):  # noqa: F811
    scalars, tensors = _table()['nes_grad_partial_sweep']
    with pytest.raises(RuntimeError, match=match):
        _call('nes_grad_partial_sweep', scalars, {**tensors, 'hp': (bad, COUNT)})
