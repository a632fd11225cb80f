"""The argument checks of the host-stepped sweep entry points (des_nes_perturb_sweep, des_policy_act_sweep,
des_obs_parts_reduce_runs) and of their wrappers in ops_host_sweep, without a GPU.  The entry points answer every case
before any CUDA work: the batch shape (n_runs, run_size), the 2^28 member bound, the 2048-member run limit, NULL pointers
(the table included), n_runs 0 and every shape limit of des_policy_act.  The wrappers check every tensor they pass (dtype,
contiguity, element count, device; the table too) before they reject a CPU tensor, as ops does; ops_sweep and ops_runs
list them."""
import ctypes as C
import inspect
import re

import pytest
import torch

from distributedes_b200 import ops, ops_host_sweep, ops_runs, ops_sweep
from lib_fixture import lib  # noqa: F401
from test_op_arguments_cpu import COUNT, FREE, MULTIPLE, ROW, _variants, z

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
PA = 'des_perturb'
AC = 'des_policy_act_sweep'
RD = 'des_obs_parts_reduce_runs'


def _p(null):
    return None if null else D


def perturb(lib, R=2, N=4, P=113, null=False, null_hp=False):
    return lib.des_nes_perturb_sweep(_p(null), _p(null), R, N, P, _p(null_hp), 0, None)


def act(lib, R=2, N=4, d0=3, H=16, A=1, reps=10, P=None, null=False, null_hp=False, alive=True, t=0):
    from distributedes_b200._lib import Dims
    if P is None:
        P = max(int(lib.des_param_count(d0, H, A)), 1)
    return lib.des_policy_act_sweep(_p(null), None, _p(null), P, _p(null), D if alive else None, None, Dims(d0, H, A, 0),
                                    reps, 1.0, _p(null_hp), 0, R, N, t, None)


def reduce(lib, R=2, N=4, d0=3, null=False):
    return lib.des_obs_parts_reduce_runs(_p(null), _p(null), R, N, d0, None)


BATCH = {
    'neg_runs': (dict(R=-1), -1, '%s: need n_runs >= 0 and run_size >= 1 (got -1 and 4)'),
    'size_0': (dict(N=0), -1, '%s: need n_runs >= 0 and run_size >= 1 (got 2 and 0)'),
    'size_2049': (dict(N=2049), -5, '%s: run_size 2049 > 2048: batches hold runs of up to 2048 members (a larger '
                                    'population fills the GPU alone)'),
    'past_2^28': (dict(R=(1 << 28) // 64 + 1, N=64), -1, '%%s: n_runs x run_size = %d x 64 members, past 2^28'
                  % ((1 << 28) // 64 + 1)),
    'null_zero_runs': (dict(R=0, null=True), 0, None),
    'null_runs': (dict(null=True), -1, '%s: NULL pointer'),
}
TABLE = {'null_table': (dict(null_hp=True), -1, '%s: NULL pointer'),
         'null_zero_runs_table': (dict(R=0, null=True, null_hp=True), 0, None)}

PINS = {}
for who, fn in (('des_nes_perturb_sweep', perturb), (AC, act), (RD, reduce)):
    for case, (kw, rc, msg) in list(BATCH.items()) + (list(TABLE.items()) if fn is not reduce else []):
        PINS[who, case] = (fn, kw, rc, None if msg is None else msg % who)
PINS['des_nes_perturb_sweep', 'P_0'] = (perturb, dict(P=0), -1, 'des_nes_perturb_sweep: bad size P=0')
for case, kw, msg in (
        ('hidden_48', dict(H=48), 'hidden must be 16, 32, 64, 96 or 128 (got 48)'),
        ('state_dim_0', dict(d0=0), 'state_dim must be in [1, 32] (got 0)'),
        ('state_dim_33', dict(d0=33), 'state_dim must be in [1, 32] (got 33)'),
        ('action_dim_9', dict(A=9), 'action_dim must be in [1, 8] (got 9)'),
        ('reps_0', dict(reps=0), 'repetitions must be in [1, 16] (the action-noise counter is member*16 + repetition; '
                                 'got 0)'),
        ('reps_17', dict(reps=17), 'repetitions must be in [1, 16] (the action-noise counter is member*16 + '
                                   'repetition; got 17)'),
        ('P_wrong', dict(P=371), 'rows have P = 371, the (3,16,1) MLP needs 353'),
        ('t_negative', dict(t=-1), 'step index must be in [0, 2^31)'),
        ('t_2^31', dict(t=1 << 31), 'step index must be in [0, 2^31)'),
        ('no_alive', dict(alive=False), 'NULL alive mask')):
    PINS[AC, case] = (act, kw, -1, '%s: %s' % (AC, msg))
PINS[RD, 'state_dim_0'] = (reduce, dict(d0=0), -1, '%s: state_dim must be in [1, 511] (got 0)' % RD)
PINS[RD, 'state_dim_512'] = (reduce, dict(d0=512), -1, '%s: state_dim must be in [1, 511] (got 512)' % RD)


@pytest.mark.parametrize('entry,case', sorted(PINS))
def test_host_sweep_entry_point_rejects_before_cuda_work(lib, entry, case):  # noqa: F811
    fn, kw, status, message = PINS[entry, case]
    assert fn(lib, **kw) == status
    if message is not None:
        assert lib.des_last_error().decode() == message


# ---- the wrappers ----------------------------------------------------------------------------------------------------
d0, H, A, R, N, REPS = 3, 16, 1, 3, 4, 2
W = 2 * d0 + 1


def _table():
    """op -> (its non-tensor arguments, {tensor argument: (tensor, kind)} with the anchor first) of one valid call."""
    P = ops.param_count(d0, H, A)
    hp = (z(R, 40, dtype=torch.uint8), COUNT)
    return {
        'nes_perturb_sweep': (dict(run_size=N, generation=0), dict(theta=(z(R, P), FREE), hp=hp,
                                                                    out=(z(R * N, P), COUNT))),
        'policy_act_sweep': (dict(state_dim=d0, hidden=H, action_dim=A, repetitions=REPS, clip=2.0, generation=0,
                                  run_size=N, t=0),
                             dict(rows=(z(R * N, P), ROW), obs=(z(R * N, REPS, d0), COUNT),
                                  alive=(z(R * N, REPS, dtype=torch.uint8), COUNT), hp=hp, obs_stats=(z(R, W), COUNT),
                                  stat_part=(z(R * N, W, dtype=torch.float64), COUNT), out=(z(R * N, REPS, A), COUNT))),
        'obs_parts_reduce_runs': (dict(state_dim=d0, run_size=N),
                                  dict(parts=(z(R * N, W, dtype=torch.float64), MULTIPLE),
                                       out=(z(R, W, dtype=torch.float64), COUNT))),
    }


def _call(name, scalars, tensors):
    getattr(ops_host_sweep, name)(**scalars, **{k: t for k, (t, _) in tensors.items()})


def test_every_op_has_a_row_and_ops_sweep_and_ops_runs_list_it(lib):  # noqa: F811
    public = {n for n, f in vars(ops_host_sweep).items()
              if inspect.isfunction(f) and f.__module__ == ops_host_sweep.__name__ and not n.startswith('_')}
    assert set(_table()) == public
    for name in public:
        assert getattr(ops_sweep, name) is getattr(ops_runs, name) is getattr(ops_host_sweep, name), name


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
    (torch.empty(R, 40, dtype=torch.uint8, device='meta'), r'hp is on meta'),
])
@pytest.mark.parametrize('op', ['nes_perturb_sweep', 'policy_act_sweep'])
def test_a_table_of_the_wrong_dtype_length_or_device_is_refused(lib, op, bad, match):  # noqa: F811
    scalars, tensors = _table()[op]
    with pytest.raises(RuntimeError, match=match):
        _call(op, scalars, {**tensors, 'hp': (bad, COUNT)})


def test_rows_and_parts_must_be_whole_runs(lib):  # noqa: F811
    scalars, tensors = _table()['policy_act_sweep']
    with pytest.raises(RuntimeError, match='rows has 12 rows, not a whole number of runs of run_size 5'):
        _call('policy_act_sweep', dict(scalars, run_size=5), tensors)
    scalars, tensors = _table()['obs_parts_reduce_runs']
    with pytest.raises(RuntimeError, match='parts has 84 entries, not a whole number of runs of 5 rows'):
        _call('obs_parts_reduce_runs', dict(scalars, run_size=5), tensors)
