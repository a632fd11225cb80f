"""The argument checks of the sweep entry points (des_*_sweep), without a GPU: the batch shape (n_runs, run_size), the
2^28 member bound, the 2048-member run limit, NULL pointers (the table included), noiseless batches and the workspace.
Every case is answered before any CUDA work; each pins the status and the exact message.  The table's layout: the
ctypes mirror of des_run_hp is the header's 40 bytes, field by field (the C side pins the same with a static_assert)."""
import ctypes as C

import pytest
import torch

from lib_fixture import lib  # noqa: F401

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
P = 3 * 16 + 16 + 16 * 16 + 16 + 16 + 1
BIG = 1 << 20                # a workspace size no case here is short of


def _calls(lib, _lib):
    """entry -> f(n_runs, run_size, null, null_hp, noiseless, ws_bytes) issuing one call; null passes NULL for every
    tensor pointer, null_hp NULL for the table."""
    def p(null):
        return None if null else D

    def rollout(R, N, null, null_hp, noiseless, ws):
        return lib.des_rollout_eval_sweep(p(null), None, p(null), p(null), None, 0, _lib.Dims(3, 16, 1, 200), 10, 2.0,
                                          p(null_hp), 0, None, R, N, noiseless, p(null), ws, None)

    def grad(R, N, null, null_hp, noiseless, ws):
        return lib.des_nes_grad_partial_sweep(p(null), p(null), R, N, P, p(null_hp), 0, None, p(null), ws, None)

    def apply(R, N, null, null_hp, noiseless, ws):
        return lib.des_nes_apply_sweep(p(null), p(null), p(null), None, None, p(null), P, R, N, p(null_hp), 0.9, 0.999,
                                       1e-8, p(null), None)

    return {'des_rollout_eval_sweep': rollout, 'des_nes_grad_partial_sweep': grad, 'des_nes_apply_sweep': apply}


# case -> (n_runs, run_size, null tensors, null table, noiseless, workspace bytes)
CASES = {
    'neg_runs': (-1, 4, False, False, 0, BIG),
    'neg_size': (2, -4, False, False, 0, BIG),
    'size_0': (2, 0, False, False, 0, BIG),
    'size_2049': (2, 2049, False, False, 0, BIG),
    'past_2^28': ((1 << 28) // 64 + 1, 64, False, False, 0, BIG),
    'huge_runs': (1 << 62, 2, False, False, 0, BIG),
    'null_zero_runs': (0, 4, True, True, 0, 0),
    'null_runs': (2, 4, True, False, 0, BIG),
    'null_table': (2, 4, False, True, 0, BIG),
    'noiseless_4': (2, 4, False, False, 1, BIG),
    'small_ws': (3, 4, False, False, 0, 16),
}

E = 'des_rollout_eval_sweep'
G = 'des_nes_grad_partial_sweep'
A = 'des_nes_apply_sweep'

PINS = {}
for who in (E, G, A):
    for case, (R, N) in (('neg_runs', (-1, 4)), ('neg_size', (2, -4)), ('size_0', (2, 0))):
        PINS[who, case] = (-1, '%s: need n_runs >= 0 and run_size >= 1 (got %d and %d)' % (who, R, N))
    PINS[who, 'size_2049'] = (-5, '%s: run_size 2049 > 2048: batches hold runs of up to 2048 members (a larger population '
                                  'fills the GPU alone)' % who)
    PINS[who, 'past_2^28'] = (-1, '%s: n_runs x run_size = %d x 64 members, past 2^28' % (who, (1 << 28) // 64 + 1))
    PINS[who, 'huge_runs'] = (-1, '%s: n_runs x run_size = %d x 2 members, past 2^28' % (who, 1 << 62))
    PINS[who, 'null_zero_runs'] = (0, None)
    PINS[who, 'null_runs'] = (-1, '%s: NULL pointer' % who)
    PINS[who, 'null_table'] = (-1, '%s: NULL pointer' % who)
PINS[E, 'noiseless_4'] = (-1, '%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 (got 4)' % E)
PINS[E, 'small_ws'] = (-4, '%s: workspace 16 B < required 672 B' % E)
PINS[G, 'small_ws'] = (-4, '%s: workspace 16 B < required %d B' % (G, 3 * 4 * 4 * ((P + 3) // 4)))


@pytest.mark.parametrize('entry,case', sorted(PINS))
def test_sweep_entry_point_rejects_before_cuda_work(lib, entry, case):  # noqa: F811
    from distributedes_b200 import _lib
    rc = _calls(lib, _lib)[entry](*CASES[case])
    status, message = PINS[entry, case]
    assert rc == status
    if message is not None:
        assert lib.des_last_error().decode() == message


def test_the_table_mirror_has_the_header_layout(lib):  # noqa: F811
    from distributedes_b200 import _lib, ops_sweep
    assert C.sizeof(_lib.RunHp) == ops_sweep.HP_BYTES == 40
    assert [(n, getattr(_lib.RunHp, n).offset) for n, _ in _lib.RunHp._fields_] == [
        ('seed', 0), ('sigma', 8), ('learning_rate', 16), ('weight_decay', 24), ('action_noise_std', 32)]


def test_run_table_rows_read_back_through_the_mirror():
    from distributedes_b200 import _lib, ops_sweep
    t = ops_sweep.run_table([3, -1, 1 << 40], [0.1, 0.2, 0.3], 0.05, [0.0, 0.005, 0.01], 0.25, 'cpu')
    assert t.dtype == torch.uint8 and t.shape == (3, 40) and t.is_contiguous()
    rows = [_lib.RunHp.from_buffer_copy(bytes(r.tolist())) for r in t]
    assert [r.seed for r in rows] == [3, (1 << 64) - 1, 1 << 40]              # a uint64_t, as ctypes passes ops' seed
    assert [r.sigma for r in rows] == [0.1, 0.2, 0.3]
    assert [r.learning_rate for r in rows] == [0.05] * 3
    assert [r.weight_decay for r in rows] == [0.0, 0.005, 0.01]
    assert [r.action_noise_std for r in rows] == [0.25] * 3
    assert ops_sweep.run_table(7, 0.1, 0.1, 0.0, 0.0, 'cpu').shape == (1, 40)
    assert ops_sweep.run_table(7, 0.1, 0.1, 0.0, 0.0, 'cpu', runs=4).shape == (4, 40)
    with pytest.raises(ValueError, match='sigma has 2 entries; a sweep of 3 runs'):
        ops_sweep.run_table([1, 2, 3], [0.1, 0.2], 0.1, 0.0, 0.0, 'cpu')


def test_pins_cover_every_entry_point():
    from distributedes_b200 import _lib
    assert {e for e, _ in PINS} == set(_calls(None, _lib))
    for e in (E, G, A):
        assert {'neg_runs', 'size_2049', 'past_2^28', 'null_zero_runs', 'null_runs', 'null_table'} <= {
            c for x, c in PINS if x == e}
