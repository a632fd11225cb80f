"""The argument checks of the entry points that take a shard of the population, without a GPU: member range, whole
pairs of a mirrored shard, NULL pointers and policy widths.  Every input here is answered before any CUDA work, so the
library answers it on any machine.  Each case pins the status code and the exact message; where several checks fail
at once the pin also fixes which one is reported."""
import ctypes as C

import pytest

from lib_fixture import lib  # noqa: F401

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
NULL = None
TAPE = (24, 64, 4, 128)      # d0, H, A, T
P_TAPE = 24 * 64 + 64 + 64 * 64 + 64 + 64 * 4 + 4


def _param_count(d0, H, A):
    return d0 * H + H + H * H + H + H * A + A


def _calls(lib, _lib):
    """entry name -> f(off, n, null, H) issuing one call; null=True passes NULL for every pointer."""
    def p(null):
        return NULL if null else D

    def noise_fill(off, n, null, H):
        return lib.des_noise_fill(p(null), n, 37, 0, 0, off, 0, None)

    def perturb(name):
        return lambda off, n, null, H: getattr(lib, name)(p(null), p(null), n, 37, 0.1, 0, 0, off, None)

    def nes_eval(name):
        return lambda off, n, null, H: getattr(lib, name)(p(null), p(null), p(null), p(null), _lib.Dims(*TAPE), 0.1, 1.0,
                                                          0, 0, None, off, n, 2, None, 0, None)

    def grad(name):
        return lambda off, n, null, H: getattr(lib, name)(p(null), p(null), n, P_TAPE, 0, 0, None, off, D, 1 << 20, None)

    def rollout(name):
        return lambda off, n, null, H: getattr(lib, name)(p(null), None, None, p(null), None, 0, _lib.Dims(3, H, 1, 200),
                                                          10, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0, None, 0, None)

    def solutions(off, n, null, H):
        return lib.des_rollout_eval_solutions(p(null), None, None, p(null), None, 0, _lib.Dims(3, H, 1, 200), 10, 2.0, 0.0,
                                              0, 0, off, n, None, 0, None)

    def act(off, n, null, H):
        d0, A = 24, 4
        return lib.des_policy_act(p(null), None, p(null), _param_count(d0, H, A), p(null), p(null), None,
                                  _lib.Dims(d0, H, A, 1), 8, 1.0, 0.0, 0, 0, off, n, 0, None)

    return {
        'des_noise_fill': noise_fill,
        'des_nes_perturb': perturb('des_nes_perturb'),
        'des_nes_perturb_mirrored': perturb('des_nes_perturb_mirrored'),
        'des_nes_eval': nes_eval('des_nes_eval'),
        'des_nes_eval_mirrored': nes_eval('des_nes_eval_mirrored'),
        'des_nes_grad_partial': grad('des_nes_grad_partial'),
        'des_nes_grad_partial_mirrored': grad('des_nes_grad_partial_mirrored'),
        'des_rollout_eval': rollout('des_rollout_eval'),
        'des_rollout_eval_mirrored': rollout('des_rollout_eval_mirrored'),
        'des_rollout_eval_solutions': solutions,
        'des_policy_act': act,
    }


# case -> (member_offset, n, null pointers, hidden)
CASES = {
    'neg_offset_odd': (-1, 2, False, 16),
    'neg_offset_even': (-2, 2, False, 16),
    'odd_offset': (1, 2, False, 16),
    'odd_count': (0, 3, False, 16),
    'past_2^28': ((1 << 28) - 2, 4, False, 16),
    'past_2^32': ((1 << 32) - 2, 4, False, 16),
    'null_zero_count': (0, 0, True, 16),
    'null_count': (0, 2, True, 16),
    'bad_width': (0, 2, False, 48),
}

# (entry, case) -> (status, message); a message of None is not checked (status DES_OK).  Recorded from the library before
# the shard checks were shared between the entry points.
PINS = {
    ('des_noise_fill', 'neg_offset_odd'): (-1, 'des_noise_fill: member index must fit 32 bits'),
    ('des_noise_fill', 'neg_offset_even'): (-1, 'des_noise_fill: member index must fit 32 bits'),
    ('des_noise_fill', 'past_2^32'): (-1, 'des_noise_fill: member index must fit 32 bits'),
    ('des_noise_fill', 'null_zero_count'): (0, None),
    ('des_noise_fill', 'null_count'): (-1, 'des_noise_fill: eps_out_dev is NULL'),
    ('des_nes_perturb', 'neg_offset_odd'): (-1, 'des_nes_perturb: member index must fit 32 bits'),
    ('des_nes_perturb', 'neg_offset_even'): (-1, 'des_nes_perturb: member index must fit 32 bits'),
    ('des_nes_perturb', 'past_2^32'): (-1, 'des_nes_perturb: member index must fit 32 bits'),
    ('des_nes_perturb', 'null_zero_count'): (0, None),
    ('des_nes_perturb', 'null_count'): (-1, 'des_nes_perturb: NULL pointer'),
    ('des_nes_perturb_mirrored', 'neg_offset_odd'): (-1, 'des_nes_perturb_mirrored: a mirrored shard holds whole pairs: member_offset (-1) and n_members (2) must be even'),
    ('des_nes_perturb_mirrored', 'neg_offset_even'): (-1, 'des_nes_perturb_mirrored: member index must fit 32 bits'),
    ('des_nes_perturb_mirrored', 'odd_offset'): (-1, 'des_nes_perturb_mirrored: a mirrored shard holds whole pairs: member_offset (1) and n_members (2) must be even'),
    ('des_nes_perturb_mirrored', 'odd_count'): (-1, 'des_nes_perturb_mirrored: a mirrored shard holds whole pairs: member_offset (0) and n_members (3) must be even'),
    ('des_nes_perturb_mirrored', 'past_2^32'): (-1, 'des_nes_perturb_mirrored: member index must fit 32 bits'),
    ('des_nes_perturb_mirrored', 'null_zero_count'): (0, None),
    ('des_nes_perturb_mirrored', 'null_count'): (-1, 'des_nes_perturb_mirrored: NULL pointer'),
    ('des_nes_eval', 'neg_offset_odd'): (-1, 'des_nes_eval: member index must fit 32 bits'),
    ('des_nes_eval', 'neg_offset_even'): (-1, 'des_nes_eval: member index must fit 32 bits'),
    ('des_nes_eval', 'past_2^32'): (-1, 'des_nes_eval: member index must fit 32 bits'),
    ('des_nes_eval', 'null_zero_count'): (0, None),
    ('des_nes_eval', 'null_count'): (-1, 'des_nes_eval: NULL pointer'),
    ('des_nes_eval_mirrored', 'neg_offset_odd'): (-1, 'des_nes_eval_mirrored: member index must fit 32 bits'),
    ('des_nes_eval_mirrored', 'neg_offset_even'): (-1, 'des_nes_eval_mirrored: member index must fit 32 bits'),
    ('des_nes_eval_mirrored', 'odd_offset'): (-1, 'des_nes_eval_mirrored: a mirrored shard holds whole pairs: member_offset (1) and n_local (2) must be even'),
    ('des_nes_eval_mirrored', 'odd_count'): (-1, 'des_nes_eval_mirrored: a mirrored shard holds whole pairs: member_offset (0) and n_local (3) must be even'),
    ('des_nes_eval_mirrored', 'past_2^32'): (-1, 'des_nes_eval_mirrored: member index must fit 32 bits'),
    ('des_nes_eval_mirrored', 'null_zero_count'): (0, None),
    ('des_nes_eval_mirrored', 'null_count'): (-1, 'des_nes_eval_mirrored: NULL pointer'),
    ('des_nes_grad_partial', 'neg_offset_odd'): (-1, 'des_nes_grad_partial: member index must fit 32 bits'),
    ('des_nes_grad_partial', 'neg_offset_even'): (-1, 'des_nes_grad_partial: member index must fit 32 bits'),
    ('des_nes_grad_partial', 'past_2^32'): (-1, 'des_nes_grad_partial: member index must fit 32 bits'),
    ('des_nes_grad_partial', 'null_zero_count'): (-1, 'des_nes_grad_partial: partial_out_dev is NULL'),
    ('des_nes_grad_partial', 'null_count'): (-1, 'des_nes_grad_partial: partial_out_dev is NULL'),
    ('des_nes_grad_partial_mirrored', 'neg_offset_odd'): (-1, 'des_nes_grad_partial_mirrored: member index must fit 32 bits'),
    ('des_nes_grad_partial_mirrored', 'neg_offset_even'): (-1, 'des_nes_grad_partial_mirrored: member index must fit 32 bits'),
    ('des_nes_grad_partial_mirrored', 'odd_offset'): (-1, 'des_nes_grad_partial_mirrored: a mirrored shard holds whole pairs: member_offset (1) and n_local (2) must be even'),
    ('des_nes_grad_partial_mirrored', 'odd_count'): (-1, 'des_nes_grad_partial_mirrored: a mirrored shard holds whole pairs: member_offset (0) and n_local (3) must be even'),
    ('des_nes_grad_partial_mirrored', 'past_2^32'): (-1, 'des_nes_grad_partial_mirrored: member index must fit 32 bits'),
    ('des_nes_grad_partial_mirrored', 'null_zero_count'): (-1, 'des_nes_grad_partial_mirrored: partial_out_dev is NULL'),
    ('des_nes_grad_partial_mirrored', 'null_count'): (-1, 'des_nes_grad_partial_mirrored: partial_out_dev is NULL'),
    ('des_rollout_eval', 'neg_offset_odd'): (-1, 'des_rollout_eval: bad member range'),
    ('des_rollout_eval', 'neg_offset_even'): (-1, 'des_rollout_eval: bad member range'),
    ('des_rollout_eval', 'past_2^28'): (-1, 'des_rollout_eval: bad member range'),
    ('des_rollout_eval', 'past_2^32'): (-1, 'des_rollout_eval: bad member range'),
    ('des_rollout_eval', 'null_zero_count'): (0, None),
    ('des_rollout_eval', 'null_count'): (-1, 'des_rollout_eval: NULL pointer'),
    ('des_rollout_eval', 'bad_width'): (-1, 'des_rollout_eval: hidden must be 16 or a multiple of 32, <= 128 (got 48)'),
    ('des_rollout_eval_mirrored', 'neg_offset_odd'): (-1, 'des_rollout_eval_mirrored: a mirrored shard holds whole pairs: member_offset (-1) and n_local (2) must be even'),
    ('des_rollout_eval_mirrored', 'neg_offset_even'): (-1, 'des_rollout_eval_mirrored: a mirrored shard holds whole pairs: member_offset (-2) and n_local (2) must be even'),
    ('des_rollout_eval_mirrored', 'odd_offset'): (-1, 'des_rollout_eval_mirrored: a mirrored shard holds whole pairs: member_offset (1) and n_local (2) must be even'),
    ('des_rollout_eval_mirrored', 'odd_count'): (-1, 'des_rollout_eval_mirrored: a mirrored shard holds whole pairs: member_offset (0) and n_local (3) must be even'),
    ('des_rollout_eval_mirrored', 'past_2^28'): (-1, 'des_rollout_eval_mirrored: bad member range'),
    ('des_rollout_eval_mirrored', 'past_2^32'): (-1, 'des_rollout_eval_mirrored: bad member range'),
    ('des_rollout_eval_mirrored', 'null_zero_count'): (0, None),
    ('des_rollout_eval_mirrored', 'null_count'): (-1, 'des_rollout_eval_mirrored: NULL pointer'),
    ('des_rollout_eval_mirrored', 'bad_width'): (-1, 'des_rollout_eval_mirrored: hidden must be 16 or a multiple of 32, <= 128 (got 48)'),
    ('des_rollout_eval_solutions', 'neg_offset_odd'): (-1, 'des_rollout_eval_solutions: bad member range'),
    ('des_rollout_eval_solutions', 'neg_offset_even'): (-1, 'des_rollout_eval_solutions: bad member range'),
    ('des_rollout_eval_solutions', 'past_2^28'): (-1, 'des_rollout_eval_solutions: bad member range'),
    ('des_rollout_eval_solutions', 'past_2^32'): (-1, 'des_rollout_eval_solutions: bad member range'),
    ('des_rollout_eval_solutions', 'null_zero_count'): (0, None),
    ('des_rollout_eval_solutions', 'null_count'): (-1, 'des_rollout_eval_solutions: NULL pointer'),
    ('des_rollout_eval_solutions', 'bad_width'): (-1, 'des_rollout_eval_solutions: hidden must be 16 or a multiple of 32, <= 128 (got 48)'),
    ('des_policy_act', 'neg_offset_odd'): (-1, 'des_policy_act: bad member range'),
    ('des_policy_act', 'neg_offset_even'): (-1, 'des_policy_act: bad member range'),
    ('des_policy_act', 'past_2^28'): (-1, 'des_policy_act: bad member range'),
    ('des_policy_act', 'past_2^32'): (-1, 'des_policy_act: bad member range'),
    ('des_policy_act', 'null_zero_count'): (-1, 'des_policy_act: NULL alive mask'),
    ('des_policy_act', 'null_count'): (-1, 'des_policy_act: NULL alive mask'),
    ('des_policy_act', 'bad_width'): (-1, 'des_policy_act: hidden must be 16, 32, 64, 96 or 128 (got 48)'),
}


@pytest.mark.parametrize('entry,case', sorted(PINS))
def test_entry_point_rejects_before_cuda_work(lib, entry, case):
    from distributedes_b200 import _lib
    off, n, null, H = CASES[case]
    rc = _calls(lib, _lib)[entry](off, n, null, H)
    status, message = PINS[entry, case]
    assert rc == status
    if message is not None:
        assert lib.des_last_error().decode() == message


def test_pins_cover_every_entry_point_and_case():
    from distributedes_b200 import _lib
    entries = set(_calls(None, _lib))
    assert {e for e, _ in PINS} == entries
    for e in entries:
        assert {'neg_offset_odd', 'neg_offset_even', 'null_zero_count', 'null_count'} <= {c for x, c in PINS if x == e}
    phrases = [m for m in (v[1] for v in PINS.values()) if m]
    for phrase in ('whole pairs', 'multiple of 32', 'must fit 32 bits', 'bad member range', 'NULL pointer'):
        assert any(phrase in m for m in phrases), phrase

