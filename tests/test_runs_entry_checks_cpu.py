"""The argument checks of the run-batched entry points (des_*_runs), without a GPU: the batch shape (n_runs, run_size),
the 2^28 member bound, the 2048-member run limit, NULL pointers, the policy width, noiseless batches, the rank's two
members and the workspace.  Every case is answered before any CUDA work; each pins the status and the exact message."""
import ctypes as C

import pytest

from lib_fixture import lib  # noqa: F401

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
P = 3 * 16 + 16 + 16 * 16 + 16 + 16 + 1
BIG = 1 << 20                # a workspace size no case here is short of


def _calls(lib, _lib):
    """entry -> f(n_runs, run_size, null, H, noiseless, ws_bytes) issuing one call; null passes NULL for every pointer."""
    def p(null):
        return None if null else D

    def rollout(R, N, null, H, noiseless, ws):
        return lib.des_rollout_eval_runs(p(null), None, p(null), p(null), None, 0, _lib.Dims(3, H, 1, 200), 10, 0.1, 2.0,
                                         0.0, 0, 0, None, R, N, noiseless, p(null), ws, None)

    def rank(R, N, null, H, noiseless, ws):
        return lib.des_centered_rank_runs(p(null), None, p(null), R, N, p(null), ws, None)

    def grad(R, N, null, H, noiseless, ws):
        return lib.des_nes_grad_partial_runs(p(null), p(null), R, N, P, 0, 0, None, p(null), ws, None)

    def apply(R, N, null, H, noiseless, ws):
        return lib.des_nes_apply_runs(p(null), p(null), p(null), None, None, p(null), P, R, N,
                                      _lib.Opt(0.1, 0.1, 0.005, 0.9, 0.999, 1e-8), p(null), None)

    def merge(R, N, null, H, noiseless, ws):
        return lib.des_obs_stats_merge_totals_runs(p(null), p(null), 3, R, None)

    return {'des_rollout_eval_runs': rollout, 'des_centered_rank_runs': rank, 'des_nes_grad_partial_runs': grad,
            'des_nes_apply_runs': apply, 'des_obs_stats_merge_totals_runs': merge}


# case -> (n_runs, run_size, null pointers, hidden, noiseless, workspace bytes)
CASES = {
    'neg_runs': (-1, 4, False, 16, 0, BIG),
    'neg_size': (2, -4, False, 16, 0, BIG),
    'size_1': (3, 1, False, 16, 0, BIG),          # a valid batch everywhere but the rank
    'size_2049': (2, 2049, False, 16, 0, BIG),
    'past_2^28': ((1 << 28) // 64 + 1, 64, False, 16, 0, BIG),
    'huge_runs': (1 << 62, 2, False, 16, 0, BIG),
    'null_zero_runs': (0, 4, True, 16, 0, 0),
    'null_runs': (2, 4, True, 16, 0, BIG),
    'bad_width': (2, 4, False, 48, 0, BIG),
    'noiseless_4': (2, 4, False, 16, 1, BIG),
    'small_ws': (3, 4, False, 16, 0, 16),
}

E = 'des_rollout_eval_runs'
K = 'des_centered_rank_runs'
G = 'des_nes_grad_partial_runs'
A = 'des_nes_apply_runs'
M = 'des_obs_stats_merge_totals_runs'


def _shape(who, R, N, lo):
    return (-1, '%s: need n_runs >= 0 and run_size >= %d (got %d and %d)' % (who, lo, R, N))


def _past(who, R, N):
    return (-1, '%s: n_runs x run_size = %d x %d members, past 2^28' % (who, R, N))


def _over(who):
    return (-5, '%s: run_size 2049 > 2048: batches hold runs of up to 2048 members (a larger population fills the GPU '
                'alone)' % who)


PINS = {}
for who, lo in ((E, 1), (K, 2), (G, 1), (A, 1)):
    PINS[who, 'neg_runs'] = _shape(who, -1, 4, lo)
    PINS[who, 'neg_size'] = _shape(who, 2, -4, lo)
    PINS[who, 'size_2049'] = _over(who)
    PINS[who, 'past_2^28'] = _past(who, (1 << 28) // 64 + 1, 64)
    PINS[who, 'huge_runs'] = _past(who, 1 << 62, 2)
    PINS[who, 'null_zero_runs'] = (0, None)
    PINS[who, 'null_runs'] = (-1, '%s: NULL pointer' % who)
PINS[K, 'size_1'] = _shape(K, 3, 1, 2)
PINS[E, 'bad_width'] = (-1, '%s: hidden must be 16 or a multiple of 32, <= 128 (got 48)' % E)
PINS[E, 'noiseless_4'] = (-1, '%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 (got 4)' % E)
PINS[K, 'small_ws'] = (-4, '%s: workspace 16 B < required 48 B' % K)
PINS[G, 'small_ws'] = (-4, '%s: workspace 16 B < required %d B' % (G, 3 * 4 * 4 * ((P + 3) // 4)))
PINS[M, 'neg_runs'] = (-1, '%s: need 0 <= n_runs <= 2^28 (got -1)' % M)
PINS[M, 'huge_runs'] = (-1, '%s: need 0 <= n_runs <= 2^28 (got %d)' % (M, 1 << 62))
PINS[M, 'null_zero_runs'] = (0, None)
PINS[M, 'null_runs'] = (-1, '%s: NULL pointer' % M)


@pytest.mark.parametrize('entry,case', sorted(PINS))
def test_run_entry_point_rejects_before_cuda_work(lib, entry, case):  # noqa: F811
    from distributedes_b200 import _lib
    rc = _calls(lib, _lib)[entry](*CASES[case])
    status, message = PINS[entry, case]
    assert rc == status
    if message is not None:
        assert lib.des_last_error().decode() == message


def test_the_rollout_needs_a_workspace_for_the_totals(lib):  # noqa: F811
    from distributedes_b200 import _lib
    rc = lib.des_rollout_eval_runs(D, None, D, D, None, 0, _lib.Dims(3, 16, 1, 200), 10, 0.1, 2.0, 0.0, 0, 0, None, 3, 4,
                                   0, D, 16, None)
    assert rc == -4
    assert lib.des_last_error().decode() == 'des_rollout_eval_runs: workspace 16 B < required 672 B'


def test_workspace_queries_answer_zero_for_a_batch_they_cannot_run(lib):  # noqa: F811
    assert lib.des_rank_runs_workspace_bytes(3, 4) == 48
    assert lib.des_grad_runs_workspace_bytes(3, 4, P) == 3 * lib.des_grad_workspace_bytes(4, P)
    for R, N in ((0, 4), (-1, 4), (2, 2049), ((1 << 28) // 64 + 1, 64)):
        assert lib.des_rank_runs_workspace_bytes(R, N) == 0
        assert lib.des_grad_runs_workspace_bytes(R, N, P) == 0


def test_pins_cover_every_entry_point():
    from distributedes_b200 import _lib
    assert {e for e, _ in PINS} == set(_calls(None, _lib))
    for e in (E, K, G, A):
        assert {'neg_runs', 'neg_size', 'size_2049', 'past_2^28', 'null_zero_runs', 'null_runs'} <= {c for x, c in PINS
                                                                                                      if x == e}
