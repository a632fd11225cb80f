"""The argument checks of the genetic-algorithm sweep entry points and their wrappers, without a GPU:
des_rollout_eval_ga_sweep, des_ga_rows_sweep and des_ga_order_runs refuse bad batches, table sizes, NULL pointers,
overlapping tables and small workspaces before any CUDA work (des_rollout_eval_ga_sweep also what des_rollout_eval_sweep
refuses, with its message under its own name); n_runs = 0 does nothing and accepts NULL pointers; the wrappers check their
tensors in ops._ptr, and ga_table refuses counts out of range before it writes the table."""
import ctypes as C

import pytest

torch = pytest.importorskip('torch')

from lib_fixture import lib  # noqa: F401,E402
from oracle import nes_oracle as orc  # noqa: E402

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
P = orc.param_count(3, 16, 1)


def _msg(lib):
    return lib.des_last_error().decode()


def _dims(h=16, T=200):
    from distributedes_b200 import _lib
    return _lib.Dims(3, h, 1, T)


def _eval(lib, n_runs=2, run_size=4, rows=2, null=False, env=0, h=16, reps=10, T=200):
    p = None if null else D
    return lib.des_rollout_eval_ga_sweep(p, None, None, p, p, rows, None, env, _dims(h, T), reps, 2.0, p, 0, None, n_runs,
                                         run_size, None, 0, None)


# case -> (kwargs of _eval, status, message)
EVAL = {
    'run_size_1': (dict(run_size=1, rows=1), -1, 'des_rollout_eval_ga_sweep: need n_runs >= 0 and run_size >= 2 (got 2 '
                   'and 1)'),
    'negative_runs': (dict(n_runs=-1), -1, 'des_rollout_eval_ga_sweep: need n_runs >= 0 and run_size >= 2 (got -1 and 4)'),
    'run_size_2049': (dict(run_size=2049), -5, 'des_rollout_eval_ga_sweep: run_size 2049 > 2048: batches hold runs of up '
                      'to 2048 members (a larger population fills the GPU alone)'),
    'past_2^28': (dict(n_runs=1 << 27, run_size=4), -1, 'des_rollout_eval_ga_sweep: n_runs x run_size = 134217728 x 4 '
                  'members, past 2^28'),
    'rows_0': (dict(rows=0), -1, 'des_rollout_eval_ga_sweep: table_rows must be in [1, run_size = 4] (got 0)'),
    'rows_past_N': (dict(rows=5), -1, 'des_rollout_eval_ga_sweep: table_rows must be in [1, run_size = 4] (got 5)'),
    'null': (dict(null=True), -1, 'des_rollout_eval_ga_sweep: NULL pointer'),
}


@pytest.mark.parametrize('case', list(EVAL))
def test_rollout_eval_ga_sweep_refuses(lib, case):  # noqa: F811
    kw, rc, msg = EVAL[case]
    assert _eval(lib, **kw) == rc and _msg(lib) == msg


@pytest.mark.parametrize('kw', [dict(env=1), dict(h=48), dict(reps=0), dict(reps=11), dict(T=0)])
def test_rollout_eval_ga_sweep_refuses_what_des_rollout_eval_sweep_refuses(lib, kw):  # noqa: F811
    rc = lib.des_rollout_eval_sweep(D, None, None, D, None, kw.get('env', 0), _dims(kw.get('h', 16), kw.get('T', 200)),
                                    kw.get('reps', 10), 2.0, D, 0, None, 2, 4, 0, None, 0, None)
    ev = (rc, _msg(lib))
    assert ev[0] != 0 and _eval(lib, **kw) == ev[0]
    assert _msg(lib) == ev[1].replace('des_rollout_eval_sweep', 'des_rollout_eval_ga_sweep', 1)


def test_rollout_eval_ga_sweep_needs_a_workspace_for_totals(lib):  # noqa: F811
    rc = lib.des_rollout_eval_ga_sweep(D, None, D, D, D, 2, None, 0, _dims(), 10, 2.0, D, 0, None, 2, 4, D, 8, None)
    assert rc == -4 and _msg(lib) == 'des_rollout_eval_ga_sweep: workspace 8 B < required %d B' % (8 * 7 * 8)


def test_zero_runs_do_nothing(lib):  # noqa: F811
    assert _eval(lib, n_runs=0, null=True) == 0
    assert lib.des_ga_rows_sweep(None, None, None, 2, P, None, 0, 0, 4, None, None) == 0
    assert lib.des_ga_order_runs(None, None, None, 2, 0, 4, None, 0, None) == 0
    assert lib.des_ga_order_runs_workspace_bytes(0, 4) == 0


def _rows(lib, out=D, parents=C.c_void_p(1 << 20), rows=2, p=9, n_runs=2, run_size=4, members=None, null=False):
    ptr = None if null else D
    return lib.des_ga_rows_sweep(None if null else out, None if null else parents, ptr, rows, p, ptr, 0, n_runs,
                                 run_size, members, None)


@pytest.mark.parametrize('kw,rc,msg', [
    (dict(run_size=1, rows=1), -1, 'des_ga_rows_sweep: need n_runs >= 0 and run_size >= 2 (got 2 and 1)'),
    (dict(run_size=4096), -5, 'des_ga_rows_sweep: run_size 4096 > 2048: batches hold runs of up to 2048 members (a larger '
     'population fills the GPU alone)'),
    (dict(p=0), -1, 'des_ga_rows_sweep: bad size (P=0)'),
    (dict(rows=0), -1, 'des_ga_rows_sweep: table_rows must be in [1, run_size = 4] (got 0)'),
    (dict(rows=5), -1, 'des_ga_rows_sweep: table_rows must be in [1, run_size = 4] (got 5)'),
    (dict(null=True), -1, 'des_ga_rows_sweep: NULL pointer'),
])
def test_ga_rows_sweep_refuses(lib, kw, rc, msg):  # noqa: F811
    assert _rows(lib, **kw) == rc and _msg(lib) == msg


def test_ga_rows_sweep_refuses_rows_that_overlap_the_parents(lib):  # noqa: F811
    base = 1 << 20                                           # parents: 2 runs x 2 rows x 9 floats
    msg = 'des_ga_rows_sweep: rows_out overlaps parents (the table is double-buffered)'
    for out, members in ((base, None), (base + 4 * 9 * 3, None), (base - 4 * 9 * 8 + 4, None), (base + 4, D)):
        assert _rows(lib, out=C.c_void_p(out), members=members) == -1 and _msg(lib) == msg


@pytest.mark.parametrize('n_runs,N,rows,null,ws,rc,msg', [
    (2, 1, 1, False, None, -1, 'des_ga_order_runs: need n_runs >= 0 and run_size >= 2 (got 2 and 1)'),
    (2, 2049, 2, False, None, -5, 'des_ga_order_runs: run_size 2049 > 2048: batches hold runs of up to 2048 members (a '
     'larger population fills the GPU alone)'),
    (2, 4, 0, False, None, -1, 'des_ga_order_runs: table_rows must be in [1, run_size = 4] (got 0)'),
    (2, 4, 5, False, None, -1, 'des_ga_order_runs: table_rows must be in [1, run_size = 4] (got 5)'),
    (2, 4, 2, True, None, -1, 'des_ga_order_runs: NULL pointer'),
    (2, 4, 2, False, 8, -4, None),
])
def test_ga_order_runs_refuses(lib, n_runs, N, rows, null, ws, rc, msg):  # noqa: F811
    p = None if null else D
    assert lib.des_ga_order_runs(p, p, p, rows, n_runs, N, D if ws else None, ws or 0, None) == rc
    need = lib.des_ga_order_runs_workspace_bytes(n_runs, N)
    assert _msg(lib) == (msg or 'des_ga_order_runs: workspace 8 B < required %d B' % need)


def test_ga_order_runs_workspace_covers_the_rank(lib):  # noqa: F811
    for R, N in ((1, 2), (10, 64), (3, 2048)):
        assert lib.des_ga_order_runs_workspace_bytes(R, N) >= 3 * 4 * R * N + lib.des_rank_runs_workspace_bytes(R, N)
    assert lib.des_ga_order_runs_workspace_bytes(2, 1) == 0 and lib.des_ga_order_runs_workspace_bytes(2, 2049) == 0


# ---- the wrappers ----------------------------------------------------------------------------------------------------
def test_ga_table_refuses_counts_out_of_range():
    from distributedes_b200.ops_ga_sweep import ga_table
    assert ga_table([1, 3], [1, 2], [3, 2], 3, 'cpu').tolist() == [[1, 1, 3, 0], [3, 2, 2, 0]]
    for args, match in (([[0], [0], [1]], 'run 0 has n_parents 0, not in \\[1, table_rows = 3\\]'),
                        ([[4], [0], [1]], 'run 0 has n_parents 4, not in \\[1, table_rows = 3\\]'),
                        ([[1, 2], [0, 3], [1, 1]], 'run 1 has n_elites 3, not in \\[0, n_parents = 2\\]'),
                        ([[1], [-1], [1]], 'run 0 has n_elites -1'),
                        ([[1], [0], [0]], 'run 0 has truncation 0, not in \\[1, table_rows = 3\\]'),
                        ([[1], [0], [4]], 'run 0 has truncation 4')):
        with pytest.raises(ValueError, match=match):
            ga_table(*args, 3, 'cpu')


def test_wrappers_check_their_tensors():
    from distributedes_b200 import ops_runs
    parents = torch.zeros((2, 3, P))
    ga = ops_runs.ga_table([1, 1], [0, 0], [3, 3], 3, 'cpu')
    hp = ops_runs.run_table([0, 1], 0.1, 0.0, 0.0, 0.0, 'cpu')
    kw = dict(hidden=16, horizon=5, repetitions=2, clip=2.0, run_size=4)
    with pytest.raises(RuntimeError, match='parents must be a 3-D tensor \\[R, table_rows, P\\]'):
        ops_runs.rollout_eval_ga_sweep(torch.zeros((6, P)), ga, hp, **kw)
    with pytest.raises(RuntimeError, match='parents has %d entries, the \\(3,16,1\\) MLP needs R x table_rows x P = %d'
                                           % (6 * (P + 1), 6 * P)):
        ops_runs.rollout_eval_ga_sweep(torch.zeros((2, 3, P + 1)), ga, hp, **kw)
    with pytest.raises(RuntimeError, match='ga must be torch.int32'):
        ops_runs.rollout_eval_ga_sweep(parents, ga.long(), hp, **kw)
    with pytest.raises(RuntimeError, match='ga has 4 entries, needs one 16-byte row per run: 8'):
        ops_runs.rollout_eval_ga_sweep(parents, ga[:1], hp, **kw)
    with pytest.raises(RuntimeError, match='hp has 40 entries, needs one 40-byte row per run: 80'):
        ops_runs.rollout_eval_ga_sweep(parents, ga, hp[:1], **kw)
    with pytest.raises(RuntimeError, match='episodes_out has 5 entries, needs 16'):
        ops_runs.rollout_eval_ga_sweep(parents, ga, hp, episodes_out=torch.zeros(5), **kw)
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops_runs.rollout_eval_ga_sweep(parents, ga, hp, **kw)
    with pytest.raises(RuntimeError, match='members must be torch.int32'):
        ops_runs.ga_rows_sweep(parents, ga, hp, generation=0, run_size=4, members=torch.zeros((2, 3)))
    with pytest.raises(RuntimeError, match='members has 4 entries, needs 6'):
        ops_runs.ga_rows_sweep(parents, ga, hp, generation=0, run_size=4, members=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(RuntimeError, match='out has %d entries, needs %d' % (P, 8 * P)):
        ops_runs.ga_rows_sweep(parents, ga, hp, generation=0, run_size=4, out=torch.zeros(P))
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops_runs.ga_rows_sweep(parents, ga, hp, generation=0, run_size=4)
    with pytest.raises(RuntimeError, match='fitness must be a 2-D tensor'):
        ops_runs.ga_order_runs(torch.zeros(8), ga, 3, workspace=torch.zeros(1))
    with pytest.raises(RuntimeError, match='out must be torch.int32'):
        ops_runs.ga_order_runs(torch.zeros((2, 4)), ga, 3, workspace=torch.zeros(1), out=torch.zeros((2, 3)))
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops_runs.ga_order_runs(torch.zeros((2, 4)), ga, 3, workspace=torch.zeros(1))
