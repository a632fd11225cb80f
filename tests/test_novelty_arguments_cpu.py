"""Novelty search's entry points and wrappers refuse bad arguments without a GPU: des_rollout_eval_bc everything
des_rollout_eval refuses (under its own name) and a NULL behaviour output; des_novelty and des_ns_shape their sizes,
ranges, NULL pointers, overlap and workspace, before any CUDA work; n = 0 does nothing.  The wrappers check their
tensors in ops._ptr."""
import ctypes as C

import pytest

torch = pytest.importorskip('torch')

from lib_fixture import lib  # noqa: F401
from oracle import nes_oracle as orc

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
H = 16
P = orc.param_count(3, H, 1)


def _msg(lib):
    return lib.des_last_error().decode()


# (env, H, repetitions, tape_len, member_offset, n_local, null pointers, workspace bytes with totals requested or None)
EVAL = {
    'bad_env': (1, 32, 10, 200, 0, 2, False, None),
    'bad_width': (0, 48, 10, 200, 0, 2, False, None),
    'reps_0': (0, 32, 0, 200, 0, 2, False, None),
    'reps_11': (0, 32, 11, 200, 0, 2, False, None),
    'tape_0': (0, 32, 10, 0, 0, 2, False, None),
    'neg_offset': (0, 32, 10, 200, -2, 2, False, None),
    'past_2^28': (0, 32, 10, 200, (1 << 28) - 2, 4, False, None),
    'null_count': (0, 32, 10, 200, 0, 2, True, None),
    'small_workspace': (0, 32, 10, 200, 0, 2, False, 8),
}


@pytest.mark.parametrize('case', list(EVAL))
def test_rollout_eval_bc_refuses_what_des_rollout_eval_refuses(lib, case):  # noqa: F811
    from distributedes_b200 import _lib
    env, h, reps, T, off, n, null, ws = EVAL[case]
    p, tot, dims = None if null else D, None if ws is None else D, _lib.Dims(3, h, 1, T)
    wsp = None if ws is None else D
    rc = lib.des_rollout_eval(p, None, tot, p, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0, wsp, ws or 0,
                              None)
    ev = (rc, _msg(lib))
    rc = lib.des_rollout_eval_bc(p, None, tot, p, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0, p, wsp,
                                 ws or 0, None)
    assert ev[0] != 0 and rc == ev[0]
    assert _msg(lib) == ev[1].replace('des_rollout_eval', 'des_rollout_eval_bc', 1)


def test_rollout_eval_bc_needs_its_output(lib):  # noqa: F811
    from distributedes_b200 import _lib
    dims = _lib.Dims(3, 16, 1, 200)
    assert lib.des_rollout_eval_bc(D, None, None, D, None, 0, dims, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 2, 0, None, None, 0,
                                   None) == -1
    assert _msg(lib) == 'des_rollout_eval_bc: NULL pointer'
    assert lib.des_rollout_eval_bc(None, None, None, None, None, 0, dims, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 0, 0, None,
                                   None, 0, None) == 0


@pytest.mark.parametrize('n,A,d,k,null,msg', [
    (-1, 5, 3, 10, False, 'des_novelty: n must be in [0, 2^31) (got -1)'),
    (1 << 31, 5, 3, 10, False, 'des_novelty: n must be in [0, 2^31) (got 2147483648)'),
    (4, 0, 3, 10, False, 'des_novelty: the archive must have [1, 2^31) rows (got 0)'),
    (4, 1 << 31, 3, 10, False, 'des_novelty: the archive must have [1, 2^31) rows (got 2147483648)'),
    (4, 5, 0, 10, False, 'des_novelty: d must be in [1, 32] (got 0)'),
    (4, 5, 33, 10, False, 'des_novelty: d must be in [1, 32] (got 33)'),
    (4, 5, 3, 0, False, 'des_novelty: k must be in [1, 32] (got 0)'),
    (4, 5, 3, 33, False, 'des_novelty: k must be in [1, 32] (got 33)'),
    (4, 5, 3, 10, True, 'des_novelty: NULL pointer'),
])
def test_novelty_refuses(lib, n, A, d, k, null, msg):  # noqa: F811
    p = None if null else D
    assert lib.des_novelty(p, p, n, p, A, d, k, None) == -1
    assert _msg(lib) == msg


def test_novelty_takes_an_archive_of_up_to_int32_max_rows(lib):  # noqa: F811
    # the largest archive passes the range checks (the NULL pointer is what stops this call), one row more does not
    assert lib.des_novelty(None, None, 4, None, (1 << 31) - 1, 1, 10, None) == -1
    assert _msg(lib) == 'des_novelty: NULL pointer'
    assert lib.des_novelty(None, None, 4, None, 1 << 31, 1, 10, None) == -1
    assert _msg(lib) == 'des_novelty: the archive must have [1, 2^31) rows (got 2147483648)'


def test_novelty_of_no_queries_does_nothing(lib):  # noqa: F811
    assert lib.des_novelty(None, None, 0, None, 5, 3, 10, None) == 0


@pytest.mark.parametrize('N,w,null,ws,rc,msg', [
    (1, 0.5, False, None, -1, 'des_ns_shape: N=1, need 2 <= N < 2^31'),
    (4, -0.1, False, None, -1, 'des_ns_shape: reward_weight must be in [0, 1] (got -0.1)'),
    (4, 1.5, False, None, -1, 'des_ns_shape: reward_weight must be in [0, 1] (got 1.5)'),
    (4, float('nan'), False, None, -1, 'des_ns_shape: reward_weight must be in [0, 1] (got nan)'),
    (4, 0.5, True, None, -1, 'des_ns_shape: NULL pointer'),
    (4, 0.5, False, 8, -4, None),
])
def test_ns_shape_refuses(lib, N, w, null, ws, rc, msg):  # noqa: F811
    out, f, nov = (None, None, None) if null else (C.c_void_p(1 << 20), C.c_void_p(2 << 20), C.c_void_p(3 << 20))
    assert lib.des_ns_shape(out, f, nov, N, w, D if ws else None, ws or 0, None) == rc
    need = lib.des_ns_shape_workspace_bytes(N)
    assert _msg(lib) == (msg or 'des_ns_shape: workspace 8 B < required %d B' % need)


def test_ns_shape_refuses_an_output_over_an_input(lib):  # noqa: F811
    base = 1 << 20
    for out, f, nov in ((base, base, 2 * base), (base + 8, base, 2 * base), (2 * base - 8, base * 3, 2 * base)):
        rc = lib.des_ns_shape(C.c_void_p(out), C.c_void_p(f), C.c_void_p(nov), 4, 0.5, D, 1 << 30, None)
        assert rc == -1 and _msg(lib) == 'des_ns_shape: shaped_out overlaps an input'


def test_ns_shape_workspace_covers_both_ranks(lib):  # noqa: F811
    for N in (2, 2048, 2049, 65536):
        assert lib.des_ns_shape_workspace_bytes(N) >= 4 * N + lib.des_rank_workspace_bytes(N, N)
    assert lib.des_ns_shape_workspace_bytes(1) == 0


def test_wrappers_check_their_tensors():
    from distributedes_b200 import ops
    q, a = torch.zeros((4, 3)), torch.zeros((5, 3))
    with pytest.raises(RuntimeError, match='queries must be a 2-D tensor'):
        ops.novelty(torch.zeros(3), a, 10)
    with pytest.raises(RuntimeError, match='archive must be a 2-D tensor'):
        ops.novelty(q, torch.zeros(3), 10)
    with pytest.raises(RuntimeError, match='archive must be torch.float32'):
        ops.novelty(q, a.double(), 10)
    with pytest.raises(RuntimeError, match='archive rows have 2 entries, the queries 3'):
        ops.novelty(q, torch.zeros((5, 2)), 10)
    with pytest.raises(RuntimeError, match='queries must be torch.float32'):
        ops.novelty(q.double(), a, 10)
    with pytest.raises(RuntimeError, match='out has 3 entries, needs 4'):
        ops.novelty(q, a, 10, out=torch.zeros(3))
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.novelty(q, a, 10)
    f = torch.zeros(4)
    with pytest.raises(RuntimeError, match='fitness must be torch.float32'):
        ops.ns_shape(f.double(), f, 0.5, workspace=torch.zeros(1))
    with pytest.raises(RuntimeError, match='novelty has 3 entries, needs 4'):
        ops.ns_shape(f, torch.zeros(3), 0.5, workspace=torch.zeros(1))
    with pytest.raises(RuntimeError, match='out must be torch.float32'):
        ops.ns_shape(f, f.clone(), 0.5, workspace=torch.zeros(1), out=torch.zeros(4, dtype=torch.float64))
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.ns_shape(f, f.clone(), 0.5, workspace=torch.zeros(1))
    kw = dict(hidden=H, horizon=5, repetitions=2, sigma=0.1, clip=2.0, seed=1, n_local=3)
    theta = torch.zeros(P)
    with pytest.raises(RuntimeError, match='bc_out has 6 entries, needs 9'):
        ops.rollout_eval_bc(theta, bc_out=torch.zeros((2, 3)), **kw)
    with pytest.raises(RuntimeError, match='bc_out must be torch.float32'):
        ops.rollout_eval_bc(theta, bc_out=torch.zeros((3, 3), dtype=torch.float64), **kw)
    with pytest.raises(RuntimeError, match='theta has %d entries' % (P + 1)):
        ops.rollout_eval_bc(torch.zeros(P + 1), bc_out=torch.zeros((3, 3)), **kw)
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.rollout_eval_bc(theta, bc_out=torch.zeros((3, 3)), **kw)
