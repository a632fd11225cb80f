"""The argument checks of the genetic algorithm's novelty-search entry points, without a GPU.  Every input here is
answered before any CUDA work, so the library answers it on any machine; each case pins the status code and the exact
message.

  - des_rollout_eval_ga_bc refuses everything des_rollout_eval_ga refuses, with the message under its own name, and a
    NULL bc_out; n_local == 0 does nothing and accepts NULL pointers;
  - des_ns_ga_order refuses N outside [2, 2^24], T outside [1, N], a weight outside [0, 1], NULL pointers and a short
    workspace; its workspace covers des_ns_shape's and five vectors;
  - the wrappers check their tensors in ops._ptr.
"""
import ctypes as C

import pytest

torch = pytest.importorskip('torch')

from lib_fixture import lib  # noqa: F401,E402
from oracle import nes_oracle as orc  # noqa: E402

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
H = 16
P = orc.param_count(3, H, 1)


def _msg(lib):
    return lib.des_last_error().decode()


# des_rollout_eval's cases (test_ga_cpu.EVAL) and des_rollout_eval_ga's own: (env, H, repetitions, tape_len,
# member_offset, n_local, n_parents, n_elites, noiseless, null pointers, workspace bytes with totals requested or None)
GA_CASES = {
    'bad_env': (1, 32, 10, 200, 0, 2, 2, 1, 0, False, None),
    'bad_width': (0, 48, 10, 200, 0, 2, 2, 1, 0, False, None),
    'reps_0': (0, 32, 0, 200, 0, 2, 2, 1, 0, False, None),
    'reps_11': (0, 32, 11, 200, 0, 2, 2, 1, 0, False, None),
    'tape_0': (0, 32, 10, 0, 0, 2, 2, 1, 0, False, None),
    'neg_offset': (0, 32, 10, 200, -2, 2, 2, 1, 0, False, None),
    'past_2^28': (0, 32, 10, 200, (1 << 28) - 2, 4, 2, 1, 0, False, None),
    'null_count': (0, 32, 10, 200, 0, 2, 2, 1, 0, True, None),
    'small_workspace': (0, 32, 10, 200, 0, 2, 2, 1, 0, False, 8),
    'noiseless': (0, 16, 10, 200, 0, 2, 2, 0, 1, False, None),
    'n_parents_0': (0, 16, 10, 200, 0, 2, 0, 0, 0, False, None),
    'elites_past_parents': (0, 16, 10, 200, 0, 2, 2, 3, 0, False, None),
    'elites_negative': (0, 16, 10, 200, 0, 2, 2, -1, 0, False, None),
}


@pytest.mark.parametrize('case', list(GA_CASES))
def test_rollout_eval_ga_bc_refuses_what_des_rollout_eval_ga_refuses(lib, case):  # noqa: F811
    from distributedes_b200 import _lib
    env, h, reps, T, off, n, n_parents, n_elites, noiseless, null, ws = GA_CASES[case]
    p, tot, dims = None if null else D, None if ws is None else D, _lib.Dims(3, h, 1, T)
    wsp = None if ws is None else D
    rc = lib.des_rollout_eval_ga(p, None, tot, p, n_parents, n_elites, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None,
                                 off, n, noiseless, wsp, ws or 0, None)
    ev = (rc, _msg(lib))
    rc = lib.des_rollout_eval_ga_bc(p, None, tot, p, n_parents, n_elites, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None,
                                    off, n, noiseless, p, wsp, ws or 0, None)
    assert ev[0] != 0 and rc == ev[0]
    want = ev[1].replace('des_rollout_eval_ga', 'des_rollout_eval_ga_bc', 1)
    if case == 'noiseless':
        want = want.replace('use des_rollout_eval on it', 'use des_rollout_eval_bc on it')
    assert _msg(lib) == want


def test_rollout_eval_ga_bc_needs_its_behaviour_buffer(lib):  # noqa: F811
    from distributedes_b200 import _lib
    dims = _lib.Dims(3, 16, 1, 200)
    rc = lib.des_rollout_eval_ga_bc(D, None, None, D, 2, 1, None, 0, dims, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 2, 0, None,
                                    None, 0, None)
    assert rc == -1 and _msg(lib) == 'des_rollout_eval_ga_bc: NULL pointer'
    assert lib.des_rollout_eval_ga_bc(None, None, None, None, 1, 0, None, 0, dims, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 0, 0,
                                      None, None, 0, None) == 0


@pytest.mark.parametrize('N,T,w,null,ws,rc,msg', [
    (1, 1, 0.5, False, None, -1, 'des_ns_ga_order: N=1, need 2 <= N <= 2^24 (above, two centered ranks can round to '
                                 'one fp32 key)'),
    ((1 << 24) + 1, 2, 0.5, False, None, -1, 'des_ns_ga_order: N=16777217, need 2 <= N <= 2^24 (above, two centered '
                                             'ranks can round to one fp32 key)'),
    (4, 0, 0.5, False, None, -1, 'des_ns_ga_order: T must be in [1, N = 4] (got 0)'),
    (4, 5, 0.5, False, None, -1, 'des_ns_ga_order: T must be in [1, N = 4] (got 5)'),
    (4, 2, -0.1, False, None, -1, 'des_ns_ga_order: reward_weight must be in [0, 1] (got -0.1)'),
    (4, 2, 1.5, False, None, -1, 'des_ns_ga_order: reward_weight must be in [0, 1] (got 1.5)'),
    (4, 2, float('nan'), False, None, -1, 'des_ns_ga_order: reward_weight must be in [0, 1] (got nan)'),
    (4, 2, 0.5, True, None, -1, 'des_ns_ga_order: NULL pointer'),
    (4, 2, 0.5, False, 8, -4, None),
])
def test_ns_ga_order_refuses(lib, N, T, w, null, ws, rc, msg):  # noqa: F811
    p = None if null else D
    assert lib.des_ns_ga_order(p, p, p, N, T, w, D if ws else None, ws or 0, None) == rc
    need = lib.des_ns_ga_order_workspace_bytes(N)
    assert _msg(lib) == (msg or 'des_ns_ga_order: workspace 8 B < required %d B' % need)


def test_ns_ga_order_takes_2_to_the_24_members(lib):  # noqa: F811
    N = 1 << 24
    need = lib.des_ns_ga_order_workspace_bytes(N)
    assert lib.des_ns_ga_order(D, D, D, N, N, 0.5, D, need - 1, None) == -4       # past the size checks
    assert _msg(lib) == 'des_ns_ga_order: workspace %d B < required %d B' % (need - 1, need)


def test_ns_ga_order_workspace_covers_the_shaping_and_the_rank(lib):  # noqa: F811
    for N in (2, 2048, 2049, 65536):
        assert lib.des_ns_ga_order_workspace_bytes(N) >= 5 * 4 * N + lib.des_ns_shape_workspace_bytes(N)
        assert lib.des_ns_shape_workspace_bytes(N) >= lib.des_rank_workspace_bytes(N, N)
    assert lib.des_ns_ga_order_workspace_bytes(1) == 0


def test_wrappers_check_their_tensors():
    from distributedes_b200 import ops
    parents = torch.zeros((2, P))
    kw = dict(hidden=H, horizon=5, repetitions=2, sigma=0.1, clip=2.0, seed=1, n_local=3)
    with pytest.raises(RuntimeError, match='parents must be a 2-D tensor'):
        ops.rollout_eval_ga_bc(torch.zeros(P), 0, bc_out=torch.zeros((3, 3)), **kw)
    with pytest.raises(RuntimeError, match='parents has %d entries, the \\(3,16,1\\) MLP needs n_parents x P = %d'
                                           % (2 * (P + 1), 2 * P)):
        ops.rollout_eval_ga_bc(torch.zeros((2, P + 1)), 0, bc_out=torch.zeros((3, 3)), **kw)
    with pytest.raises(RuntimeError, match='bc_out has 6 entries, needs 9'):
        ops.rollout_eval_ga_bc(parents, 0, bc_out=torch.zeros((2, 3)), **kw)
    with pytest.raises(RuntimeError, match='bc_out must be torch.float32'):
        ops.rollout_eval_ga_bc(parents, 0, bc_out=torch.zeros((3, 3), dtype=torch.float64), **kw)
    with pytest.raises(RuntimeError, match='bc_out must be a torch.Tensor'):
        ops.rollout_eval_ga_bc(parents, 0, bc_out=None, **kw)
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.rollout_eval_ga_bc(parents, 0, bc_out=torch.zeros((3, 3)), **kw)
    with pytest.raises(RuntimeError, match='out must be torch.int32'):
        ops.ns_ga_order(torch.zeros(4), torch.zeros(4), 0.5, 2, workspace=torch.zeros(1), out=torch.zeros(2))
    with pytest.raises(RuntimeError, match='fitness must be torch.float32'):
        ops.ns_ga_order(torch.zeros(4, dtype=torch.float64), torch.zeros(4), 0.5, 2, workspace=torch.zeros(1))
    with pytest.raises(RuntimeError, match='novelty has 3 entries, needs 4'):
        ops.ns_ga_order(torch.zeros(4), torch.zeros(3), 0.5, 2, workspace=torch.zeros(1))
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.ns_ga_order(torch.zeros(4), torch.zeros(4), 0.5, 2, workspace=torch.zeros(1))
