"""The argument checks of the CMA-ES sweep entry points (des_noise_fill_sweep, des_rollout_eval_solutions_sweep,
des_cma_rank_mu_runs, des_cma_cov_apply_runs) and of their wrappers in ops_cma_sweep, without a GPU.  The entry points
answer every case before any CUDA work: the batch shape, the 2048-member run limit, NULL pointers (the table included),
the widths and repetitions of the rollout, a workspace too small, and n_runs 0 with NULL pointers.  The wrappers check
every tensor they pass before they reject a CPU tensor, as ops does; ops_runs lists them."""
import ctypes as C

import pytest
import torch

from distributedes_b200 import ops_cma_sweep, ops_runs
from distributedes_b200._lib import Dims
from lib_fixture import lib  # noqa: F401

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
NF, RO, RM, CA = 'des_noise_fill_sweep', 'des_rollout_eval_solutions_sweep', 'des_cma_rank_mu_runs', 'des_cma_cov_apply_runs'


def _p(null):
    return None if null else D


def noise(lib, R=2, N=4, P=353, null=False, null_hp=False):
    return lib.des_noise_fill_sweep(_p(null), R, N, P, _p(null_hp), 0, 1, None)


def rollout(lib, R=2, N=4, H=16, reps=10, horizon=200, null=False, null_hp=False, totals=False, ws_bytes=0, env=0,
            d0=3):
    return lib.des_rollout_eval_solutions_sweep(_p(null), None, D if totals else None, _p(null), None, env,
                                                Dims(d0, H, 1, horizon), reps, 2.0, _p(null_hp), 0, R, N,
                                                D if ws_bytes else None, ws_bytes, None)


def rank_mu(lib, R=2, lam=64, n=353, null=False, ws_bytes=0):
    return lib.des_cma_rank_mu_runs(_p(null), _p(null), _p(null), R, lam, n, D if ws_bytes else None, ws_bytes, None)


def cov(lib, R=2, n=353, null=False, null_decay=False):
    return lib.des_cma_cov_apply_runs(_p(null), _p(null), None, _p(null_decay), 1e-3, 1e-2, R, n, None)


PINS = {}
for who, fn in ((NF, noise), (RO, rollout)):
    PINS[who, 'neg_runs'] = (fn, dict(R=-1), -1, '%s: need n_runs >= 0 and run_size >= 1 (got -1 and 4)' % who)
    PINS[who, 'size_0'] = (fn, dict(N=0), -1, '%s: need n_runs >= 0 and run_size >= 1 (got 2 and 0)' % who)
    PINS[who, 'size_2049'] = (fn, dict(N=2049), -5, '%s: run_size 2049 > 2048: batches hold runs of up to 2048 members '
                                                    '(a larger population fills the GPU alone)' % who)
    PINS[who, 'past_2^28'] = (fn, dict(R=(1 << 28) // 64 + 1, N=64), -1, '%s: n_runs x run_size = %d x 64 members, '
                                                                         'past 2^28' % (who, (1 << 28) // 64 + 1))
    PINS[who, 'null_table'] = (fn, dict(null_hp=True), -1, '%s: NULL pointer' % who)
    PINS[who, 'null_runs'] = (fn, dict(null=True), -1, '%s: NULL pointer' % who)
    PINS[who, 'null_zero_runs'] = (fn, dict(R=0, null=True, null_hp=True), 0, None)
PINS[NF, 'P_0'] = (noise, dict(P=0), -1, '%s: bad size P=0' % NF)
for case, kw, msg in (
        ('hidden_48', dict(H=48), 'hidden must be 16 or a multiple of 32, <= 128 (got 48)'),
        ('hidden_256', dict(H=256), 'hidden must be 16 or a multiple of 32, <= 128 (got 256)'),
        ('reps_0', dict(reps=0), 'repetitions must be in [1, 10] (one warp each)'),
        ('reps_11', dict(reps=11), 'repetitions must be in [1, 10] (one warp each)'),
        ('horizon_0', dict(horizon=0), 'episode length (dims.tape_len) must be >= 1'),
        ('env_1', dict(env=1), 'unknown environment 1 (0 = Pendulum-v0)'),
        ('state_dim_4', dict(d0=4), 'Pendulum-v0 has state_dim 3, action_dim 1')):
    PINS[RO, case] = (rollout, kw, -1, '%s: %s' % (RO, msg))
PINS[RO, 'workspace_small'] = (rollout, dict(totals=True, ws_bytes=8 * 7 * 8 - 1), -4,
                               '%s: workspace 447 B < required 448 B' % RO)
PINS[RO, 'workspace_missing'] = (rollout, dict(totals=True), -4, '%s: workspace 0 B < required 448 B' % RO)
PINS[RM, 'neg_runs'] = (rank_mu, dict(R=-1), -1, '%s: bad sizes n_runs=-1 lambda=64 n=353' % RM)
PINS[RM, 'neg_lambda'] = (rank_mu, dict(lam=-1), -1, '%s: bad sizes n_runs=2 lambda=-1 n=353' % RM)
PINS[RM, 'n_0'] = (rank_mu, dict(n=0), -1, '%s: bad sizes n_runs=2 lambda=64 n=0' % RM)
PINS[RM, 'n_too_large'] = (rank_mu, dict(n=46340 * 16 + 1), -1, '%s: n too large' % RM)
PINS[RM, 'null'] = (rank_mu, dict(null=True), -1, '%s: NULL pointer' % RM)
PINS[RM, 'past_2^40'] = (rank_mu, dict(R=1 << 21, n=1024), -1, '%s: n_runs x n x n or n_runs x lambda x n (2097152, 64, '
                                                                 '1024) floats past 2^40' % RM)
PINS[RM, 'lambda_past_2^40'] = (rank_mu, dict(lam=1 << 62, n=1024), -1, '%s: n_runs x n x n or n_runs x lambda x n (2, %d, '
                                                                        '1024) floats past 2^40' % (RM, 1 << 62))
PINS[CA, 'past_2^40'] = (cov, dict(R=1 << 21, n=1024), -1, '%s: n_runs x n x n past 2^40' % CA)
PINS[RM, 'null_zero_runs'] = (rank_mu, dict(R=0, null=True), 0, None)
PINS[RM, 'workspace_missing'] = (rank_mu, dict(n=2048), -4, None)
PINS[RM, 'workspace_small'] = (rank_mu, dict(n=4481, ws_bytes=1024), -4, None)
PINS[CA, 'neg_runs'] = (cov, dict(R=-1), -1, '%s: bad sizes n_runs=-1 n=353' % CA)
PINS[CA, 'n_0'] = (cov, dict(n=0), -1, '%s: bad sizes n_runs=2 n=0' % CA)
PINS[CA, 'null'] = (cov, dict(null=True), -1, '%s: NULL pointer' % CA)
PINS[CA, 'null_decay'] = (cov, dict(null_decay=True), -1, '%s: NULL pointer' % CA)
PINS[CA, 'null_zero_runs'] = (cov, dict(R=0, null=True, null_decay=True), 0, None)


@pytest.mark.parametrize('entry,case', sorted(PINS))
def test_cma_sweep_entry_point_rejects_before_cuda_work(lib, entry, case):  # noqa: F811
    fn, kw, status, message = PINS[entry, case]
    assert fn(lib, **kw) == status
    if message is not None:
        assert lib.des_last_error().decode() == message


def test_rank_mu_runs_workspace_is_one_runs_tensor_core_workspace(lib):  # noqa: F811
    for lam, n in ((64, 353), (16, 2048), (100, 4481)):
        assert lib.des_cma_rank_mu_runs_workspace_bytes(5, lam, n) == lib.des_cma_rank_mu_workspace_bytes(n, lam)
    assert lib.des_cma_rank_mu_runs_workspace_bytes(5, 64, 353) == 0
    assert lib.des_cma_rank_mu_runs_workspace_bytes(0, 64, 4481) == 0
    msg = '%s: workspace 1024 B < required %d B' % (RM, lib.des_cma_rank_mu_workspace_bytes(4481, 64))
    assert rank_mu(lib, n=4481, ws_bytes=1024) == -4 and lib.des_last_error().decode() == msg


# ---- the wrappers ----------------------------------------------------------------------------------------------------
R, N, P, n = 3, 4, 353, 5
F32, F64, U8 = torch.float32, torch.float64, torch.uint8


def _hp(R=R):
    from distributedes_b200.ops_sweep import run_table
    return run_table(list(range(R)), 1.0, 0.0, 0.0, 0.0, 'cpu', runs=R)


WRAPPERS = {
    'noise_hp_dtype': (lambda: ops_cma_sweep.noise_fill_sweep(torch.zeros((R, 40)), N, P, 0),
                       'hp must be torch.uint8, got torch.float32'),
    'noise_hp_rows': (lambda: ops_cma_sweep.noise_fill_sweep(_hp()[:, :39].contiguous(), N, P, 0),
                      'hp has 117 entries, needs one 40-byte row per run: 120'),
    'noise_out_count': (lambda: ops_cma_sweep.noise_fill_sweep(_hp(), N, P, 0, out=torch.empty((R * N, P - 1))),
                        'out has %d entries, needs %d' % (R * N * (P - 1), R * N * P)),
    'noise_cpu': (lambda: ops_cma_sweep.noise_fill_sweep(_hp(), N, P, 0), 'hp is a CPU tensor'),
    'rollout_rows_dtype': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P), dtype=F64), _hp(),
                                                                             hidden=16, clip=2.0, run_size=N),
                           'rows must be torch.float32'),
    'rollout_rows_count': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P + 1)), _hp(),
                                                                             hidden=16, clip=2.0, run_size=N),
                           'rows has %d entries, the \\(3,16,1\\) MLP needs n x P = %d' % (R * N * (P + 1), R * N * P)),
    'rollout_not_whole_runs': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N + 1, P)), _hp(),
                                                                                 hidden=16, clip=2.0, run_size=N),
                               'rows has 13 rows, not a whole number of runs of run_size 4'),
    'rollout_stats_count': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P)), _hp(), hidden=16,
                                                                              clip=2.0, run_size=N,
                                                                              obs_stats=torch.zeros(7)),
                            'obs_stats has 7 entries, needs 21'),
    'rollout_totals_dtype': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P)), _hp(),
                                                                               hidden=16, clip=2.0, run_size=N,
                                                                               totals_out=torch.zeros((R, 7))),
                             'totals_out must be torch.float64'),
    'rollout_table_runs': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P)), _hp(2),
                                                                             hidden=16, clip=2.0, run_size=N),
                           'hp has 80 entries, needs one 40-byte row per run: 120'),
    'rollout_cpu': (lambda: ops_cma_sweep.rollout_eval_solutions_sweep(torch.zeros((R * N, P)), _hp(), hidden=16,
                                                                      clip=2.0, run_size=N), 'rows is a CPU tensor'),
    'rank_mu_2d': (lambda: ops_cma_sweep.cma_rank_mu_runs(torch.zeros((N, n)), torch.zeros((R, N))),
                   'Y must be a 3-D tensor'),
    'rank_mu_w_count': (lambda: ops_cma_sweep.cma_rank_mu_runs(torch.zeros((R, N, n)), torch.zeros((R, N + 1))),
                        'w has 15 entries, needs 12'),
    'rank_mu_w_dtype': (lambda: ops_cma_sweep.cma_rank_mu_runs(torch.zeros((R, N, n)), torch.zeros((R, N), dtype=F64)),
                        'w must be torch.float32'),
    'rank_mu_out_count': (lambda: ops_cma_sweep.cma_rank_mu_runs(torch.zeros((R, N, n)), torch.zeros((R, N)),
                                                                 out=torch.zeros((R, n, n - 1))),
                          'out has 60 entries, needs 75'),
    'rank_mu_cpu': (lambda: ops_cma_sweep.cma_rank_mu_runs(torch.zeros((R, N, n)), torch.zeros((R, N))),
                    'Y is a CPU tensor'),
    'cov_not_square': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n + 1)), torch.zeros((R, n, n)), None,
                                                                torch.ones(R, dtype=F64), c1=0.1, cmu=0.1),
                       'Cmat must be \\[R, n, n\\]'),
    'cov_dC_count': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n)), torch.zeros((R, n, n - 1)), None,
                                                              torch.ones(R, dtype=F64), c1=0.1, cmu=0.1),
                     'dC has 60 entries, needs 75'),
    'cov_pc_count': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n)), torch.zeros((R, n, n)),
                                                              torch.zeros(n), torch.ones(R, dtype=F64), c1=0.1, cmu=0.1),
                     'pc has 5 entries, needs 15'),
    'cov_decay_dtype': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n)), torch.zeros((R, n, n)), None,
                                                                 torch.ones(R), c1=0.1, cmu=0.1),
                        'decay must be torch.float64'),
    'cov_decay_count': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n)), torch.zeros((R, n, n)), None,
                                                                 torch.ones(R + 1, dtype=F64), c1=0.1, cmu=0.1),
                        'decay has 4 entries, needs 3'),
    'cov_cpu': (lambda: ops_cma_sweep.cma_cov_apply_runs(torch.zeros((R, n, n)), torch.zeros((R, n, n)), None,
                                                         torch.ones(R, dtype=F64), c1=0.1, cmu=0.1),
                'Cmat is a CPU tensor'),
}


@pytest.mark.parametrize('case', sorted(WRAPPERS))
def test_cma_sweep_wrappers_check_every_tensor_before_the_device(case):
    fn, match = WRAPPERS[case]
    with pytest.raises(RuntimeError, match=match):
        fn()


def test_ops_runs_lists_the_cma_sweep_ops():
    for name in ('noise_fill_sweep', 'rollout_eval_solutions_sweep', 'cma_rank_mu_runs', 'cma_cov_apply_runs'):
        assert getattr(ops_runs, name) is getattr(ops_cma_sweep, name)
