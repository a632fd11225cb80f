"""CPU-only checks: the C-ABI library loads and exports every symbol include/des_b200.h declares, the ctypes
signature table covers the header, argument validation happens before any CUDA work, host helpers."""
import os
import re
import subprocess

import numpy as np
import pytest

from lib_fixture import lib  # noqa: F401

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, 'include', 'des_b200.h')


def header_symbols():
    txt = open(HEADER).read()
    return sorted(set(re.findall(r'DES_API\s+[\w\s\*]+?\b(des_\w+)\s*\(', txt)))


def test_header_declares_the_expected_surface():
    syms = header_symbols()
    assert len(syms) >= 25
    for must in ['des_nes_eval', 'des_centered_rank', 'des_nes_grad_partial', 'des_nes_apply', 'des_cma_rank_mu',
                 'des_cma_cov_apply', 'des_noise_fill', 'des_session_generation_host', 'des_last_error']:
        assert must in syms


def test_library_exports_every_header_symbol(lib):
    from distributedes_b200 import _lib
    out = subprocess.run(['nm', '-D', '--defined-only', _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r' T (des_\w+)', out))
    missing = [s for s in header_symbols() if s not in exported]
    assert not missing, missing
    # and nothing but the C ABI leaks out of the shared object
    assert all(s.startswith('des_') for s in re.findall(r' T (\w+)', out))


def test_ctypes_table_matches_header(lib):
    from distributedes_b200 import _lib
    assert sorted(_lib.SIGNATURES) == header_symbols()


def test_struct_layouts_match_header(lib):
    import ctypes as C
    from distributedes_b200 import _lib
    assert C.sizeof(_lib.Dims) == 16 and C.sizeof(_lib.Opt) == 48 and C.sizeof(_lib.State) == 32


def test_pure_functions_and_workspace_sizes_without_gpu(lib):
    assert lib.des_param_count(3, 64, 1) == 4481          # SURVEY table, confirmed on StandardFCNet(3,1,64)
    assert lib.des_param_count(24, 64, 4) == 6020
    assert lib.des_param_count(24, 256, 4) == 73220
    assert lib.des_param_count(0, 64, 1) < 0
    assert lib.des_rank_workspace_bytes(2048, 1000) == 4000            # counting rank: one int32 count per member
    assert lib.des_rank_workspace_bytes(4096, 16) > 3 * 4096 * 4       # bucketed rank: keys and grouped keys/indices of all N
    # the rank-mu kernel is picked from n alone: only the tensor-core shapes need a workspace
    from distributedes_b200 import ops
    assert ops.CMA_TC_MIN_N == 2048
    assert lib.des_cma_rank_mu_workspace_bytes(2047, 64) == 0 < lib.des_cma_rank_mu_workspace_bytes(2048, 64)
    assert lib.des_cma_rank_mu_workspace_bytes(4096, 0) == 0
    assert lib.des_grad_workspace_bytes(0, 10) == 0
    assert lib.des_grad_workspace_bytes(4096, 6020) >= 6020 * 4
    assert b'sm_90a' in lib.des_version()


def test_argument_validation_precedes_cuda(lib):
    """Bad arguments are rejected with DES_ERR_INVALID_ARGUMENT and a message, with no GPU present."""
    import ctypes as C
    from distributedes_b200 import _lib
    rc = lib.des_centered_rank(None, None, None, 1, 0, 1, None, 0, None)
    assert rc == -1 and b'N >= 2' in lib.des_last_error()
    rc = lib.des_nes_eval(None, None, None, None, _lib.Dims(0, 64, 1, 8), 0.1, 1.0, 0, 0, None, 0, 1, 0, None, 0, None)
    assert rc == -1 and b'bad dims' in lib.des_last_error()
    rc = lib.des_nes_eval(None, None, None, None, _lib.Dims(3, 64, 1, 8), 0.1, 1.0, 0, 0, None, 0, 1, 0, None, 0, None)
    assert rc == -1 and b'NULL' in lib.des_last_error()
    rc = lib.des_nes_grad_partial(None, None, 4, 10, 0, 0, None, 0, None, 0, None)
    assert rc == -1
    # a short workspace is DES_ERR_WORKSPACE, never a quiet switch to another kernel (dummy pointers: nothing is launched)
    dummy = C.c_void_p(256)
    short = lib.des_rank_workspace_bytes(2048, 4096)                   # what the counting rank would need
    rc = lib.des_centered_rank(dummy, None, dummy, 4096, 0, 4096, dummy, short, None)
    assert rc == -4 and b'workspace' in lib.des_last_error()
    rc = lib.des_cma_rank_mu(dummy, dummy, dummy, 64, 2048, 0, None, 0, None)
    assert rc == -4 and b'workspace' in lib.des_last_error()
    sess = C.c_void_p()
    theta = (C.c_float * 4481)()
    rc = lib.des_session_create(C.byref(sess), 0, _lib.Dims(3, 64, 1, 8), 1, 0, 1, _lib.Opt(0.1, 0.1, 0.005, 0.9, 0.999, 1e-8),
                                2.0, 0, 0, theta)
    assert rc == -1 and b'population split' in lib.des_last_error()
    with pytest.raises(RuntimeError, match='status -1'):
        _lib.check(rc, 'des_session_create')


def test_no_cuda_device_is_an_error_not_a_fallback(lib):
    import ctypes as C
    import torch
    from distributedes_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip('this check is for the GPU-less container')
    assert lib.des_device_count() == 0
    sess = C.c_void_p()
    theta = (C.c_float * 4481)()
    rc = lib.des_session_create(C.byref(sess), 0, _lib.Dims(3, 64, 1, 8), 16, 0, 16,
                                _lib.Opt(0.1, 0.1, 0.005, 0.9, 0.999, 1e-8), 2.0, 0, 0, theta)
    assert rc == -3 and b'no CPU fallback' in lib.des_last_error()
    from distributedes_b200 import ops
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.centered_rank(torch.zeros(4))
    from distributedes_b200.utils import fitness_shift
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        fitness_shift([1.0, 2.0])


def test_host_model_codec_matches_reference_layout(golden_dir):
    """model.py get_weight/set_weight: flat layout pinned by the reference's named parameters."""
    from distributedes_b200.model import StandardFCNet, param_count
    g = np.load(os.path.join(golden_dir, 'forward.npz'))
    for tag in ('pend', 'b64', 'b256'):
        d0, H, A, _ = (int(v) for v in g[tag + '_dims'])
        net = StandardFCNet(d0, A, H)
        assert net.get_weight().size == param_count(d0, H, A)
        net.set_weight(g[tag + '_flat'].astype(np.float64))
        assert net.get_weight().dtype == np.float32 and np.array_equal(net.get_weight(), g[tag + '_flat'])
        for ours, name in zip(net.parameters(), ('fc1w', 'fc1b', 'fc2w', 'fc2b', 'fc3w', 'fc3b')):
            assert np.array_equal(ours, g[tag + '_' + name])
        with pytest.raises(AssertionError):
            net.set_weight(np.zeros(3))


def test_shard_bounds_cover_population():
    from distributedes_b200.engine import shard_bounds
    for N in (2, 7, 16, 4096, 65536, 65537):
        for G in (1, 2, 3, 8):
            spans = [shard_bounds(N, G, r) for r in range(G)]
            assert spans[0][0] == 0 and sum(n for _, n in spans) == N
            for (s0, n0), (s1, _) in zip(spans, spans[1:]):
                assert s0 + n0 == s1
            assert max(n for _, n in spans) - min(n for _, n in spans) <= 1
    with pytest.raises(ValueError):
        shard_bounds(10, 2, 2)


def test_config_surface_matches_reference_attributes():
    from distributedes_b200.config import BipedalWalkerConfig, PendulumConfig
    c = PendulumConfig(64)
    for attr in ['task', 'env_fn', 'repetitions', 'test_repetitions', 'action_dim', 'state_dim', 'hidden_size',
                 'model_fn', 'initial_weight', 'reward_to_fitness', 'pop_size', 'num_workers', 'max_steps', 'opt',
                 'weight_decay', 'action_noise_std', 'tag', 'action_clip', 'target', 'sigma', 'learning_rate']:
        assert hasattr(c, attr), attr
    assert (c.state_dim, c.action_dim, len(c.initial_weight)) == (3, 1, 4481)
    assert c.pop_size == 30 and c.weight_decay == 0.005 and c.opt.beta1 == 0.9       # config.py:18-22
    assert np.array_equal(c.action_clip(np.asarray([-3.0, 0.5, 3.0])), [-2.0, 0.5, 2.0])   # config.py:29
    b = BipedalWalkerConfig(64)
    assert (b.state_dim, b.action_dim, len(b.initial_weight)) == (24, 4, 6020)


def test_closed_loop_config_and_packed_cma_validation_without_gpu(lib):
    """ClosedLoopPendulumConfig keeps the reference's PendulumConfig values (config.py:8-9, 26-31); the device environment
    has no host-side step; des_rollout_eval / the packed CMA entry points validate their arguments before touching CUDA."""
    from distributedes_b200 import _lib
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(64)
    assert (c.task, c.state_dim, c.action_dim, len(c.initial_weight)) == ('Pendulum-v0', 3, 1, 4481)
    assert (c.repetitions, c.test_repetitions, c.clip, c.closed_loop, c.normalize_obs) == (10, 10, 2.0, True, True)
    with pytest.raises(RuntimeError, match='stepped on the GPU'):
        c.env_fn().reset()
    d = _lib.Dims(3, 64, 1, 200)
    rc = lib.des_rollout_eval(None, None, None, None, None, 7, d, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 4, 0, None, 0, None)
    assert rc == -1 and b'unknown environment' in lib.des_last_error()
    rc = lib.des_rollout_eval(None, None, None, None, None, 0, _lib.Dims(3, 48, 1, 200), 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 4, 0,
                              None, 0, None)
    assert rc == -1 and b'multiple of 32' in lib.des_last_error()
    rc = lib.des_rollout_eval(None, None, None, None, None, 0, d, 11, 0.1, 2.0, 0.0, 0, 0, None, 0, 4, 0, None, 0, None)
    assert rc == -1 and b'repetitions' in lib.des_last_error()
    rc = lib.des_rollout_eval(None, None, None, None, None, 0, d, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 4, 0, None, 0, None)
    assert rc == -1 and b'NULL' in lib.des_last_error()
    assert lib.des_rollout_eval(None, None, None, None, None, 0, d, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 0, 0, None, 0, None) == 0
    # packed CMA payload: upper-triangular tiles of 64 (n <= 2048) or 128
    assert lib.des_cma_packed_elems(1024) == 16 * 17 // 2 * 64 * 64
    assert lib.des_cma_packed_elems(4096) == 32 * 33 // 2 * 128 * 128
    assert lib.des_cma_packed_elems(300) == 5 * 6 // 2 * 64 * 64 and lib.des_cma_packed_elems(0) == 0
    assert lib.des_cma_rank_mu(None, None, None, 4, 16, 1, None, 0, None) == -1
    assert lib.des_cma_cov_apply_packed(None, None, None, 16, 1.0, 0.0, 0.0, None) == -1


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under distributedes_b200/ (nor the GPU arm of bench.py) may import it."""
    import glob
    pkg = os.path.join(REPO, 'distributedes_b200')
    for f in glob.glob(os.path.join(pkg, '**', '*'), recursive=True):
        if os.path.isfile(f) and f.endswith(('.py', '.cu', '.cuh', '.h')):
            txt = open(f).read()
            assert not re.search(r'^\s*(from|import)\s+oracle', txt, re.M), f
            assert not re.search(r'#\s*include\s*["<][^">]*oracle', txt), f          # comments may cite it, code may not
    bench = open(os.path.join(REPO, 'bench.py')).read()
    ours = bench.split('def run_ours')[1].split("if __name__ == '__main__'")[0]
    assert not re.search(r'^\s*(from|import)\s+oracle', ours, re.M)      # only the cpu subprocess leg uses it


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm the driver times next to ours): one JSON line with the contract's keys."""
    import json
    import sys
    r = subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0',
                        '--pop', '256', '--hidden', '64', '--tape-len', '128', '--cpu-sample', '32'],
                       capture_output=True, text=True, timeout=300, cwd=REPO)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1                                     # exactly one line on stdout
    d = json.loads(lines[0])
    for key in ['impl', 'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
                'vs_baseline', 'dtype', 'data', 'config', 'cpu_baseline', 'e2e']:
        assert key in d, key
    assert d['impl'] == 'reference' and d['metric'] == 'nes_policy_evals_per_sec' and d['higher_is_better'] is True
    # the reference run verbatim where oracle/_ref travelled with the snapshot, else the numpy port (and it says which)
    have_ref = os.path.exists(os.path.join(REPO, 'oracle', '_ref', 'natural_es.py'))
    assert d['cpu_baseline']['kind'] == ('reference' if have_ref else 'port')
    assert d['cpu_baseline']['cores'] >= 1 and d['value'] > 0 and 'port' in d['cpu_baseline']
    assert d['e2e'] == {'value': d['value'], 'unit': d['unit'], 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}
    assert 'workload' in d['config']


def test_host_normaliser_matches_reference_arithmetic():
    """utils.SharedStats.feed / merge and StaticNormalizer.__call__ restate utils.py:37-96 in the reference's fp32
    operation order: the expected values below are that arithmetic (StaticNormalizer's pass-through and scaling,
    utils.py:48-51, and the Chan merge, utils.py:85-96) written out on 5-dim RandomState(0) observations."""
    from distributedes_b200.utils import SharedStats, StaticNormalizer
    rs = np.random.RandomState(0)
    a = StaticNormalizer(5)
    for _ in range(50):
        o = rs.randn(5).astype(np.float32)
        assert np.array_equal(a(o), o)                      # empty offline statistics: pass-through (utils.py:48-49)
    assert a.online_stats.n[0] == 50
    A = SharedStats(5)
    A.merge(a.online_stats)
    assert np.array_equal(A.m, a.online_stats.m) and A.n[0] == 50
    A.merge(SharedStats(5))                                 # merging empty statistics is a no-op
    assert A.n[0] == 50 and np.all(np.isfinite(A.v))
    b = StaticNormalizer(5)
    b.offline_stats.load(A)
    o = np.asarray([1, 2, 3, 4, 5], dtype=np.float32)
    want = (o - A.m) / (A.v + np.float32(1e-6)) ** np.float32(.5)
    assert np.array_equal(b(o), want.astype(np.float32))
    B = SharedStats(5)
    for _ in range(30):
        B.feed((rs.randn(5) * 3 + 1).astype(np.float32))
    n0, m0, v0 = A.n[0], A.m.copy(), A.v.copy()
    A.merge(B)
    n = n0 + B.n[0]
    delta = B.m - m0
    assert np.allclose(A.m, m0 + delta * B.n[0] / n, rtol=1e-6)
    assert np.allclose(A.v, (v0 * n0 + B.v * B.n[0] + delta * delta * n0 * B.n[0] / n) / n, rtol=1e-6)
