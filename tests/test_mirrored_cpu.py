"""Mirrored (antithetic) sampling without a GPU: the oracle against the reference's own natural_es.train() run on explicit
+-eps pairs (tests/golden/train_b64_mirrored.npz, train_closed_mirrored_pend.npz, oracle/make_golden.py), the
pair-form gradient, the evenness rules of the engines and the C entry points, checkpoints, and sharded NESEngine runs
under gloo with 2 and 3 ranks against the single-process chain."""
import ctypes as C
import os

import numpy as np
import pytest

import cpu_ops
import mirrored_support as ms
from lib_fixture import lib  # noqa: F401
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from ranks import spawn


def test_noise_mirrored_rows_are_signed_plain_rows():
    P = 37
    e = mo.noise_mirrored(5, 2, 6, 8, P)
    p = orc.noise(5, 2, 3, 4, P)
    assert np.array_equal(e[0::2], p) and np.array_equal(e[1::2], -p)
    assert np.array_equal(mo.noise_mirrored(5, 2, 7, 3, P), e[1:4])       # any window of the same members


def test_oracle_matches_reference_train_on_mirrored_pairs(golden_dir):
    g = np.load(os.path.join(golden_dir, 'train_b64_mirrored.npz'))
    d0, H, A, T = (int(v) for v in g['dims'])
    N, seed, sigma, lr, wd, clip = int(g['N']), int(g['seed']), float(g['sigma']), float(g['lr']), float(g['wd']), \
        float(g['clip'])
    assert N % 2 == 0 and (d0, H, A) == (24, 64, 4)
    obs, target = orc.synthetic_tape(T, d0, A)
    theta, opt = g['theta0'], orc.Adam()
    for gen in range(int(g['gens'])):
        out = mo.nes_generation(theta, opt, obs, target, sigma=sigma, clip=clip, seed=seed, gen=gen, N=N, d0=d0, H=H, A=A,
                                weight_decay=wd, learning_rate=lr)
        ref_g = g['grad_after_wd'][gen]
        assert np.linalg.norm(out['gradient'] * (1 - wd) - ref_g) <= 1e-9 * np.linalg.norm(ref_g), gen
        assert np.linalg.norm(out['update'] - g['update'][gen]) <= 1e-6 * np.linalg.norm(g['update'][gen])
        assert np.max(np.abs(out['theta'] - g['theta'][gen])) <= 1e-6
        theta = out['theta']
        rew = orc.tape_fitness(orc.forward(theta, obs, d0, H, A), target, clip)
        assert abs(rew - g['test_rewards'][gen + 1]) < 5e-6 * abs(g['test_rewards'][gen + 1])


def test_oracle_matches_reference_train_on_mirrored_closed_loop_pendulum(golden_dir):
    g = np.load(os.path.join(golden_dir, 'train_closed_mirrored_pend.npz'))
    H, N, reps, seed, gens = int(g['H']), int(g['N']), int(g['reps']), int(g['seed']), int(g['gens'])
    assert (H, N % 2) == (16, 0)
    recs = list(ms.closed_chain(g['theta0'].copy(), H, N, reps, seed, float(g['sigma']), float(g['lr']), float(g['wd']),
                                gens))
    assert list(g['train_steps']) == [k * N * reps * po.HORIZON for k in range(gens + 1)]
    for gen, r in enumerate(recs):
        assert abs(r['test'].mean() - g['test_rewards'][gen]) <= 1e-5 * abs(g['test_rewards'][gen])
        assert np.allclose(r['stats'], g['stats'][gen], rtol=2e-4, atol=2e-5)
        scale = np.abs(g['grad_after_wd'][gen]).max()
        assert np.abs(r['grad_after_wd'] - g['grad_after_wd'][gen]).max() <= (1e-12 if gen == 0 else 1e-5) * scale
        assert np.abs(r['theta'] - g['theta'][gen]).max() <= 2e-6


@pytest.mark.parametrize('N,P', [(2, 5), (64, 37), (250, 301)])
def test_pair_form_gradient_equals_generic_gradient_on_explicit_rows(N, P):
    s = orc.fitness_shift(np.random.RandomState(N).randn(N))
    generic = orc.nes_gradient(mo.noise_mirrored(3, 4, 0, N, P), s, 0.05)
    pair = mo.nes_gradient_streamed(s, 0.05, 3, 4, P, chunk=17)
    assert np.max(np.abs(pair - generic)) <= 1e-13 * np.max(np.abs(generic))


def _tape_engine(N, mirrored=True, **kw):
    from distributedes_b200.engine import NESEngine
    d0, H, A, T = 3, 8, 1, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    return NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=N, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
                     target=target, sigma=0.1, learning_rate=0.1, clip=2.0, seed=11, device='cpu', kernels=cpu_ops,
                     mirrored=mirrored, **kw)


def test_odd_population_is_rejected():
    with pytest.raises(ValueError, match='even pop_size'):
        _tape_engine(7)
    from distributedes_b200.engine import RolloutEngine
    with pytest.raises(ValueError, match='even pop_size'):
        RolloutEngine(hidden=16, pop_size=9, theta0=orc.synthetic_theta(3, 16, 1), sigma=0.1, learning_rate=0.1,
                      device='cpu', kernels=cpu_ops, mirrored=True)
    e = _tape_engine(8)
    assert (e.offset, e.n_local, e.mirrored) == (0, 8, True)


def test_config_defaults_to_plain_sampling():
    from distributedes_b200.config import ClosedLoopPendulumConfig, SynthTapeConfig
    assert SynthTapeConfig().mirrored is False and ClosedLoopPendulumConfig(16).mirrored is False


def test_mirrored_entry_points_reject_odd_shards_before_any_cuda_work(lib):
    from distributedes_b200 import _lib
    dummy = C.c_void_p(256)
    tape = _lib.Dims(24, 64, 4, 128)
    pend = _lib.Dims(3, 64, 1, 200)
    for off, n in ((1, 4), (2, 3)):
        rc = lib.des_nes_eval_mirrored(dummy, dummy, dummy, dummy, tape, 0.1, 1.0, 0, 0, None, off, n, 2, None, 0, None)
        assert rc == -1 and b'whole pairs' in lib.des_last_error()
        rc = lib.des_nes_grad_partial_mirrored(dummy, dummy, n, 6020, 0, 0, None, off, dummy, 1 << 20, None)
        assert rc == -1 and b'whole pairs' in lib.des_last_error()
        rc = lib.des_rollout_eval_mirrored(dummy, None, None, dummy, None, 0, pend, 10, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0,
                                           None, 0, None)
        assert rc == -1 and b'whole pairs' in lib.des_last_error()
        rc = lib.des_nes_perturb_mirrored(dummy, dummy, n, 6020, 0.1, 0, 0, off, None)
        assert rc == -1 and b'whole pairs' in lib.des_last_error()
    rc = lib.des_rollout_eval_mirrored(dummy, None, None, dummy, None, 0, pend, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 1, 1,
                                       None, 0, None)
    assert rc == -1
    rc = lib.des_rollout_eval_mirrored(dummy, None, None, dummy, None, 0, pend, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 2, 1,
                                       None, 0, None)
    assert rc == -1 and b'noiseless' in lib.des_last_error()
    # the workspace query of the plain reduction sizes the mirrored one; a short one is DES_ERR_WORKSPACE
    rc = lib.des_nes_grad_partial_mirrored(dummy, dummy, 64, 6020, 0, 0, None, 0, dummy, 16, None)
    assert rc == -4 and b'workspace' in lib.des_last_error()
    # empty shards are valid and enqueue nothing that needs a device
    assert lib.des_nes_eval_mirrored(None, None, None, None, tape, 0.1, 1.0, 0, 0, None, 0, 0, 2, None, 0, None) == 0
    assert lib.des_rollout_eval_mirrored(None, None, None, None, None, 0, pend, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 0, 0,
                                         None, 0, None) == 0


def test_checkpoint_records_the_sampling_mode(tmp_path):
    from distributedes_b200 import natural_es
    plain, mirrored = _tape_engine(8, mirrored=False), _tape_engine(8)
    path = str(tmp_path / 'ck.npz')
    natural_es.save_checkpoint(mirrored, path)
    assert bool(np.load(path)['mirrored'])
    with pytest.raises(ValueError, match='mirrored=True'):
        natural_es.load_checkpoint(plain, path)
    natural_es.save_checkpoint(plain, path)
    with pytest.raises(ValueError, match='mirrored=False'):
        natural_es.load_checkpoint(mirrored, path)
    # a checkpoint from before the option existed has no key: a plain run
    with np.load(path) as z:
        old = {k: z[k] for k in z.files if k != 'mirrored'}
    np.savez(path, **old)
    with pytest.raises(ValueError, match='mirrored=False'):
        natural_es.load_checkpoint(mirrored, path)


def _worker(N, gens):
    eng = _tape_engine(N)
    fits = []
    for _ in range(gens):
        eng.generation()
        fits.append(eng.fitness_all.numpy().copy())
    return dict(offset=eng.offset, n_local=eng.n_local, theta=eng.theta.numpy(), fits=np.stack(fits))


@pytest.mark.parametrize('N,world', [(22, 2), (22, 3), (8, 3)])
def test_sharded_mirrored_generation_equals_single_process(N, world):
    """Shards are whole pairs (shard_bounds over N/2 pairs, scaled by 2), also when the pairs do not split evenly."""
    gens = 2
    res = spawn(world, _worker, N, gens)
    offs = [(int(r['offset']), int(r['n_local'])) for r in res]
    assert all(o % 2 == 0 and n % 2 == 0 for o, n in offs) and sum(n for _, n in offs) == N
    assert all(offs[k][0] + offs[k][1] == offs[k + 1][0] for k in range(world - 1))
    for r in res[1:]:
        assert np.array_equal(r['theta'], res[0]['theta']) and np.array_equal(r['fits'], res[0]['fits'])
    d0, H, A, T = 3, 8, 1, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    theta, opt = orc.synthetic_theta(d0, H, A), orc.Adam()
    for gen in range(gens):
        out = mo.nes_generation(theta, opt, obs, target, sigma=0.1, clip=2.0, seed=11, gen=gen, N=N, d0=d0, H=H, A=A,
                                weight_decay=0.005, learning_rate=0.1)
        assert np.allclose(res[0]['fits'][gen], out['fitness'], rtol=1e-6)
        theta = out['theta']
    assert np.max(np.abs(res[0]['theta'] - theta)) <= 2e-6
