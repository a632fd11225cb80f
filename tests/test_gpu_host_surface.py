"""The reference-facing surfaces on a real GPU: natural_es.train()/test()/Worker, utils.Evaluator/fitness_shift/Adam,
and the host-buffer C session (des_session_generation_host) — each against the oracle chain."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc

pytestmark = pytest.mark.gpu


def relnorm(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


def oracle_chain(theta0, obs, target, fits, *, sigma, lr, wd, clip, seed, N, d0, H, A):
    """theta after len(fits) generations, ranks taken from the GPU's fitness (layered parity)."""
    theta, opt, outs = theta0, orc.Adam(), []
    for gen, fit in enumerate(fits):
        out = orc.nes_generation(theta, opt, obs, target, sigma=sigma, clip=clip, seed=seed, gen=gen, N=N, d0=d0, H=H, A=A,
                                 weight_decay=wd, learning_rate=lr, fitness=fit)
        theta = out['theta']
        outs.append(out)
    return theta, outs


def test_train_matches_reference_shape_and_oracle_chain():
    """natural_es.train(config): same return triple as natural_es.py:99, test rewards = noiseless fitness of theta_g."""
    from distributedes_b200 import natural_es
    from distributedes_b200.config import PendulumConfig
    cfg = PendulumConfig(hidden_size=64, tape_len=32)
    cfg.pop_size, cfg.sigma, cfg.learning_rate, cfg.seed = 16, 0.1, 0.1, 5
    cfg.max_steps = 3 * cfg.pop_size * 32 + 1              # stop after 4 collections = 3 updates (natural_es.py:82-84)
    eng = natural_es.build_engine(cfg)
    fits = []
    real_rank = eng.rank_and_reduce

    def spy():
        fits.append(eng.fitness_all.cpu().numpy().astype(np.float64))
        return real_rank()
    eng.rank_and_reduce = spy
    rewards, steps, stamps = natural_es.train(cfg, engine=eng)
    assert len(rewards) == len(steps) == len(stamps) == 4 and steps == [0, 512, 1024, 1536]
    env = cfg.env_fn()
    # fitness itself (fp32 path) vs oracle, generation 0
    ref_fit = orc.evaluate_population(cfg.initial_weight, env.obs, env.target, 0.1, 2.0, 5, 0, 0, 16, 3, 64, 1)
    assert np.max(np.abs(fits[0] - ref_fit) / np.abs(ref_fit)) < 2e-5
    theta, outs = oracle_chain(cfg.initial_weight, env.obs, env.target, fits, sigma=0.1, lr=0.1, wd=0.005, clip=2.0, seed=5,
                               N=16, d0=3, H=64, A=1)
    assert np.max(np.abs(eng.theta_numpy() - theta)) <= 1e-5 * np.max(np.abs(theta - cfg.initial_weight))
    for g in range(3):                                    # test() of natural_es.py:54 = fitness of theta_g
        th = cfg.initial_weight if g == 0 else outs[g - 1]['theta']
        ref = orc.tape_fitness(orc.forward(th, env.obs, 3, 64, 1), env.target, 2.0)
        assert abs(rewards[g] - ref) < 2e-5 * abs(ref)
    m, ste = natural_es.test(cfg, cfg.initial_weight, None, engine=eng)
    assert abs(m - rewards[0]) < 1e-6 * abs(m) and ste == 0.0


def test_evaluator_fitness_shift_adam_surfaces(golden_dir):
    from distributedes_b200.config import BipedalWalkerConfig
    from distributedes_b200.utils import Adam, Evaluator, StaticNormalizer, fitness_shift
    cfg = BipedalWalkerConfig(hidden_size=64, tape_len=16)
    ev = Evaluator(cfg, StaticNormalizer(cfg.state_dim))
    cost, steps = ev.eval(cfg.initial_weight)             # utils.py:116-124: (-mean return, steps)
    env = cfg.env_fn()
    ref = orc.tape_fitness(orc.forward(cfg.initial_weight, env.obs, 24, 64, 4), env.target, 1.0)
    assert steps == 16 and abs(-cost - ref) < 2e-5 * abs(ref)
    g = np.load(os.path.join(golden_dir, 'fitness_shift.npz'))
    for i in range(6):                                    # reference fitness_shift outputs
        assert np.max(np.abs(fitness_shift(g['x%d' % i]) - g['y%d' % i])) <= 6e-8
    a = np.load(os.path.join(golden_dir, 'adam.npz'))     # reference Adam trajectory
    opt = Adam()
    for t in range(len(a['g'])):
        step = opt.update(a['g'][t].astype(np.float32))
        ref_step = orc.Adam() if t == 0 else None
        assert step.shape == a['step'][t].shape
    ours, ref_opt = Adam(), orc.Adam()
    for t in range(len(a['g'])):
        g32 = a['g'][t].astype(np.float32)
        assert np.max(np.abs(ours.update(g32) - ref_opt.update(g32.astype(np.float64)))) <= 2e-7


@pytest.mark.parametrize('precision,ftol', [(0, 2e-5), (2, 3e-5)])
def test_c_session_generation_host(precision, ftol):
    """des_session_generation_host through ctypes with plain host (numpy) buffers: three generations."""
    from distributedes_b200 import _lib
    lib = _lib.load()
    d0, H, A, T, N = 24, 64, 4, 128, 256
    obs, target = orc.synthetic_tape(T, d0, A)
    theta0 = orc.synthetic_theta(d0, H, A)
    P = theta0.size
    sess = C.c_void_p()
    opt = _lib.Opt(0.1, 0.1, 0.005, 0.9, 0.999, 1e-8)
    _lib.check(lib.des_session_create(C.byref(sess), 0, _lib.Dims(d0, H, A, T), N, 0, N, opt, 1.0, 77, precision,
                                      theta0.ctypes.data_as(C.c_void_p)), 'create')
    try:
        fit = np.empty(N, np.float32); upd = np.empty(P, np.float32); th = np.empty(P, np.float32)
        fits, ths, upds = [], [], []
        for gen in range(3):
            _lib.check(lib.des_session_generation_host(sess, obs.ctypes.data_as(C.c_void_p), target.ctypes.data_as(C.c_void_p),
                                                       None, fit.ctypes.data_as(C.c_void_p), upd.ctypes.data_as(C.c_void_p),
                                                       th.ctypes.data_as(C.c_void_p)), 'generation')
            fits.append(fit.astype(np.float64)); ths.append(th.copy()); upds.append(upd.copy())
    finally:
        lib.des_session_destroy(sess)
    ref_fit = orc.evaluate_population(theta0, obs, target, 0.1, 1.0, 77, 0, 0, N, d0, H, A)
    assert np.max(np.abs(fits[0] - ref_fit) / np.abs(ref_fit)) < ftol
    theta, outs = oracle_chain(theta0, obs, target, fits, sigma=0.1, lr=0.1, wd=0.005, clip=1.0, seed=77, N=N, d0=d0, H=H, A=A)
    keep_all = np.ones(P, dtype=bool)
    for gen in range(1, 3):          # from the 2nd Adam step on the update is well conditioned: 1e-5 in both norms
        assert relnorm(upds[gen], outs[gen]['update']) <= 1e-5
        # max norm where Adam's normalisation does not amplify the noise error: step = m/(sqrt(v)+eps) divides the ~4e-6
        # (MUFU Box-Muller) error of partial[j] by sqrt(v_j), so entries whose gradient was small in this AND the previous
        # generation (v_j tiny) carry it magnified by max|g|/|g_j|; they are excluded, as in __graft_entry__.smoke
        gmax = np.max(np.abs(outs[gen]['gradient']))
        keep = (np.abs(outs[gen]['gradient']) > 0.02 * gmax) & (np.abs(outs[gen - 1]['gradient']) > 0.02 * gmax)
        assert keep.mean() > 0.5
        keep_all &= keep
        assert np.max(np.abs(upds[gen] - outs[gen]['update'])[keep]) <= 1e-5 * np.max(np.abs(outs[gen]['update']))
    scale = np.max(np.abs(theta - theta0))
    assert np.max(np.abs(ths[-1] - theta)[keep_all]) <= 1e-5 * scale and np.max(np.abs(ths[-1] - theta)) <= 1e-4 * scale
    assert relnorm(ths[-1] - theta0, theta - theta0) <= 1e-5
    # a shard session refuses the whole-generation call (explicit phases + collectives are required)
    sess2 = C.c_void_p()
    _lib.check(lib.des_session_create(C.byref(sess2), 0, _lib.Dims(d0, H, A, T), N, 0, N // 2, opt, 1.0, 77, 0,
                                      theta0.ctypes.data_as(C.c_void_p)), 'create')
    rc = lib.des_session_generation_host(sess2, None, None, None, None, None, None)
    lib.des_session_destroy(sess2)
    assert rc == -1 and b'shard' in lib.des_last_error()


def test_multi_runs_files_and_checkpoint_resume(tmp_path):
    """natural_es.py:113-124 bookkeeping: pickle of [[rewards, steps, timestamps], ...] + log file; and a checkpoint
    taken mid-run resumes to bit-identical parameters."""
    import pickle
    from distributedes_b200 import natural_es
    from distributedes_b200.config import PendulumConfig
    cfg = PendulumConfig(hidden_size=64, tape_len=32)
    cfg.pop_size, cfg.tag, cfg.max_generations = 16, 'NES-64', 2
    stats = natural_es.multi_runs(cfg, runs=2, log_dir=str(tmp_path / 'log'), data_dir=str(tmp_path / 'data'))
    with open(tmp_path / 'data' / ('NES-64-stats-%s.bin' % cfg.task), 'rb') as f:
        on_disk = pickle.load(f)
    assert len(on_disk) == 2 and all(len(run) == 3 for run in on_disk) and on_disk[0][0] == stats[0][0]
    assert stats[0][0] == stats[1][0]                  # runs are independent and deterministic (no optimiser leak)
    log = (tmp_path / 'log' / ('NES-64-%s.txt' % cfg.task)).read_text()
    assert 'Run 0' in log and 'Train: iteration 0,' in log and 'Test: total steps 0,' in log
    # checkpoint / resume
    a = natural_es.build_engine(cfg)
    for _ in range(2):
        a.generation()
    natural_es.save_checkpoint(a, str(tmp_path / 'ck.bin'))
    for _ in range(2):
        a.generation()
    b = natural_es.build_engine(cfg)
    natural_es.load_checkpoint(b, str(tmp_path / 'ck.bin'))
    for _ in range(2):
        b.generation()
    assert np.array_equal(a.theta_numpy(), b.theta_numpy())
