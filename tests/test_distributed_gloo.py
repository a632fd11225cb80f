"""world_size=2 on CPU with gloo: the sharded generation (engine.NESEngine host logic) must produce exactly the
single-process result: members split across ranks (even and ragged), fitness gathered by the zero-padded
all-reduce, partial sums all-reduced, identical update on every rank.  Also the launcher's timeout."""
import multiprocessing
import time

import numpy as np
import pytest

import cpu_ops
from ranks import spawn


def _worker(N, gens, normalize=False):
    from distributedes_b200.engine import NESEngine
    from oracle import nes_oracle as orc
    d0, H, A, T = 3, 8, 1, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    theta0 = orc.synthetic_theta(d0, H, A)
    eng = NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=N, theta0=theta0, obs=obs, target=target,
                    sigma=0.1, learning_rate=0.1, clip=2.0, seed=11, device='cpu', kernels=cpu_ops,
                    normalize_obs=normalize)
    fits = []
    for _ in range(gens):
        eng.generation()
        fits.append(eng.fitness_all.numpy().copy())
    return dict(offset=eng.offset, n_local=eng.n_local, theta=eng.theta.numpy(), fits=np.stack(fits))


@pytest.mark.parametrize('N,world', [(10, 2), (11, 2), (3, 2)])
def test_sharded_generation_equals_single_process(N, world):
    from oracle import nes_oracle as orc
    gens = 2
    res = spawn(world, _worker, N, gens)
    # shards tile the population
    assert res[0]['offset'] == 0 and sum(r['n_local'] for r in res) == N
    # every rank ends with bit-identical parameters (no broadcast needed)
    for r in res[1:]:
        assert np.array_equal(r['theta'], res[0]['theta'])
        assert np.array_equal(r['fits'], res[0]['fits'])
    # and they equal the single-process oracle chain
    d0, H, A, T = 3, 8, 1, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    theta = orc.synthetic_theta(d0, H, A)
    opt = orc.Adam()
    for gen in range(gens):
        out = orc.nes_generation(theta, opt, obs, target, sigma=0.1, clip=2.0, seed=11, gen=gen, N=N, d0=d0, H=H, A=A,
                                 weight_decay=0.005, learning_rate=0.1)
        assert np.allclose(res[0]['fits'][gen], out['fitness'], rtol=1e-6)
        theta = out['theta']
    assert np.max(np.abs(res[0]['theta'] - theta)) <= 2e-6


def test_sharded_generation_with_observation_normaliser():
    """normalize_obs=True under gloo: every rank merges identical online statistics (no collective), so the two ranks
    stay bit-identical and equal the single-process chain with the oracle's ObsStats."""
    from oracle import nes_oracle as orc
    N, world, gens = 9, 2, 3
    thetas = [r['theta'] for r in spawn(world, _worker, N, gens, True)]
    assert np.array_equal(thetas[0], thetas[1])
    d0, H, A, T = 3, 8, 1, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    theta, opt, stats = orc.synthetic_theta(d0, H, A), orc.Adam(), orc.ObsStats(d0)
    for gen in range(gens):
        obs_n = np.stack([stats.normalize(o) for o in obs])
        theta = orc.nes_generation(theta, opt, obs_n, target, sigma=0.1, clip=2.0, seed=11, gen=gen, N=N, d0=d0, H=H, A=A,
                                   weight_decay=0.005, learning_rate=0.1)['theta']
        stats.merge_tape(obs, N * T)
    assert np.max(np.abs(thetas[0] - theta)) <= 2e-6


def _sleep(seconds):
    time.sleep(seconds)


def test_spawn_kills_every_rank_after_its_timeout():
    """A rank that never returns fails spawn with TimeoutError instead of hanging the suite, and leaves no process."""
    before = set(multiprocessing.active_children())
    with pytest.raises(TimeoutError):
        spawn(2, _sleep, 300, timeout=10)
    assert not set(multiprocessing.active_children()) - before
