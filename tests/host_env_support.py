"""Test support for host-stepped environments (engine.HostEnvEngine): the shapes of Pendulum-v0 for the configs' probe,
and natural_es.train restated with the oracle's episode loop (oracle/pendulum_oracle.py)."""
import numpy as np

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po


class PendulumProbe:
    """The shapes of Pendulum-v0 with the classic gym API, for the configs' probe (PendulumBatch does the stepping)."""
    class _Box:
        def __init__(self, n):
            self.shape = (n,)
    observation_space, action_space = _Box(3), _Box(1)


def host_chain(theta, d0, H, A, clip, N, reps, seed, sigma, lr, wd, gens, make_env):
    """natural_es.train on a host-stepped environment, restated with the oracle: yields per collection k = 0..gens a
    record of the test returns, fitness, steps and — for k < gens — statistics after the merge, gradient and theta."""
    P = theta.size
    stats = (np.zeros(d0, np.float32), np.zeros(d0, np.float32), np.float32(0))
    opt = orc.Adam()
    train_env, test_env = make_env(N * reps), make_env(reps)
    for gen in range(gens + 1):
        test, _, _ = po.episodes(theta[None], test_env, d0, H, A, clip, gen, [po.TEST_MEMBER], reps, stats, seed)
        eps = orc.noise(seed, gen, 0, N, P)
        ret, steps, (osum, osq, cnt) = po.episodes(orc.perturb(theta, sigma, eps), train_env, d0, H, A, clip, gen,
                                                   np.arange(N), reps, stats, seed)
        rec = dict(test=test[0], fitness=ret.mean(1), steps=steps)
        if gen < gens:
            stats = po.merge_totals(stats, osum, osq, cnt)
            grad = orc.nes_gradient(eps, orc.fitness_shift(rec['fitness']), sigma)
            theta, _ = orc.nes_update(theta, grad, opt, wd, lr)
            rec.update(stats=np.concatenate([stats[0], stats[1], [stats[2]]]), grad_after_wd=grad - wd * grad,
                       theta=theta)
        yield rec
