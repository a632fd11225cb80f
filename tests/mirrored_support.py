"""Test support for mirrored sampling: the oracle's chain of mirrored closed-loop generations."""
import numpy as np

from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po


def closed_chain(theta, H, N, reps, seed, sigma, lr, wd, gens, horizon=po.HORIZON):
    """Single-process chain of mirrored closed-loop generations with the oracle; yields per-generation records."""
    P = theta.size
    stats = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    opt = orc.Adam()
    for gen in range(gens):
        test = po.test_returns(theta, H, seed, gen, reps, stats, horizon)
        fit, (osum, osq, cnt) = mo.closed_fitness(theta, H, sigma, seed, gen, 0, N, reps, stats, horizon)
        stats = po.merge_totals(stats, osum, osq, cnt)
        grad = mo.nes_gradient_streamed(orc.fitness_shift(fit), sigma, seed, gen, P)
        theta, _ = orc.nes_update(theta, grad, opt, wd, lr)
        yield dict(test=test, fitness=fit, stats=np.concatenate([stats[0], stats[1], [stats[2]]]),
                   grad_after_wd=grad - wd * grad, theta=theta)
