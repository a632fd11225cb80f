"""CPU oracle for mirrored (antithetic) sampling — TEST INFRASTRUCTURE ONLY, like oracle/nes_oracle.py on which it builds.

Mirrored sampling (Salimans et al. 2017, the method the reference's README cites) draws members in pairs that share one
eps: the contract of the *_mirrored entry points of include/des_b200.h is

    eps_mirrored[m] = (-1)^(m & 1) * eps[m >> 1],      eps = nes_oracle.noise (stream 0)

so members 2p and 2p+1 are theta + sigma*eps_p and theta - sigma*eps_p.  Everything else of a generation (forward,
fitness, fitness_shift over all N members, Adam) is the plain chain of nes_oracle.py; environment reset states and
action noise stay keyed by the global member index.  Pinned by tests/golden/train_b64_mirrored.npz and
train_closed_mirrored_pend.npz, written by oracle/make_golden.py from the reference's own natural_es.train() with
np.random.randn serving noise_mirrored's rows.
"""
import numpy as np

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po


def noise_mirrored(seed, gen, member_offset, n_members, P):
    """eps_mirrored[n_members, P] fp64 for the members [member_offset, member_offset + n_members)."""
    if n_members == 0:
        return np.zeros((0, P))
    m = int(member_offset) + np.arange(n_members)
    p0 = int(m[0]) >> 1
    pairs = orc.noise(seed, gen, p0, (int(m[-1]) >> 1) - p0 + 1, P)
    return np.where((m & 1)[:, None] == 1, -1.0, 1.0) * pairs[(m >> 1) - p0]


def evaluate_population(theta, obs, target, sigma, clip, seed, gen, member_offset, n_members, d0, H, A, chunk=256):
    """nes_oracle.evaluate_population over the mirrored members: tape fitness fp64 [n_members]."""
    P = orc.param_count(d0, H, A)
    out = np.empty(n_members, dtype=np.float64)
    for s in range(0, n_members, chunk):
        n = min(chunk, n_members - s)
        thetas = orc.perturb(np.asarray(theta)[None, :], sigma, noise_mirrored(seed, gen, member_offset + s, n, P))
        out[s:s + n] = orc.tape_fitness(orc.forward(thetas, obs, d0, H, A), target, clip)
    return out


def nes_gradient_streamed(shaped, sigma, seed, gen, P, chunk=256):
    """natural_es.py:91-92 over the mirrored members in pair form: sum_m s_m eps_m = sum_p (s_2p - s_2p+1) eps_p, so eps
    is regenerated once per pair (what des_nes_grad_partial_mirrored computes, here in fp64).  N even."""
    s = np.asarray(shaped, dtype=np.float64)
    N = len(s)
    assert N % 2 == 0, 'mirrored populations are even'
    c = s[0::2] - s[1::2]
    g = np.zeros(P, dtype=np.float64)
    for o in range(0, N // 2, chunk):
        n = min(chunk, N // 2 - o)
        g += c[o:o + n] @ orc.noise(seed, gen, o, n, P)
    return g / N / sigma


def nes_generation(theta32, opt, obs, target, *, sigma, clip, seed, gen, N, d0, H, A, weight_decay, learning_rate,
                   fitness=None):
    """nes_oracle.nes_generation with mirrored members and the pair-form gradient."""
    P = orc.param_count(d0, H, A)
    if fitness is None:
        fitness = evaluate_population(theta32, obs, target, sigma, clip, seed, gen, 0, N, d0, H, A)
    shaped = orc.fitness_shift(fitness)
    g = nes_gradient_streamed(shaped, sigma, seed, gen, P)
    theta_new, update = orc.nes_update(theta32, g, opt, weight_decay, learning_rate)
    return dict(fitness=np.asarray(fitness, dtype=np.float64), shaped=shaped, gradient=g, update=update, theta=theta_new)


def closed_fitness(theta, H, sigma, seed, gen, member_offset, n, reps, stats=None, horizon=po.HORIZON, clip=2.0):
    """pendulum_oracle.closed_fitness over the mirrored rows (what des_rollout_eval_mirrored writes)."""
    return po.closed_fitness(theta, H, sigma, seed, gen, member_offset, n, reps, stats, horizon, clip, noise_mirrored)
