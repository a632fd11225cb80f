"""CPU oracle for the genetic algorithm (distributedes_b200/genetic.py) — TEST INFRASTRUCTURE ONLY.

Restates the contract of include/des_b200.h ("genetic algorithm") in numpy: the parent draws (Philox stream 5), the
members' weights, the selection order and the generation loop of genetic.train(), over any evaluation of rows: the
Pendulum episodes of pendulum_oracle, host-stepped episodes (pendulum_oracle.episodes over a batch environment such as
SynthWalk's) or the tape of nes_oracle.  Parent draws and orders are exact; the members' noise is nes_oracle's (fp64
Box-Muller), so rows agree with the device within the noise contract's rounding, not bit for bit."""
import numpy as np

from oracle import nes_oracle as orc

STREAM_GA_PARENT = 5
_M32 = 0xFFFFFFFF


def parent_words(seed, gen, members):
    """The first Philox word x of (0, m, gen, 5) of each member, uint32."""
    m = np.asarray(members, dtype=np.uint64)
    return orc.philox4x32(np.zeros_like(m), m, gen & _M32, STREAM_GA_PARENT, seed & _M32, (seed >> 32) & _M32)[0]


def parents_of(seed, gen, members, n_parents, n_elites):
    """The table row each member's weights come from: m itself for an elite (m < n_elites), else (x * n_parents) >> 32."""
    m = np.asarray(members, dtype=np.int64)
    p = (parent_words(seed, gen, m).astype(np.uint64) * np.uint64(n_parents)) >> np.uint64(32)
    return np.where(m < n_elites, m, p.astype(np.int64))


def member_rows(parents, n_elites, sigma, seed, gen, members):
    """fp32 [n, P]: an elite's parent row as it is, any other member's parent row + sigma * eps_m (stream 0)."""
    parents = np.asarray(parents, dtype=np.float32)
    members = np.asarray(members, dtype=np.int64).reshape(-1)
    P = parents.shape[1]
    p = parents_of(seed, gen, members, parents.shape[0], n_elites)
    rows = parents[p].copy()
    for i, m in enumerate(members):
        if m >= n_elites:
            rows[i] = orc.perturb(parents[p[i]], np.float32(sigma), orc.noise(seed, gen, int(m), 1, P)[0])
    return rows


def order(fitness, T):
    """The members in positions 0 .. T-1 by fitness, descending: ties to the lower index, NaN last, -0 == +0."""
    f = np.asarray(fitness, dtype=np.float32).astype(np.float64)
    return np.argsort(-f, kind='stable')[:int(T)]


def train(x0, *, sigma, N, T, E, seed, generations, evaluate, test, merge=None):
    """genetic.train()'s chain: test(x0, 0); then per generation g: fitness = evaluate(rows_g, g), the order, the next
    table (the ordered members' rows), test(table[0], g + 1), merge(g).  evaluate returns (fitness[N], steps).  Returns a
    dict of rewards (the test means), steps (cumulative), and per generation: fitness, orders and tables."""
    parents = np.asarray(x0, dtype=np.float32).reshape(1, -1)
    out = dict(rewards=[test(parents[0], 0)], steps=[0], fitness=[], orders=[], tables=[])
    total = 0
    for g in range(generations):
        rows = member_rows(parents, min(E, parents.shape[0]), sigma, seed, g, np.arange(N))
        f, steps = evaluate(rows, g)
        total += steps
        o = order(f, T)
        parents = rows[o]
        out['fitness'].append(np.asarray(f))
        out['orders'].append(o)
        out['tables'].append(parents)
        out['rewards'].append(test(parents[0], g + 1))
        out['steps'].append(total)
        if merge is not None:
            merge(g)
    return out
