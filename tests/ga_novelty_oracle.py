"""CPU oracle for the genetic algorithm's novelty search (include/des_b200.h, "novelty search for the genetic
algorithm"; novelty.train_ga) — TEST INFRASTRUCTURE ONLY.  Composed from oracle/ga_oracle.py (the members' rows, the
order at w = 1) and oracle/novelty_oracle.py (fmaf32, the novelty, the NSRA-ES schedule):

  ns_ga_order   the selection order from the contract: fp32 keys fmaf(w, c_f, fp32(1 - w) * c_n) over the centered ranks
                of -fitness and -novelty, a stable sort on (key, index)
  train         genetic.train's loop with the archive and the reward-weight schedule of novelty.train_ga
"""
import numpy as np

from oracle import ga_oracle as gao
from oracle import nes_oracle as orc
from oracle import novelty_oracle as no


def keys(fitness, novelty_, w):
    """[N] fp32 keys fmaf(fp32(w), c_f, fp32(fp32(1 - w) * c_n)), c_f and c_n the fp32 centered ranks of -fitness and
    -novelty (NaN ranks last; -0 == +0)."""
    c_f = orc.fitness_shift(-np.asarray(fitness, dtype=np.float32)).astype(np.float32)
    c_n = orc.fitness_shift(-np.asarray(novelty_, dtype=np.float32)).astype(np.float32)
    t = (np.float32(1.0 - w) * c_n).astype(np.float32)
    return no.fmaf32(np.float32(w), c_f, t)


def ns_ga_order(fitness, novelty_, w, T):
    """The members in positions 0 .. T-1: ascending key, ties to the lower index."""
    k = keys(fitness, novelty_, w).astype(np.float64)
    return np.lexsort((np.arange(k.size), k))[:int(T)]


def train(x0, *, sigma, N, T, E, seed, k, w, generations, evaluate, test, merge=None):
    """novelty.train_ga restated: test(x0, 0) -> (returns, bc[d]) starts the archive; then per generation g: (fitness[N],
    bc[N, d], steps) = evaluate(rows_g, g), the novelty of bc against the archive, the order with weight w, the next
    table (the ordered members' rows), test(table[0], g + 1), whose bc joins the archive and whose mean feeds the NSRA-ES
    schedule ('adaptive': w from 1), and merge(g).  Returns a dict of rewards, steps, the archive, the weights, and per
    generation the fitness, behaviours, novelty, orders and tables."""
    parents = np.asarray(x0, dtype=np.float32).reshape(1, -1)
    adaptive = w == 'adaptive'
    w = 1.0 if adaptive else float(w)
    ret, bc = test(parents[0], 0)
    best = np.mean(ret)
    out = dict(rewards=[best], steps=[0], archive=[bc], weights=[], fitness=[], bcs=[], novelty=[], orders=[], tables=[])
    total, stall = 0, 0
    for g in range(generations):
        rows = gao.member_rows(parents, min(E, parents.shape[0]), sigma, seed, g, np.arange(N))
        f, bcs, steps = evaluate(rows, g)
        total += steps
        nov = no.novelty_fp32(bcs, np.stack(out['archive']), k)
        o = ns_ga_order(f, nov, w, T)
        out['weights'].append(w)
        parents = rows[o]
        for name, x in (('fitness', f), ('bcs', bcs), ('novelty', nov), ('orders', o), ('tables', parents)):
            out[name].append(np.asarray(x))
        ret, bc = test(parents[0], g + 1)
        out['archive'].append(bc)
        mean = np.mean(ret)
        improved = bool(mean > best)
        best = mean if improved else best
        if adaptive:
            w, stall = no.adapt(w, stall, improved)
        out['rewards'].append(mean)
        out['steps'].append(total)
        if merge is not None:
            merge(g)
    out['archive'] = np.stack(out['archive'])
    return out
