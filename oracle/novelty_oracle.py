"""CPU oracle for novelty search (include/des_b200.h, "novelty search") — TEST INFRASTRUCTURE ONLY.

  novelty          brute-force k-nearest-neighbour novelty in fp64 (exact squared distances)
  novelty_integer  novelty_fp32 for integer-valued rows, vectorised
  novelty_fp32     the kernel's arithmetic: fp32 differences, fmaf accumulation in j order, (d2, index) order with NaN
                   last, __fsqrt_rn, fp64 mean in that order
  blend            fmaf(w, s_f, fp32(1 - w) * s_n) in fp32 over the centered ranks
  adapt            the NSRA-ES schedule of the reward weight
  select           the meta-population's draw of the next agent
  FinalObs, behaviours, closed_episodes     the behaviour characterisation from pendulum_oracle's episode loop
  train            the novelty-search training loop over caller-supplied evaluations and tests
"""
import numpy as np

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

ADAPT_STEP, ADAPT_PATIENCE = 0.05, 10


# ---- arithmetic ------------------------------------------------------------------------------------------------------
def fmaf32(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded: the fp32 product is exact in fp64, the fp64 sum is rounded to odd (TwoSum's
    error term moves an inexact even result one ulp toward the exact value), and round-to-odd at 53 bits followed by
    round-to-nearest at 24 bits is round-to-nearest of the exact sum."""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    r = np.asarray(p + c, dtype=np.float64)
    z = r - p
    err = (p - (r - z)) + (c - z)
    even = (r.view(np.uint64) & np.uint64(1)) == 0
    fix = (err != 0) & even & np.isfinite(r)
    r = np.where(fix, np.nextafter(r, np.where(err > 0, np.inf, -np.inf)), r)
    return r.astype(np.float32)


def sq_distances_fp32(queries, archive):
    """d2[n, A] fp32: fmaf(diff_j, diff_j, d2) from +0 in j order, diff_j = q_j - a_j in fp32."""
    q = np.asarray(queries, dtype=np.float32)
    a = np.asarray(archive, dtype=np.float32)
    d2 = np.zeros((q.shape[0], a.shape[0]), dtype=np.float32)
    for j in range(q.shape[1]):
        diff = (q[:, j:j + 1] - a[None, :, j]).astype(np.float32)
        d2 = fmaf32(diff, diff, d2)
    return d2


def _mean_of_nearest(d2, k, sqrt):
    """Per row: the first min(k, A) entries in (d2, index) order with NaN last (a stable argsort), their sqrt summed in
    fp64 in that order, divided by the count."""
    keff = min(int(k), d2.shape[1])
    out = np.empty(d2.shape[0], dtype=np.float64)
    for i, row in enumerate(d2):
        order = np.argsort(row, kind='stable')[:keff]
        s = 0.0
        for j in order:
            s += float(sqrt(row[j]))
        out[i] = s / keff
    return out


def novelty_fp32(queries, archive, k):
    """des_novelty's result [n] fp32, bit for bit."""
    d2 = sq_distances_fp32(queries, archive)
    return _mean_of_nearest(d2, k, lambda x: np.sqrt(np.float32(x))).astype(np.float32)


def novelty_integer(queries, archive, k, chunk=256):
    """novelty_fp32 for integer-valued rows (NaN allowed) whose squared distances stay below 2^24, where every fp32
    operation of the contract is exact: d2 from one fp64 matrix product, the (d2, index) order as one int64 key.  Fast
    enough for 4096 x 100 000 rows."""
    q = np.asarray(queries, dtype=np.float64)
    a = np.asarray(archive, dtype=np.float64)
    keff, A = min(int(k), a.shape[0]), a.shape[0]
    a_nan = np.isnan(a).any(1)
    a0 = np.where(a_nan[:, None], 0.0, a)
    aa, idx = (a0 * a0).sum(1), np.arange(A, dtype=np.int64)
    out = np.empty(q.shape[0], dtype=np.float32)
    for lo in range(0, q.shape[0], chunk):
        qc = q[lo:lo + chunk]
        q_nan = np.isnan(qc).any(1)
        q0 = np.where(q_nan[:, None], 0.0, qc)
        d2 = np.rint((q0 * q0).sum(1)[:, None] + aa[None, :] - 2.0 * (q0 @ a0.T)).astype(np.int64)
        assert d2.max(initial=0) < 1 << 24
        d2[:, a_nan] = 1 << 30                       # NaN: after every number
        d2[q_nan, :] = 1 << 30
        key = (d2 << 32) | idx[None, :]
        sel = np.partition(key, keff - 1, axis=1)[:, :keff] if keff < A else key
        sel = np.sort(sel, axis=1)
        d = sel >> 32
        vals = np.where(d == 1 << 30, np.nan, np.sqrt(d.astype(np.float32)).astype(np.float64))
        s = np.zeros(len(qc))
        for j in range(keff):
            s += vals[:, j]
        out[lo:lo + chunk] = (s / keff).astype(np.float32)
    return out


def novelty(queries, archive, k):
    """[n] fp64 novelty from exact squared distances of the fp32 inputs (the reference the fp32 kernel approximates)."""
    q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    a = np.asarray(archive, dtype=np.float32).astype(np.float64)
    d2 = ((q[:, None, :] - a[None, :, :]) ** 2).sum(-1)
    return _mean_of_nearest(d2, k, np.sqrt)


def blend(fitness, novelty_, w):
    """des_ns_shape: fmaf(fp32(w), s_f, fp32(fp32(1 - w) * s_n)) over the fp32 centered ranks."""
    s_f = orc.fitness_shift(fitness).astype(np.float32)
    s_n = orc.fitness_shift(novelty_).astype(np.float32)
    t = (np.float32(1.0 - w) * s_n).astype(np.float32)
    return fmaf32(np.float32(w), s_f, t)


def adapt(w, stall, improved):
    """NSRA-ES after a generation's test: (w, stall) -> (w, stall)."""
    if improved:
        return min(1.0, w + ADAPT_STEP), 0
    stall += 1
    if stall >= ADAPT_PATIENCE:
        return max(0.0, w - ADAPT_STEP), 0
    return w, stall


def select(rng, nov):
    """The draw of the next agent from the novelty of each agent's behaviour: non-finite counts as 0, all zero uniform."""
    p = np.where(np.isfinite(nov), np.asarray(nov, dtype=np.float64), 0.0)
    return int(rng.choice(len(p), p=p / p.sum() if p.sum() > 0 else None))


# ---- behaviour characterisation --------------------------------------------------------------------------------------
class FinalObs:
    """A batch-protocol environment (distributedes_b200/envs.py) that keeps, per slot, the fp32 observation returned by
    the step that ended its episode."""

    def __init__(self, env, d0):
        self.env, self.d0, self.num_envs = env, int(d0), env.num_envs
        self.final = np.zeros((self.num_envs, self.d0), dtype=np.float32)

    def reset(self, keys):
        self.final[:] = 0
        return self.env.reset(keys)

    def step(self, actions, alive):
        obs, r, done = self.env.step(actions, alive)
        ended = np.asarray(alive, dtype=bool) & np.asarray(done, dtype=bool)
        self.final[ended] = np.asarray(obs, dtype=np.float32).reshape(self.num_envs, self.d0)[ended]
        return obs, r, done


def behaviours(final, n, reps):
    """[n, d0] fp32: each member's final observations summed in fp64 in episode order, divided by reps."""
    f = final.reshape(n, reps, -1)
    s = np.zeros((n, f.shape[2]))
    for r in range(reps):
        s += f[:, r].astype(np.float64)
    return (s / reps).astype(np.float32)


def closed_episodes(rows, H, seed, gen, members, reps, stats=None, horizon=po.HORIZON, clip=2.0, act_noise=0.0):
    """pendulum_oracle.rollouts of rows[n, P] with the behaviour: (returns[n, reps], (sum, sum of squares, count),
    bc[n, 3])."""
    members = np.asarray(members, dtype=np.int64).reshape(-1)
    env = FinalObs(po.PendulumBatch(members.size * reps, seed, horizon), po.D0)
    ret, _, totals = po.episodes(rows, env, po.D0, H, po.A, clip, gen, members, reps, stats, seed,
                                 int(members[0]) if members.size else 0, act_noise)
    return ret, totals, behaviours(env.final, members.size, reps)


# ---- the training loop -----------------------------------------------------------------------------------------------
def train(thetas, *, N, sigma, lr, wd, seeds, k, w, generations, evaluate, test, merge, rng_seed):
    """novelty.train restated over M agents starting from thetas[M] (fp32), agent m under seeds[m].  evaluate(m, rows,
    gen) -> (fitness[N] fp32, bc[N, d] fp32, steps) evaluates agent m's members and keeps their observation totals;
    test(m, theta, gen) -> (returns, bc[d]) runs its test episodes; merge(m) merges the totals of agent m's last
    evaluation into its statistics after its step.  w is a float or 'adaptive'.  The gradient is the device's: the fp32
    partial sum of shaped x noise, / N / sigma.  Returns rewards, steps, the archive, the selections, the weights each generation shaped with, final thetas."""
    M = len(thetas)
    thetas = [np.asarray(t, dtype=np.float32).copy() for t in thetas]
    opts, gens = [orc.Adam() for _ in range(M)], [0] * M
    adaptive = w == 'adaptive'
    w = 1.0 if adaptive else float(w)
    archive, agent_bc, rewards, steps, selected, weights = [], [None] * M, [], [], [], []
    rng = np.random.Generator(np.random.PCG64(rng_seed))
    best, stall, total, m, it = -np.inf, 0, 0, 0, 0
    while True:
        for a in (range(M) if it == 0 else [m]):
            ret, bc = test(a, thetas[a], gens[a])
            agent_bc[a] = bc
            archive.append(bc)
            mean = np.mean(ret)
            improved = bool(mean > best)
            best = mean if improved else best
            if it == 0 and a == 0:
                rewards.append(mean)
            if it > 0:
                rewards.append(mean)
                if adaptive:
                    w, stall = adapt(w, stall, improved)
        steps.append(total)
        m = 0 if M == 1 else select(rng, novelty_fp32(np.stack(agent_bc), np.stack(archive), k))
        selected.append(m)
        P = thetas[m].size
        eps = orc.noise(seeds[m], gens[m], 0, N, P)
        fit, bcs, n_steps = evaluate(m, orc.perturb(thetas[m], sigma, eps), gens[m])
        total += n_steps
        it += 1
        if it > generations:
            break
        shaped = blend(fit, novelty_fp32(bcs, np.stack(archive), k), w)
        weights.append(w)
        partial = np.float32(shaped.astype(np.float64) @ eps).astype(np.float64)
        thetas[m], _ = orc.nes_update(thetas[m], partial / N / sigma, opts[m], wd, lr)
        merge(m)
        gens[m] += 1
    return dict(rewards=rewards, steps=steps, archive=np.stack(archive), selected=selected, weights=weights,
                thetas=thetas)
