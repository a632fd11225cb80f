"""CPU oracle for closed-loop rollouts (SURVEY.md 8f row 3) — TEST INFRASTRUCTURE ONLY.

Restates, for the reference's PendulumConfig (config.py:26-31), what ``Evaluator.eval`` does per member
(utils.py:116-124 -> single_run utils.py:126-139): reset the environment, then until done: normalise the observation
(utils.py:48-51), forward the policy (model.py:34-39), add action noise (utils.py:133), clip (config.py:29), step.

The environment is a third-party dependency that is absent here: OpenAI ``gym`` (imported at config.py:1; the reference
pins no version — 'Pendulum-v0' with a 200-step TimeLimit exists in gym 0.9-0.17).  Its published dynamics are restated
in ``pendulum_step`` below, the only restatement: oracle/gym_stub's Pendulum-v0 steps through it too.  This part is
therefore "parity unpinned" against gym itself.  What IS pinned: the rollout loop around it —
tests/golden/train_closed_pend.npz is produced by the reference's own natural_es.train() running verbatim over
oracle/gym_stub's Pendulum-v0, see oracle/make_golden.py.

Reset states come from the counter RNG (stream 2) so every process can regenerate them:
  Philox(counter = (repetition, member, generation, 2), key = seed) -> u = (low 23 bits + 0.5) / 2^23,
  theta = (2 u0 - 1) pi, theta_dot = 2 u1 - 1     (gym: uniform(-[pi, 1], [pi, 1]))
Test episodes (natural_es.py:101-110, no perturbation) use member index 0x40000000.
"""
import numpy as np

from oracle import nes_oracle as orc

STREAM_ENV_RESET = 2
STREAM_ACT_NOISE = 3
TEST_MEMBER = 0x40000000
HORIZON = 200
D0, A = 3, 1


def reset_states(seed, gen, members, reps):
    """[n, reps] initial (theta, theta_dot), fp64."""
    members = np.asarray(members, dtype=np.uint64).reshape(-1, 1)
    r = np.arange(reps, dtype=np.uint64).reshape(1, -1)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    x0, x1, _, _ = orc.philox4x32(r + 0 * members, members + 0 * r, np.uint64(gen & 0xFFFFFFFF),
                                      np.uint64(STREAM_ENV_RESET), k0, k1)
    u0 = ((x0 & np.uint64(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
    u1 = ((x1 & np.uint64(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
    return (2.0 * u0 - 1.0) * np.pi, (2.0 * u1 - 1.0)


def pendulum_obs(th, thdot):
    return np.stack([np.cos(th), np.sin(th), thdot], axis=-1)


def pendulum_step(th, thdot, u):
    """gym Pendulum-v0 dynamics (g = 10, m = l = 1, dt = 0.05, max_speed 8, max_torque 2). Returns th, thdot, reward."""
    u = np.clip(u, -2.0, 2.0)
    an = ((th + np.pi) % (2 * np.pi)) - np.pi
    cost = an ** 2 + 0.1 * thdot ** 2 + 0.001 * u ** 2
    nthdot = thdot + (-3 * 10.0 / 2 * np.sin(th + np.pi) + 3.0 * u) * 0.05
    nth = th + nthdot * 0.05
    nthdot = np.clip(nthdot, -8.0, 8.0)
    return nth, nthdot, -cost


def rollouts(flat, H, seed, gen, members, reps, stats=None, horizon=HORIZON, clip=2.0, act_noise=0.0, tanh=np.tanh,
             trace=False):
    """Episodes of the policies flat[n, P] (already perturbed), `reps` each.

    stats: None or (m[3], v[3], n) — StaticNormalizer offline stats (identity while n == 0).
    Returns (returns[n, reps] fp64, obs_sum[3], obs_sumsq[3], count) over the RAW observations seen; with trace, also
    (obs[n, reps, horizon, 3] fp32, u[n, reps, horizon] the torque applied after the environment's clamp).
    tanh replaces the activation (sensitivity checks with a deliberately wrong one)."""
    flat = np.asarray(flat, dtype=np.float32)
    n = flat.shape[0]
    W1, b1, W2, b2, W3, b3 = [w.astype(np.float64) for w in orc.unflatten(flat, D0, H, A)]
    th, thdot = reset_states(seed, gen, members, reps)
    total = np.zeros((n, reps))
    osum, osq, cnt = np.zeros(3), np.zeros(3), 0
    use = stats is not None and float(stats[2]) != 0.0
    if use:
        m32 = np.asarray(stats[0], np.float32)
        s32 = np.sqrt(np.asarray(stats[1], np.float32) + np.float32(1e-6)).astype(np.float32)
    members = np.asarray(members, dtype=np.uint64).reshape(-1)
    obs_tr, u_tr = [], []
    for t in range(horizon):
        o = pendulum_obs(th, thdot).astype(np.float32)                  # FloatTensor cast, utils.py:42-44 / model.py:35
        osum += o.astype(np.float64).sum((0, 1))
        osq += (o.astype(np.float64) ** 2).sum((0, 1))
        cnt += n * reps
        x = ((o - m32) / s32).astype(np.float32) if use else o
        x = x.astype(np.float64)
        h1 = tanh(np.einsum('nhk,nrk->nrh', W1, x) + b1[:, None, :])
        h2 = tanh(np.einsum('nhk,nrk->nrh', W2, h1) + b2[:, None, :])
        act = (np.einsum('nak,nrk->nra', W3, h2) + b3[:, None, :])[..., 0]
        if act_noise:
            k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
            ep = (members.reshape(-1, 1) * np.uint64(16) + np.arange(reps, dtype=np.uint64).reshape(1, -1)) & np.uint64(0xFFFFFFFF)
            x0, x1, _, _ = orc.philox4x32(np.uint64(t) + 0 * ep, ep, np.uint64(gen & 0xFFFFFFFF),
                                              np.uint64(STREAM_ACT_NOISE), k0, k1)
            z0, _ = orc.box_muller(x0, x1)
            act = act + z0 * act_noise
        act = np.clip(act.astype(np.float32).astype(np.float64), -clip, clip)
        if trace:
            obs_tr.append(o)
            u_tr.append(np.clip(act, -2.0, 2.0))
        th, thdot, r = pendulum_step(th, thdot, act)
        total += r
    if trace:
        return total, osum, osq, cnt, (np.stack(obs_tr, axis=2), np.stack(u_tr, axis=2))
    return total, osum, osq, cnt


def closed_fitness(theta, H, sigma, seed, gen, member_offset, n, reps, stats=None, horizon=HORIZON, clip=2.0):
    """Mean return over the repetitions for members [offset, offset+n): what des_rollout_eval writes."""
    eps = orc.noise(seed, gen, member_offset, n, orc.param_count(D0, H, A))
    flat = orc.perturb(theta, sigma, eps)
    ret, osum, osq, cnt = rollouts(flat, H, seed, gen, np.arange(member_offset, member_offset + n), reps, stats, horizon, clip)
    return ret.mean(1), (osum, osq, cnt)


def test_returns(theta, H, seed, gen, reps, stats=None, horizon=HORIZON, clip=2.0):
    """natural_es.py:101-110 on the unperturbed theta: `reps` episodes from the test reset stream."""
    flat = np.asarray(theta, np.float32).reshape(1, -1)
    ret, _, _, _ = rollouts(flat, H, seed, gen, [TEST_MEMBER], reps, stats, horizon, clip)
    return ret[0]


def merge_totals(stats, osum, osq, cnt):
    """Chan merge (utils.py:85-96) of a batch given by its raw sums into stats = (m, v, n); returns fp32 (m, v, n)."""
    m, v, nA = np.asarray(stats[0], np.float64), np.asarray(stats[1], np.float64), float(stats[2])
    nB = float(cnt)
    mb = osum / nB
    vb = np.maximum(osq / nB - mb * mb, 0.0)
    n = nA + nB
    delta = mb - m
    m2 = m + delta * nB / n
    v2 = (v * nA + vb * nB + delta * delta * nA * nB / n) / n
    return m2.astype(np.float32), v2.astype(np.float32), np.float32(n)
