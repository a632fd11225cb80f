"""CPU oracle for closed-loop episodes (SURVEY.md 8f row 3) — TEST INFRASTRUCTURE ONLY.

Restates what ``Evaluator.eval`` does per member (utils.py:116-124 -> single_run utils.py:126-139): reset the
environment, then until done: normalise the observation (utils.py:48-51), forward the policy (model.py:34-39), add
action noise (utils.py:133), clip (config.py:29), step.  Each part is written once, for des_rollout_eval (Pendulum
stepped on the device) and des_policy_act (environments stepped on the host) alike:

  policy_actions   one policy step of the population; for A = 1 the action des_rollout_eval takes
  action_noise     the action-noise normals (stream 3)
  reset_states, pendulum_obs, pendulum_step, PendulumBatch    Pendulum-v0, also as a batch-protocol environment
  episodes         the episode loop over any batch-protocol environment (distributedes_b200/envs.py)
  rollouts, closed_fitness, test_returns     fixed-horizon Pendulum episodes: what des_rollout_eval computes

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
_M32 = 0xFFFFFFFF


# ---- the policy step -------------------------------------------------------------------------------------------------
def action_noise(seed, gen, members, reps, t, A):
    """[n, reps, A] normals of the action-noise contract: action c of episode (m, r) at step t is normal c % 4 of the
    quad Philox(t + (c/4) 2^31, 16 m + r, gen, 3)."""
    members = np.asarray(members, dtype=np.uint64).reshape(-1, 1)
    ep = members * np.uint64(16) + np.arange(reps, dtype=np.uint64).reshape(1, -1)
    out = np.zeros((members.shape[0], reps, A))
    for q in range((A + 3) // 4):
        x0, x1, x2, x3 = orc.philox4x32(t + q * 2 ** 31, ep, gen, STREAM_ACT_NOISE, seed & _M32, (seed >> 32) & _M32)
        z = np.stack(orc.box_muller(x0, x1) + orc.box_muller(x2, x3), axis=-1)
        k = min(4, A - 4 * q)
        out[..., 4 * q:4 * q + k] = z[..., :k]
    return out


def policy_actions(rows, obs, alive, d0, H, A, clip, stats=None, act_noise=0.0, seed=0, gen=0, member_offset=0, t=0,
                   tanh=np.tanh):
    """fp64 forward of the fp32 rows[n, P] on obs[n, reps, d0] (raw, fp32): normalise in fp32 (utils.py:48-51), forward,
    noise of the members [member_offset, member_offset + n), clip of the fp32-rounded action (np.clip keeps NaN); dead
    slots 0.  Returns [n, reps, A] fp64.
    stats: None or (m[d0], v[d0], n) — StaticNormalizer offline stats (identity while n == 0).
    tanh replaces the activation (sensitivity checks with a deliberately wrong one)."""
    rows = np.asarray(rows, dtype=np.float32)
    n = rows.shape[0]
    reps = obs.shape[1]
    W1, b1, W2, b2, W3, b3 = [w.astype(np.float64) for w in orc.unflatten(rows, d0, H, A)]
    o = np.asarray(obs, dtype=np.float32)
    if stats is not None and float(stats[2]) != 0.0:
        m32 = np.asarray(stats[0], np.float32)
        s32 = np.sqrt(np.asarray(stats[1], np.float32) + np.float32(1e-6)).astype(np.float32)
        o = ((o - m32) / s32).astype(np.float32)
    alive = np.asarray(alive, dtype=bool).reshape(n, reps)
    x = np.where(alive[..., None], o.astype(np.float64), 0.0)
    h1 = tanh(np.einsum('nhk,nrk->nrh', W1, x) + b1[:, None, :])
    h2 = tanh(np.einsum('nhk,nrk->nrh', W2, h1) + b2[:, None, :])
    act = np.einsum('nak,nrk->nra', W3, h2) + b3[:, None, :]
    if act_noise:
        act = act + act_noise * action_noise(seed, gen, np.arange(member_offset, member_offset + n), reps, t, A)
    act = np.clip(act.astype(np.float32).astype(np.float64), -clip, clip)
    return np.where(alive[..., None], act, 0.0)


def accumulate_stats(part, obs, alive):
    """The documented order of des_policy_act's statistics: per member row, slots in repetition order."""
    n, reps, d0 = obs.shape
    for i in range(n):
        for r in range(reps):
            if alive[i, r]:
                o = obs[i, r].astype(np.float64)
                part[i, :d0] += o
                part[i, d0:2 * d0] += o * o
                part[i, 2 * d0] += 1.0


# ---- Pendulum-v0 -----------------------------------------------------------------------------------------------------
def reset_states(seed, gen, members, reps):
    """Initial (theta, theta_dot) fp64 of the episodes (generation, member, repetition): [n, reps] for the members[n]
    and the repetitions 0..reps-1, or, when `reps` is an array, elementwise over the broadcast gen, members and reps
    (the keys of the batch protocol)."""
    if np.ndim(reps) == 0:
        members, reps = np.reshape(members, (-1, 1)), np.arange(reps).reshape(1, -1)
    x0, x1, _, _ = orc.philox4x32(reps, members, gen, STREAM_ENV_RESET, seed & _M32, (seed >> 32) & _M32)
    u0 = ((x0 & np.uint32(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
    u1 = ((x1 & np.uint32(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
    return (2.0 * u0 - 1.0) * np.pi, 2.0 * u1 - 1.0


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


class PendulumBatch:
    """Pendulum-v0 as a vectorised environment of the batch protocol: slot b resets from its key with reset_states, as
    des_rollout_eval does, and is done after `horizon` steps."""

    def __init__(self, B, seed, horizon=HORIZON):
        self.num_envs, self.seed, self.horizon = int(B), int(seed), int(horizon)

    def reset(self, keys):
        keys = np.asarray(keys, dtype=np.int64).reshape(-1, 3)
        self.th, self.thd = reset_states(self.seed, keys[:, 0], keys[:, 1], keys[:, 2])
        self.t = np.zeros(self.num_envs, dtype=np.int64)
        return pendulum_obs(self.th, self.thd)

    def step(self, actions, alive):
        alive = np.asarray(alive, dtype=bool)
        th, thd, r = pendulum_step(self.th, self.thd, np.asarray(actions, dtype=np.float64).reshape(-1, 1)[:, 0])
        self.th, self.thd = np.where(alive, th, self.th), np.where(alive, thd, self.thd)
        self.t += alive
        return pendulum_obs(self.th, self.thd), np.where(alive, r, 0.0), self.t >= self.horizon


# ---- episodes --------------------------------------------------------------------------------------------------------
def episodes(rows, env, d0, H, A, clip, gen, members, reps, stats=None, seed=0, noise_offset=0, act_noise=0.0,
             tanh=np.tanh, trace=False):
    """The episode loop of fitness.HostEpisodes over the batch environment `env`: episode (i, r) of the rows[n, P]
    resets with the key (gen, members[i], r) and draws its action noise as member noise_offset + i; all step in lockstep
    until every one is done.  Returns (returns[n, reps] fp64, steps, (sum, sum of squares, count) of the raw fp32
    observations of alive slots in fp64); with trace, also (obs[n, reps, T, d0] fp32, actions[n, reps, T, A])."""
    rows = np.asarray(rows, dtype=np.float32)
    n = rows.shape[0]
    B = n * reps
    keys = np.stack([np.full(B, gen), np.repeat(np.asarray(members, dtype=np.int64), reps),
                     np.tile(np.arange(reps), n)], axis=1)
    obs = env.reset(keys)
    alive = np.ones(B, dtype=bool)
    ret = np.zeros(B)
    steps, t = 0, 0
    osum, osq, cnt = np.zeros(d0), np.zeros(d0), 0
    obs_tr, act_tr = [], []
    while alive.any():
        o32 = np.asarray(obs, dtype=np.float32)
        oa = o32[alive].astype(np.float64)
        osum += oa.sum(0)
        osq += (oa * oa).sum(0)
        cnt += int(alive.sum())
        act = policy_actions(rows, o32.reshape(n, reps, d0), alive.reshape(n, reps), d0, H, A, clip, stats, act_noise,
                             seed, gen, noise_offset, t, tanh)
        if trace:
            obs_tr.append(o32.reshape(n, reps, d0))
            act_tr.append(act)
        obs, r, done = env.step(act.reshape(B, A), alive)
        ret[alive] += np.asarray(r)[alive]
        steps += int(alive.sum())
        alive &= ~np.asarray(done, dtype=bool)
        t += 1
    out = ret.reshape(n, reps), steps, (osum, osq, cnt)
    return out + ((np.stack(obs_tr, axis=2), np.stack(act_tr, axis=2)),) if trace else out


def rollouts(flat, H, seed, gen, members, reps, stats=None, horizon=HORIZON, clip=2.0, act_noise=0.0, tanh=np.tanh,
             trace=False):
    """Pendulum episodes of the policies flat[n, P] (already perturbed), `reps` each, reset and noised as the consecutive
    global members[n], as des_rollout_eval keys them.
    Returns (returns[n, reps] fp64, obs_sum[3], obs_sumsq[3], count) over the RAW observations seen; with trace, also
    (obs[n, reps, horizon, 3] fp32, u[n, reps, horizon] the torque applied after the environment's clamp)."""
    members = np.asarray(members, dtype=np.int64).reshape(-1)
    out = episodes(flat, PendulumBatch(members.size * reps, seed, horizon), D0, H, A, clip, gen, members, reps, stats,
                   seed, int(members[0]) if members.size else 0, act_noise, tanh, trace)
    ret, _, (osum, osq, cnt) = out[:3]
    if trace:
        obs, act = out[3]
        return ret, osum, osq, cnt, (obs, np.clip(act[..., 0], -2.0, 2.0))
    return ret, osum, osq, cnt


def closed_fitness(theta, H, sigma, seed, gen, member_offset, n, reps, stats=None, horizon=HORIZON, clip=2.0,
                   noise=orc.noise):
    """Mean return over the repetitions for members [offset, offset+n): what des_rollout_eval writes.  noise(seed, gen,
    member_offset, n, P) gives the members' perturbation rows (mirrored_oracle.closed_fitness passes the mirrored ones);
    the episodes stay keyed by the global member index."""
    eps = noise(seed, gen, member_offset, n, orc.param_count(D0, H, A))
    ret, osum, osq, cnt = rollouts(orc.perturb(theta, sigma, eps), H, seed, gen,
                                   np.arange(member_offset, member_offset + n), reps, stats, horizon, clip)
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
