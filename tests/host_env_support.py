"""Test support for host-stepped environments (engine.HostEnvEngine, des_policy_act): a numpy stand-in for the
policy step (cpu_ops.policy_act runs it), a vectorised Pendulum-v0 implementing the batch protocol, and the oracle's
episode loop."""
import numpy as np

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

TEST_MEMBER = 0x40000000
_M32 = 0xFFFFFFFF


def action_noise(seed, gen, members, reps, t, A):
    """[n, reps, A] normals of the action-noise contract: action c of episode (m, r) at step t is normal c % 4 of the
    quad Philox(t + (c/4) 2^31, 16 m + r, gen, 3)."""
    members = np.asarray(members, dtype=np.uint64).reshape(-1, 1)
    ep = (members * np.uint64(16) + np.arange(reps, dtype=np.uint64).reshape(1, -1)) & np.uint64(_M32)
    out = np.zeros((members.shape[0], reps, A))
    for q in range((A + 3) // 4):
        x0, x1, x2, x3 = orc.philox4x32(np.uint64((t + q * 2 ** 31) & _M32) + 0 * ep, ep, np.uint64(gen & _M32),
                                        np.uint64(po.STREAM_ACT_NOISE), seed & _M32, (seed >> 32) & _M32)
        z0, z1 = orc.box_muller(x0, x1)
        z2, z3 = orc.box_muller(x2, x3)
        z = np.stack([z0, z1, z2, z3], axis=-1)
        k = min(4, A - 4 * q)
        out[..., 4 * q:4 * q + k] = z[..., :k]
    return out


def policy_actions(rows, obs, alive, d0, H, A, clip, stats=None, act_noise=0.0, seed=0, gen=0, member_offset=0, t=0):
    """fp64 forward of the fp32 rows[n, P] on obs[n, reps, d0] (raw, fp32): normalise in fp32 (utils.py:48-51), forward,
    noise, clip of the fp32-rounded action; dead slots 0.  Returns [n, reps, A] fp64."""
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
    h1 = np.tanh(np.einsum('nhk,nrk->nrh', W1, x) + b1[:, None, :])
    h2 = np.tanh(np.einsum('nhk,nrk->nrh', W2, h1) + b2[:, None, :])
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


# ---- environments ------------------------------------------------------------------------------------------------------
class PendulumProbe:
    """The shapes of Pendulum-v0 with the classic gym API, for the configs' probe (PendulumBatch does the stepping)."""
    class _Box:
        def __init__(self, n):
            self.shape = (n,)
    observation_space, action_space = _Box(3), _Box(1)


class PendulumBatch:
    """Pendulum-v0 (oracle/pendulum_oracle.py's dynamics) as a vectorised environment of the batch protocol: slot b
    resets from the counter stream of des_rollout_eval, Philox(repetition, member, generation, 2)."""

    def __init__(self, B, seed, horizon=po.HORIZON):
        self.num_envs, self.seed, self.horizon = int(B), int(seed), int(horizon)
        self.stepped = np.zeros(self.num_envs, dtype=np.int64)

    def reset(self, keys):
        keys = np.asarray(keys, dtype=np.int64).reshape(-1, 3).astype(np.uint64)
        x0, x1, _, _ = orc.philox4x32(keys[:, 2], keys[:, 1], keys[:, 0], np.uint64(po.STREAM_ENV_RESET),
                                      self.seed & _M32, (self.seed >> 32) & _M32)
        u0 = ((x0 & np.uint32(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
        u1 = ((x1 & np.uint32(0x7FFFFF)).astype(np.float64) + 0.5) / 8388608.0
        self.th, self.thd = (2.0 * u0 - 1.0) * np.pi, 2.0 * u1 - 1.0
        self.t = np.zeros(self.num_envs, dtype=np.int64)
        return po.pendulum_obs(self.th, self.thd)

    def step(self, actions, alive):
        alive = np.asarray(alive, dtype=bool)
        th, thd, r = po.pendulum_step(self.th, self.thd, np.asarray(actions, dtype=np.float64).reshape(-1, 1)[:, 0])
        self.th, self.thd = np.where(alive, th, self.th), np.where(alive, thd, self.thd)
        self.t += alive
        self.stepped += alive
        return po.pendulum_obs(self.th, self.thd), np.where(alive, r, 0.0), self.t >= self.horizon


def episodes(rows, d0, H, A, clip, env, gen, members, reps, stats=None, seed=0, noise_offset=0, act_noise=0.0,
             feed=True):
    """The oracle's host loop: returns (returns[n, reps], steps, (sum, sum of squares, count) of the raw observations of
    alive slots when `feed`)."""
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
    while alive.any():
        o32 = np.asarray(obs, dtype=np.float32)
        if feed:
            oa = o32[alive].astype(np.float64)
            osum += oa.sum(0)
            osq += (oa * oa).sum(0)
            cnt += int(alive.sum())
        act = policy_actions(rows, o32.reshape(n, reps, d0), alive.reshape(n, reps), d0, H, A, clip, stats, act_noise,
                             seed, gen, noise_offset, t)
        obs, r, done = env.step(act.reshape(B, A), alive)
        ret[alive] += np.asarray(r)[alive]
        steps += int(alive.sum())
        alive &= ~np.asarray(done, dtype=bool)
        t += 1
    return ret.reshape(n, reps), steps, (osum, osq, cnt)


def host_chain(theta, d0, H, A, clip, N, reps, seed, sigma, lr, wd, gens, make_env):
    """natural_es.train on a host-stepped environment, restated with the oracle: yields per collection k = 0..gens a
    record of the test returns, fitness, steps and — for k < gens — statistics after the merge, gradient and theta."""
    P = theta.size
    stats = (np.zeros(d0, np.float32), np.zeros(d0, np.float32), np.float32(0))
    opt = orc.Adam()
    train_env, test_env = make_env(N * reps), make_env(reps)
    for gen in range(gens + 1):
        test, _, _ = episodes(theta[None], d0, H, A, clip, test_env, gen, [TEST_MEMBER], reps, stats, seed, feed=False)
        eps = orc.noise(seed, gen, 0, N, P)
        ret, steps, (osum, osq, cnt) = episodes(orc.perturb(theta, sigma, eps), d0, H, A, clip, train_env, gen,
                                                np.arange(N), reps, stats, seed)
        rec = dict(test=test[0], fitness=ret.mean(1), steps=steps)
        if gen < gens:
            stats = po.merge_totals(stats, osum, osq, cnt)
            grad = orc.nes_gradient(eps, orc.fitness_shift(rec['fitness']), sigma)
            theta, _ = orc.nes_update(theta, grad, opt, wd, lr)
            rec.update(stats=np.concatenate([stats[0], stats[1], [stats[2]]]), grad_after_wd=grad - wd * grad,
                       theta=theta)
        yield rec
