"""Every step of a device rollout from its observation totals alone — TEST INFRASTRUCTURE ONLY (see nes_oracle.py).

des_rollout_eval reports returns and, per launch, fp64 totals of the raw fp32 observations: T(h, r) = [sum o | sum o^2 |
count] over the member's first r episodes, each episode summed over its first h steps.  That is enough to recover every
observation of every episode:

  * the horizon does not change the prefix: an episode stops earlier, it does not run differently, so
    T(h + 1, r) - T(h, r) holds the observations at step h;
  * the repetitions do not change the episodes: the kernel steps all 10 of them and r only selects what is summed, so
    T(h, r) - T(h, r - 1) isolates episode r - 1.

The sums add fp32 values in fp64 in a fixed order (steps in time order, then episodes in order, then members), so the
double difference gives each fp32 observation (cos th, sin th, thdot) back up to a few fp64 roundings of the totals
involved (``observations``; < 1e-11 at Pendulum's magnitudes).

The torque applied at step t then follows from gym's dynamics, thdot' = thdot + (15 sin th + 3 u) * 0.05, clipped to
+-8 (``pendulum_oracle.pendulum_step``): u = ((thdot' - thdot) / 0.05 - 15 sin th) / 3.  Its resolution is the fp32
rounding of the three observations it reads: (ulp(thdot') + ulp(thdot)) / 2 / 0.15 + 5 ulp(sin th) / 2, about 3e-6 at
|thdot| < 8 (``torques``).  Steps whose observed |thdot'| is 8 may have been clamped and are skipped.
"""
import numpy as np

from . import pendulum_oracle as po

EPISODES = 10                     # episodes the kernel steps per member, whatever the repetitions
DT = 0.05
MAX_SPEED = 8.0
MAX_TORQUE = 2.0
U64 = 2.0 ** -53


def horizons(steps):
    """Horizons whose totals give the observations at t and t + 1 for every step t in `steps` (T(0, r) = 0)."""
    return sorted({h for t in steps for h in (t, t + 1, t + 2) if h >= 1})


def observations(totals, hs, d0=3, mag=None):
    """totals[len(hs), EPISODES, 2*d0+1] fp64: row (i, r) holds the totals of the launch with horizon hs[i] and
    repetitions r + 1.  Returns (obs, err), both [EPISODES, max(hs), d0]: obs[e, t] is episode e's observation at step
    t (NaN where the horizons given do not determine it), err bounds |obs - the kernel's fp32 value|.
    mag: optional magnitudes of the totals for the error bound, when `totals` is itself a difference of two tables."""
    T = np.asarray(totals, dtype=np.float64)[..., :d0]
    M = np.abs(T) if mag is None else np.asarray(mag, dtype=np.float64)[..., :d0]
    zero = np.zeros_like(T[:, :1])
    S = np.diff(np.concatenate([zero, T], axis=1), axis=1)          # episode sums S[i, e] = T(h, e + 1) - T(h, e)
    eS = U64 * (M + np.abs(S))                                      # the add that made T(h, e + 1), the subtraction
    hmax = max(hs)
    Sh = np.full((hmax + 1, EPISODES, d0), np.nan)
    Eh = np.full_like(Sh, np.nan)
    Sh[0], Eh[0] = 0.0, 0.0
    Sh[np.asarray(hs)], Eh[np.asarray(hs)] = S, eS
    obs = Sh[1:] - Sh[:-1]
    err = (Eh[1:] + Eh[:-1] + U64 * (np.abs(Sh[1:]) + np.abs(obs))) * 1.01    # + the step's add, the subtraction
    return obs.transpose(1, 0, 2), err.transpose(1, 0, 2)


def _half_ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64) / 2


def torques(obs, err):
    """From obs/err [..., T, 3] (observations at steps 0..T-1): (u[..., T-1], resolution[..., T-1], valid[..., T-1]).
    u[t] is the torque the environment applied at step t (after its own clamp at +-2), |u - applied| <= resolution
    where valid (both observations known and |thdot[t+1]| < 8)."""
    s, td, td1 = obs[..., :-1, 1], obs[..., :-1, 2], obs[..., 1:, 2]
    u = ((td1 - td) / DT - 15.0 * s) / 3.0
    res = ((_half_ulp(td1) + _half_ulp(td) + err[..., 1:, 2] + err[..., :-1, 2]) / (3.0 * DT)
           + 5.0 * (_half_ulp(s) + err[..., :-1, 1])) * 1.01 + 1e-12      # + the fp64 roundings of both formulas
    with np.errstate(invalid='ignore'):
        valid = np.isfinite(u) & (np.abs(td1) < MAX_SPEED)
    return u, res, valid


def applied(a, clip):
    """The torque the device Pendulum applies for the policy's action a: the action clip, then the environment's."""
    return np.clip(np.clip(a, -clip, clip), -MAX_TORQUE, MAX_TORQUE)


def reset_observations(seed, gen, member):
    """fp32 step-0 observations [EPISODES, 3] of `member`'s episodes (pendulum_oracle.reset_states)."""
    th, thdot = po.reset_states(seed, gen, [member], EPISODES)
    return po.pendulum_obs(th[0], thdot[0]).astype(np.float32)


def predict(obs, u):
    """pendulum_step from (th, thdot) = (atan2(sin, cos), thdot) of obs[..., t, :] with torque u[..., t]: the fp64
    observation at t + 1, [..., T-1, 3]."""
    th = np.arctan2(obs[..., :-1, 1], obs[..., :-1, 0])
    nth, nthdot, _ = po.pendulum_step(th, obs[..., :-1, 2], u)
    return po.pendulum_obs(nth, nthdot)


def predict_tolerance(obs, u_err=0.0):
    """Bound on |predict - fp32 observation at t + 1| given |u - the applied torque| <= u_err: th from fp32 cos/sin
    (<= 2^-24 rad, carried through sin into thdot' with slope 0.75 and through thdot' into th), the roundings of thdot
    and thdot', and the fp32 rounding of the observation itself."""
    e_th = 2.0 ** -24
    e_td = _half_ulp(obs[..., :-1, 2]) + 0.75 * e_th + 3 * DT * u_err                 # thdot' before its rounding
    tol_th = e_th + DT * e_td
    return np.stack([tol_th + _half_ulp(obs[..., 1:, 0]), tol_th + _half_ulp(obs[..., 1:, 1]),
                     e_td + _half_ulp(obs[..., 1:, 2])], axis=-1) * 1.01 + 1e-11


def action_normals(seed, gen, member, T):
    """The action-noise normals of `member`'s episodes, steps 0..T-1: (z0, z1) [EPISODES, T], the first two of
    pendulum_oracle.action_noise (utils.py:133; the kernel adds z0)."""
    z = np.stack([po.action_noise(seed, gen, [member], EPISODES, t, 2)[0] for t in range(T)], axis=1)
    return z[..., 0], z[..., 1]


def normal_error(z0, z1):
    """|MUFU Box-Muller z0 - the fp64 z0| (tests/test_gpu_ops.py noise_tol): 4e-6 (1 + |z|), and 2^-22 ln 2 / r near
    r = sqrt(z0^2 + z1^2) -> 0."""
    r = np.sqrt(z0 * z0 + z1 * z1)
    return 4e-6 * (1 + np.abs(z0)) + 2.0 ** -22 * np.log(2) / np.maximum(r, 1e-4)


def simulate_totals(flat, H, seed, gen, member, hs, stats=None, clip=2.0, act_noise=0.0, tanh=np.tanh):
    """What the device's totals would be for one member, from pendulum_oracle.rollouts: the fp32 observations of all
    EPISODES episodes summed in fp64 in the kernel's order, [len(hs), EPISODES, 7] (rows as ``observations`` reads them).
    For checking the recovery on the CPU."""
    _, _, _, _, (obs, _) = po.rollouts(np.asarray(flat).reshape(1, -1), H, seed, gen, [member], EPISODES, stats,
                                       max(hs), clip, act_noise, tanh=tanh, trace=True)
    o = obs[0].astype(np.float64)                                      # [EPISODES, horizon, 3]
    out = np.zeros((len(hs), EPISODES, 7))
    for i, h in enumerate(hs):
        s = np.zeros((EPISODES, 3))
        q = np.zeros((EPISODES, 3))
        for t in range(h):                                             # steps in time order, per episode
            s = s + o[:, t]
            q = q + o[:, t] * o[:, t]
        tot = np.zeros(7)
        for r in range(EPISODES):                                      # episodes in order
            tot[:3] = tot[:3] + s[r]
            tot[3:6] = tot[3:6] + q[r]
            tot[6] = (r + 1) * h
            out[i, r] = tot
    return out
