"""Error model of the policy forward inside des_nes_eval, for tests that use the fitness as an error meter.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/nes_oracle.py).

``forward_error_bound`` is a running worst-case bound on |a_kernel - a_exact| per action, propagated layer by layer
through StandardFCNet.forward (model.py:34-39) with the arithmetic of each des_nes_eval precision:

  operand rounding   fp32  none (the FFMA kernel reads the fp32 weights and observations as they are)
                     f16   every wgmma operand rounded to fp16: 2^-11 relative, 2^-25 absolute (fp16 subnormals);
                           this includes H1, which is packed to fp16 as the A operand of layer 2
                     f16x3 x = hi + lo, both fp16: 2^-22 relative plus an absolute 2^-25 floor (lo goes subnormal
                           below |x| ~ 2^-3), and the dropped lo*lo product
  accumulation       fp32  sequential FFMA chain over K terms: K * 2^-24 * sum|terms|
                     wgmma one fp32 rounding (taken as truncation, 2^-23, twice over for the alignment of the
                           products) per m64n64k16 instruction of the chain: n_instr * 2^-22 * sum|terms|
  tanh               fp32  tanhf, 2 ulp;  f16 tanh.approx, 2^-11 relative;
                     f16x3 1 - 2/(1 + 2^(2 z log2 e)) with MUFU ex2/rcp, 2^-21 absolute plus the fp32 rounding of
                           its argument
  layer 3            exact fp32 FFMA over H terms in every precision, plus the add of b3

The bound is a plain triangle-inequality bound: errors are never assumed to cancel, so the true error of a kernel
sits far below it (the tests state the measured ratio beside every assert).  A tanh input error E is carried
through the largest |tanh'| on [|z| - E, |z| + E].

``closed_loop_bound`` is the same bound for the closed-loop policy of rollout_pendulum_kernel (csrc/des_envs.cu) and
policy_act_kernel (csrc/des_act.cu), precision 'mufu':

  normaliser         x = (o - m) / sqrtf(v + 1e-6f) in fp32: 4 * 2^-24 |x| (subtract, add, sqrtf, divide)
  layers 1 and 2     FFMA chains that start from the bias: K * 2^-24 * (|b| + sum|terms|)
  tanh               tanh_mufu, 1 - 2/(1 + ex2(x * 2 log2 e)): 5 * 2^-23 absolute (ex2.approx, the add, rcp.approx,
                     the final FFMA) plus the 2^-23 relative rounding of its argument
  layer 3            per unit group an FFMA chain over R = H/16 units, then a 4-level butterfly over the 16 groups:
                     every term passes through R + 4 roundings; then the add of b3 and the FFMA of the action noise

``forward_emulated`` rounds the operands exactly as the kernel does (numpy fp16, hi/lo split) and does everything
else in fp64: its distance from the fp64 forward is the operand-rounding part of the kernel error.
"""
from __future__ import annotations

import numpy as np

from . import nes_oracle as orc

PRECISIONS = ('fp32', 'f16', 'f16x3')

U_F16 = 2.0 ** -11          # fp16 unit roundoff (11 significant bits)
U_F16X3 = 2.0 ** -22        # hi + lo, both fp16
F16_FLOOR = 2.0 ** -25      # half the fp16 subnormal spacing
U_F32 = 2.0 ** -24
U_WGMMA = 2.0 ** -22        # per wgmma instruction, relative to the sum of |terms| it has accumulated
TANH_APPROX_REL = 2.0 ** -11
TANH_ACC_ABS = 2.0 ** -21
TANHF_REL = 2.0 ** -22      # 2 ulp
K1_PAD = 32                 # layer-1 K of the tensor-core kernel (state_dim zero-padded): 2 k16 steps


def _op_err(mag, precision):
    """Bound on |round(x) - x| for an operand of magnitude `mag`."""
    if precision == 'fp32':
        return np.zeros_like(mag)
    if precision == 'f16':
        return U_F16 * mag + F16_FLOOR
    return U_F16X3 * mag + F16_FLOOR


def _lo_mag(mag):
    """|lo| of the hi/lo split: |x - fp16(x)| <= 2^-11 |x| (normal hi) or 2^-25 (subnormal hi)."""
    return U_F16 * mag + F16_FLOOR


def _dense(v, Ev, W, EW, b, Eb, K_acc, precision, mma):
    """z = v W^T + b with |v_kernel - v| <= Ev and |W_kernel - W| <= EW (before operand rounding).
    Returns (z exact from the exact inputs, bound on |z_kernel - z|).  v [..., T, K], W [..., N, K]."""
    av, aW = np.abs(v), np.abs(W)
    mv, mW = av + Ev, aW + EW                              # magnitudes of what the kernel holds
    if mma:
        ex, eW = Ev + _op_err(mv, precision), EW + _op_err(mW, precision)
    else:
        ex, eW = Ev, EW
    mm = lambda x, y: np.einsum('...tk,...nk->...tn', x, y)
    # |x^ w^ - x w| <= ex |w^| + |x| ew
    err = mm(ex, mW + eW) + mm(av, eW)
    if mma and precision == 'f16x3':
        err = err + mm(_lo_mag(mv + ex), _lo_mag(mW + eW))   # A_lo * B_lo is not computed
    terms = mm(mv + ex, mW + eW)
    if not mma:
        err = err + K_acc * U_F32 * terms
    else:
        n_instr = (K_acc // 16) * (3 if precision == 'f16x3' else 1)
        err = err + n_instr * U_WGMMA * terms
    z = mm(v, W) + b[..., None, :]
    err = err + Eb[..., None, :] + U_F32 * (np.abs(z) + err)              # + b in fp32
    return z, err


def _tanh(z, Ez, b, precision):
    """h = tanh(z) with |z_kernel - z| <= Ez; returns (h, bound on |h_kernel - h|)."""
    h = np.tanh(z)
    lo = np.maximum(np.abs(z) - Ez, 0.0)
    slope = 1.0 - np.tanh(lo) ** 2                         # max |tanh'| on the interval
    E = slope * Ez
    if precision == 'fp32':
        E = E + TANHF_REL * (np.abs(h) + E) + 2.0 ** -40
    elif precision == 'f16':
        E = E + TANH_APPROX_REL * (np.abs(h) + E) + 2.0 ** -24
    else:
        # ex2.approx / rcp.approx / final FFMA (2^-21), and the fp32 roundings of b*2log2e and of the ex2 argument
        E = E + TANH_ACC_ABS + slope * 2.0 ** -23 * (np.abs(z) + Ez + np.abs(b)[..., None, :])
    return h, E


def forward_error_bound(flat, obs, d0, H, A, precision, dtheta=0.0):
    """Per-action worst-case bound B[..., T, A] on |a_kernel - forward(flat, obs)| for des_nes_eval at `precision`.

    flat: [..., P] the member's perturbed weights theta' (fp32 values); obs [T, d0].
    dtheta: bound on |theta'_kernel - flat| per parameter (scalar or [..., P]) when the kernel generates theta'
    by a different (but equivalent) fp32 formula than the one that produced `flat`."""
    assert precision in PRECISIONS, precision
    flat = np.asarray(flat, dtype=np.float64)
    dth = np.broadcast_to(np.asarray(dtheta, dtype=np.float64), flat.shape)
    W1, b1, W2, b2, W3, b3 = orc.unflatten(flat, d0, H, A)
    E1, Eb1, E2, Eb2, E3, Eb3 = orc.unflatten(dth, d0, H, A)
    x = np.asarray(obs, dtype=np.float64)
    mma = precision != 'fp32'
    K1 = K1_PAD if mma else ((d0 + 3) & ~3)
    z1, Ez1 = _dense(x, np.zeros_like(x), W1, E1, b1, Eb1, K1, precision, mma)
    h1, Eh1 = _tanh(z1, Ez1, b1, precision)
    z2, Ez2 = _dense(h1, Eh1, W2, E2, b2, Eb2, H, precision, mma)
    h2, Eh2 = _tanh(z2, Ez2, b2, precision)
    a, Ea = _dense(h2, Eh2, W3, E3, b3, Eb3, H, 'fp32', False)       # layer 3: fp32 FFMA in every precision
    return Ea


TANH_MUFU_ABS = 5 * 2.0 ** -23      # tanh_mufu (des_common.cuh) at an exact fp32 argument; ~2e-7 in practice
NORM_REL = 4 * U_F32                # the fp32 normaliser (o - m) / sqrtf(v + 1e-6f)
NORM_EPS = float(np.float32(1e-6))


def normalised(obs, stats=None):
    """fp64 (o - m) / sqrt(v + 1e-6f) of raw observations obs[..., d0] with fp32 stats (m, v, n); o itself when stats
    is None or n == 0 (StaticNormalizer, utils.py:48-51)."""
    o = np.asarray(obs, dtype=np.float64)
    if stats is None or float(stats[2]) == 0.0:
        return o
    m = np.asarray(stats[0], np.float32).astype(np.float64)
    v = np.asarray(stats[1], np.float32).astype(np.float64)
    return (o - m) / np.sqrt(v + NORM_EPS)


def _chain(v, Ev, W, b, K):
    """z = v W^T + b by an fp32 FFMA chain of K terms starting from b, inputs off by <= Ev: (z, bound)."""
    mm = lambda x, y: np.einsum('...tk,...nk->...tn', x, y)
    aW = np.abs(W)
    z = mm(v, W) + b[..., None, :]
    err = mm(Ev, aW)
    return z, err + K * U_F32 * (np.abs(b)[..., None, :] + mm(np.abs(v) + Ev, aW)) * (1 + 2 * K * U_F32)


def _tanh_mufu(z, Ez):
    lo = np.maximum(np.abs(z) - Ez, 0.0)
    slope = 1.0 - np.tanh(lo) ** 2
    return np.tanh(z), slope * (Ez + 2.0 ** -23 * (np.abs(z) + Ez)) + TANH_MUFU_ABS


def closed_loop_bound(flat, obs, d0, H, A, stats=None, noise=0.0, noise_err=0.0):
    """Per-action bound B[..., T, A] on |a_kernel - a*| for the closed-loop policy (precision 'mufu', see above), a* the
    fp64 forward of flat[..., P] at normalised(obs[T, d0], stats), plus `noise` (the std * z the kernel adds, [..., T, A]
    or scalar).  noise_err bounds |kernel's std * z - noise| (its MUFU Box-Muller and the fp32 std)."""
    flat = np.asarray(flat, dtype=np.float64)
    W1, b1, W2, b2, W3, b3 = orc.unflatten(flat, d0, H, A)
    x = normalised(obs, stats)
    Ex = NORM_REL * np.abs(x) if (stats is not None and float(stats[2]) != 0.0) else np.zeros_like(x)
    z1, Ez1 = _chain(x, Ex, W1, b1, d0)
    h1, Eh1 = _tanh_mufu(z1, Ez1)
    z2, Ez2 = _chain(h1, Eh1, W2, b2, H)
    h2, Eh2 = _tanh_mufu(z2, Ez2)
    mm = lambda u, w: np.einsum('...tk,...nk->...tn', u, w)
    aW3 = np.abs(W3)
    terms = mm(np.abs(h2) + Eh2, aW3)
    a = mm(h2, W3)
    Ea = mm(Eh2, aW3) + (H // 16 + 4) * U_F32 * terms * (1 + 64 * U_F32)
    mag = terms + np.abs(b3)[..., None, :]
    Ea = Ea + U_F32 * mag + U_F32 * (mag + np.abs(noise)) + np.asarray(noise_err, dtype=np.float64)   # + b3, + std*z
    return Ea * (1 + 4 * U_F32)


def closed_loop_actions(flat, obs, d0, H, A, stats=None, noise=0.0, tanh=np.tanh):
    """a* [..., T, A]: the fp64 forward of flat[..., P] at normalised(obs, stats), plus noise (unclipped).  `tanh`
    replaces the activation (sensitivity checks with a deliberately wrong one)."""
    W1, b1, W2, b2, W3, b3 = (w.astype(np.float64) for w in orc.unflatten(np.asarray(flat), d0, H, A))
    x = normalised(obs, stats)
    mm = lambda u, w: np.einsum('...tk,...nk->...tn', u, w)
    h1 = tanh(mm(x, W1) + b1[..., None, :])
    h2 = tanh(mm(h1, W2) + b2[..., None, :])
    return mm(h2, W3) + b3[..., None, :] + noise


def _f16(x):
    return np.asarray(x, dtype=np.float32).astype(np.float16).astype(np.float64)


def _split(x):
    hi = _f16(x)
    return hi, _f16(np.asarray(x, dtype=np.float64) - hi)


def forward_emulated(flat, obs, d0, H, A, precision):
    """The forward with the kernel's operand rounding and fp64 everything else: actions [..., T, A].
    f16: X, W1', H1, W2' rounded to fp16.  f16x3: each split into fp16 hi + lo, products hi*hi + lo*hi + hi*lo.
    fp32: the fp64 forward of the fp32 values (the FFMA kernel rounds no operand)."""
    assert precision in PRECISIONS, precision
    W1, b1, W2, b2, W3, b3 = (w.astype(np.float64) for w in orc.unflatten(np.asarray(flat), d0, H, A))
    x = np.asarray(obs, dtype=np.float64)
    mm = lambda u, w: np.einsum('...tk,...nk->...tn', u, w)

    def dense(u, w):
        if precision == 'fp32':
            return mm(u, w)
        if precision == 'f16':
            return mm(_f16(u), _f16(w))
        uh, ul = _split(u)
        wh, wl = _split(w)
        return mm(uh, wh) + mm(ul, wh) + mm(uh, wl)

    h1 = np.tanh(dense(x, W1) + b1[..., None, :])
    h2 = np.tanh(dense(h1, W2) + b2[..., None, :])
    return mm(h2, W3) + b3[..., None, :]


# --------------------------------------------------------------------------------------------
# Which eval_tc_kernel<H, X3, CL, NA> a shape runs (launch_tc_h in csrc/des_eval_tc.cu)
# --------------------------------------------------------------------------------------------
def tc_instantiation(H, A, T, precision):
    """(H, X3, CL, NA): a 2-CTA cluster iff the tape has an even number of 128-row tiles; NA = 4 iff A <= 4."""
    assert precision in ('f16', 'f16x3') and T % 128 == 0
    return (H, precision == 'f16x3', 2 if (T // 128) % 2 == 0 else 1, 4 if A <= 4 else 8)


def tc_passes(T):
    """128-row tiles one CTA evaluates per member (csrc/des_eval_tc.cu tc_passes)."""
    tiles = T // 128
    return tiles // 2 if tiles % 2 == 0 else tiles


def _forward_cases():
    """(d0, H, A, T): every H with T in {128, 256, 384, 512} (CL1/CL2 x one/several passes) and both action bounds,
    cycling A through {1, 2, 4} / {5, 7, 8} and d0 through the quad-aligned and generic W1 paths with the second
    layer-1 k16 step empty (d0 <= 16), partial and full."""
    a4, a8, d0s = (1, 2, 4), (5, 7, 8), (1, 3, 16, 17, 24, 31, 32)
    out, i = [], 0
    for H in (64, 128, 256):
        for T in (128, 256, 384, 512):
            for na in (4, 8):
                out.append((d0s[i % 7], H, (a4 if na == 4 else a8)[i % 3], T))
                i += 1
    return out


FORWARD_CASES = _forward_cases()


# --------------------------------------------------------------------------------------------
# Per-action probes: the action errors from fitness values alone
# --------------------------------------------------------------------------------------------
PROBE_DELTA = 2.0 ** -8


def probe_offsets(target, entries, delta=PROBE_DELTA):
    """Exactly representable offsets d_r = fp32(t_r + delta) - t_r of the flat target entries `entries`."""
    t = np.asarray(target, dtype=np.float32).reshape(-1)[np.asarray(entries)]
    return (t + np.float32(delta)).astype(np.float64) - t.astype(np.float64)


def probe_recover(f0, f, d):
    """e_r = a_r - t_r from f0 = -sum e^2 and f_r = the fitness with t_r moved by d_r:
    f_r = f0 + 2 d_r e_r - d_r^2."""
    f0 = float(f0)
    f = np.asarray(f, dtype=np.float64)
    d = np.asarray(d, dtype=np.float64)
    return (f - f0 + d * d) / (2 * d)


def probe_resolution(d, f0, f, depth):
    """Bound on |recovered e_r - e_r| from the fp32 fitness arithmetic.  A summation tree in which every term passes
    through at most `depth` fp32 roundings is off by <= depth * 2^-24 * sum|terms| = depth * 2^-24 * |f|; two more
    roundings cover the residual v - t and the final fp32 result (and the cluster's add of its halves)."""
    d = np.asarray(d, dtype=np.float64)
    mag = abs(float(f0)) + np.abs(np.asarray(f, dtype=np.float64))
    return (depth + 3) * U_F32 * mag / (2 * np.abs(d))


def tc_reduction_depth(A, T):
    """fp32 roundings a squared residual passes through in eval_tc_kernel: the thread's FFMA chain over its 2 rows x A
    actions x passes, the 2 quad shuffles and 5 warp shuffles (warps are then summed in fp64)."""
    return 2 * A * tc_passes(T) + 7


def ffma_reduction_depth(A, T):
    """eval_ffma_kernel: lane q's chain over its warp's 8 observations of a 64-row tile, 5 warp shuffles, then fp64."""
    return 8 + 5


def probe_entries(T, A, rng=None, limit=512):
    """Flat target entries to probe: all when T*A <= 1024, else every action of the rows next to the 8/16/64/128-row
    boundaries (both 128-row tiles of a cluster included) and a fixed random sample, <= `limit` in all."""
    n = T * A
    if n <= 1024:
        return np.arange(n)
    rows = sorted({r for r in range(T) if r % 64 in (0, 7, 8, 15, 16, 63) or r % 128 == 127} | {T - 1})
    picked = [r * A + q for r in rows for q in range(A)][:limit]
    rng = np.random.RandomState(T * 8 + A) if rng is None else rng
    rest = np.setdiff1d(np.arange(n), picked)
    k = max(0, limit - len(picked))
    return np.sort(np.concatenate([picked, rng.choice(rest, size=min(k, len(rest)), replace=False)])).astype(np.int64)
