"""Error model of des_cma_rank_mu, for tests that check dC = sum_k w_k y_k y_k^T entry by entry.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/nes_oracle.py).

Everything is stated for the fp32 Y [lambda, n] and w [lambda] the kernel reads; the exact result is the fp64
(Y w)^T Y of those values.  With S_ij = sum_k |w_k| |y_ki| |y_kj|, ``rank_mu_error_bound`` is a per-entry worst case
of |dC_kernel - dC_exact| for each kernel des_cma_rank_mu picks:

  ffma  csrc/des_cma.cu (n < 2048): a_ki = fl(w_k y_ki), one fp32 rounding, then one sequential fp32 FMA chain over the
        lambda members:  u S + gamma_lambda (1 + u) S,  gamma_m = m u / (1 - m u),  u = 2^-24.
  tc    csrc/des_cma_tc.cu (n >= 2048): z_ki = fl(fl(sqrt|w_k|) y_ki), two fp32 roundings; column j is scaled by
        2^-e_j so that its largest |z| lies in [2^14, 2^15) (exact); the scaled value is split into fp16 hi + lo:
        2^-22 relative plus a 2^-25 floor in units of 2^e_j (lo, then hi, go subnormal) for every nonzero z.  The
        lo*lo product is not computed.  Three wgmma per k16 step accumulate in fp32 with U_WGMMA per instruction,
        relative to the |terms| the accumulator has summed (as oracle/forward_error.py accounts it), separately over
        each of the two K halves; then one fp32 add of the halves.  The 2^(e_i + e_j) rescale is exact.

The bound is a triangle-inequality bound (errors never cancel), so the kernels sit well below it; the tests state the
measured ratios.  It is scale-covariant: multiplying column j of Y by 2^s multiplies row and column j of the bound by
2^s, as it does the kernels' errors.  fp32 underflow (values below 2^-126) is outside the model.

``rank_mu_emulated`` rounds the operands exactly as each kernel does and does the rest in fp64 ('ffma' also runs the
fp32 FMA chain); 'tc_unscaled' is the split without the per-column scale, which the bound must reject at small scales.
"""
from __future__ import annotations

import numpy as np

KERNELS = ('ffma', 'tc', 'tc_unscaled')
TC_MIN_N = 2048             # des_cma_rank_mu: n >= this runs on the tensor cores
U_F32 = 2.0 ** -24
U_F16 = 2.0 ** -11
U_SPLIT = 2.0 ** -22        # hi + lo, both fp16
F16_FLOOR = 2.0 ** -25      # half the fp16 subnormal spacing
U_WGMMA = 2.0 ** -22        # per wgmma instruction, relative to the sum of |terms| it has accumulated
TC_SCALE_EXP = 15           # a column's largest |z| is scaled into [2^14, 2^15): hi stays far below fp16's 65504
TC_BK = 64                  # members per K stage of the SYRK
WGMMA_PER_STAGE = 3 * (TC_BK // 16)     # hi*hi, lo*hi, hi*lo per k16 step


def kernel_for(n):
    return 'tc' if n >= TC_MIN_N else 'ffma'


def _numpy_gram(A, B):
    return np.asarray(A, dtype=np.float64).T @ np.asarray(B, dtype=np.float64)


def reference(Y, w, gram=_numpy_gram):
    """(dC, S) in fp64 from the fp32 values of Y and w.  gram(A, B) = A^T B in fp64 (pass a device one for large n)."""
    Y64 = np.asarray(Y, dtype=np.float32).astype(np.float64)
    w64 = np.asarray(w, dtype=np.float32).astype(np.float64)
    aY = np.abs(Y64)
    return gram(Y64 * w64[:, None], Y64), gram(aY * np.abs(w64)[:, None], aY)


def tc_operand(Y, w):
    """z = fl(fl(sqrt|w_k|) y_k) in fp32, exactly as cma_split_kernel forms it."""
    Y32, w32 = np.asarray(Y, dtype=np.float32), np.asarray(w, dtype=np.float32)
    return (np.sqrt(np.abs(w32))[:, None] * Y32).astype(np.float32)


def column_exponents(z, scaled=True):
    """e_j with max_k |z_kj| * 2^-e_j in [2^14, 2^15); 0 for an all-zero column and for one whose maximum is not finite."""
    m = np.max(np.abs(z), axis=0) if z.shape[0] else np.zeros(z.shape[1], np.float32)
    if not scaled:
        return np.zeros(z.shape[1], dtype=np.int64)
    ok = np.isfinite(m) & (m > 0)
    e = np.frexp(np.where(ok, m, 1.0).astype(np.float64))[1].astype(np.int64) - TC_SCALE_EXP
    return np.where(ok, e, 0)


def _split(x):
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def rank_mu_emulated(Y, w, kernel):
    """dC with the operand rounding of `kernel` (fp64 [n, n]).
    ffma: fl(w y) and a sequential fp32 FMA chain (emulated with an exact fp64 product and two roundings per step).
    tc / tc_unscaled: z, the per-column power-of-two scale (tc only), the fp16 hi/lo split, hi*hi + lo*hi + hi*lo with
    lo*lo dropped, fp64 sums, the exact rescale."""
    assert kernel in KERNELS, kernel
    Y32, w32 = np.asarray(Y, dtype=np.float32), np.asarray(w, dtype=np.float32)
    if kernel == 'ffma':
        A = (w32[:, None] * Y32).astype(np.float32).astype(np.float64)
        B = Y32.astype(np.float64)
        acc = np.zeros((Y32.shape[1],) * 2, dtype=np.float32)
        for k in range(Y32.shape[0]):
            acc = (acc.astype(np.float64) + np.outer(A[k], B[k])).astype(np.float32)
        return acc.astype(np.float64)
    z = tc_operand(Y32, w32)
    e = column_exponents(z, scaled=(kernel == 'tc'))
    with np.errstate(invalid='ignore', over='ignore'):
        hi, lo = _split(np.ldexp(z, -e[None, :]).astype(np.float32))
        s = np.where(w32 < 0, -1.0, 1.0)[:, None]
        out = (s * hi).T @ hi + (s * lo).T @ hi + (s * hi).T @ lo
    return np.ldexp(out, e[:, None] + e[None, :])


def tc_halves(lam):
    """Members [0, k) and [k, lambda) of the SYRK's two accumulators, and the wgmma instructions each one runs."""
    k_stages = (lam + TC_BK - 1) // TC_BK
    k_half = (k_stages + 1) // 2
    return k_half * TC_BK, (k_half * WGMMA_PER_STAGE, (k_stages - k_half) * WGMMA_PER_STAGE)


def rank_mu_error_bound(Y, w, kernel, gram=_numpy_gram, S=None):
    """Per-entry worst case B[n, n] of |dC_kernel - dC_exact| for des_cma_rank_mu's `kernel` ('ffma' or 'tc';
    'tc_unscaled' is the split without column scales).  S: the S of reference(), if already computed."""
    assert kernel in KERNELS, kernel
    Y32, w32 = np.asarray(Y, dtype=np.float32), np.asarray(w, dtype=np.float32)
    lam = Y32.shape[0]
    if S is None:
        S = reference(Y32, w32, gram)[1]
    u = U_F32
    if kernel == 'ffma':
        gamma = lam * u / (1 - lam * u)
        return (u + gamma * (1 + u)) * S
    z = tc_operand(Y32, w32)
    scale = np.ldexp(1.0, column_exponents(z, scaled=(kernel == 'tc')))[None, :]     # 2^e_j
    az = np.abs(z).astype(np.float64)
    nz = (z != 0).astype(np.float64)
    a = az / (1 - 2 * u)                                          # |sqrt|w| y| exactly, bounded through the fp32 z
    E = (2 * u + u * u) * a + U_SPLIT * az + F16_FLOOR * scale * nz   # |hi + lo - sqrt|w| y|
    L = (U_F16 * (1 + U_F16) * az + 2 * F16_FLOOR * scale) * nz       # |lo|
    H = az + E + 2 * L                                                 # |hi| + |lo|
    # |sum_k sign(w_k) ((a_ki + d_ki)(a_kj + d_kj) - lo_ki lo_kj - a_ki a_kj)| with |d| <= E
    err = gram(E, a + E) + gram(a, E) + gram(L, L)
    k_split, (n0, n1) = tc_halves(lam)
    err = err + n0 * U_WGMMA * gram(H[:k_split], H[:k_split])
    if n1:
        err = err + n1 * U_WGMMA * gram(H[k_split:], H[k_split:])
    return err + u * (S + err)                                         # acc0 + acc1 in fp32


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound over the entries (0 where both are 0; inf where got is not finite or the bound is 0 and
    the error is not)."""
    got = np.asarray(got, dtype=np.float64)
    d = np.abs(got - ref)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(d == 0, 0.0, d / bound)
    r = np.where(np.isfinite(got), r, np.inf)
    return float(np.max(r)) if r.size else 0.0


# --------------------------------------------------------------------------------------------
# The covariance blend des_cma_cov_apply[_packed]: C <- decay C + c1 pc pc^T + cmu dC
# --------------------------------------------------------------------------------------------
def cov_blend_reference(C, dC, pc, decay, c1, cmu):
    """(exact blend, sum of the absolute terms) in fp64 from the fp32 C, dC, pc the kernel reads and the fp64 constants."""
    C64 = np.asarray(C, dtype=np.float32).astype(np.float64)
    d64 = np.asarray(dC, dtype=np.float32).astype(np.float64)
    A, M = decay * C64, cmu * d64
    P = np.zeros_like(C64) if pc is None else c1 * np.outer(*(2 * [np.asarray(pc, np.float32).astype(np.float64)]))
    return A + P + M, np.abs(A) + np.abs(P) + np.abs(M)


def cov_blend_bound(T):
    """Worst case of the kernel's blend given the sum of absolute terms T: decay, c1, cmu rounded to fp32 (the kernel
    takes them as float), fl(decay C), fl(c1 pc_i) and two fused multiply-adds: 4u(1 + 4u) T."""
    return 4 * U_F32 * (1 + 4 * U_F32) * T
