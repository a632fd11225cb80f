"""Thin torch-tensor front ends for the C-ABI kernels (include/des_b200.h).

PyTorch is plumbing here: it owns device memory and the stream; every op below passes raw
pointers to libdes_b200.so, which enqueues hand-written sm_90a kernels on the current stream.
The entry points cannot see how large an allocation is, so every tensor argument goes through _ptr first: dtype,
contiguity, element count and device.  CPU tensors are an error (there is no CPU fallback).
"""
from __future__ import annotations

import ctypes as C
import functools

import torch

from . import _lib
from ._lib import Dims, Opt, PRECISIONS, State
from .envs import DeviceEnv

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32
STATE_BYTES = C.sizeof(State)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t, name, dtype, n=None, dev=None, optional=False, need='needs'):
    """The device pointer of tensor argument `name` (None for an omitted optional one), after checking in this order:
    a tensor, of `dtype` (None: any), contiguous, `n` entries where the op fixes its shape, on the op's device `dev`
    (None for the anchor, the tensor that selects the device)."""
    if t is None and optional:
        return None
    if not isinstance(t, torch.Tensor):
        raise RuntimeError('%s must be a torch.Tensor, got %s' % (name, type(t).__name__))
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError('%s must be %s, got %s' % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise RuntimeError('%s must be contiguous' % name)
    if n is not None and t.numel() != n:
        raise RuntimeError('%s has %d entries, %s %d' % (name, t.numel(), need, n))
    if dev is not None and t.device != dev:
        raise RuntimeError('%s is on %s, the op runs on %s' % (name, t.device, dev))
    return t.data_ptr()


def _ws(t, dev):
    """(pointer, bytes) of a caller's workspace: any contiguous tensor on `dev`; the library judges its size."""
    return _ptr(t, 'workspace', None, None, dev, True), 0 if t is None else t.numel() * t.element_size()


def _launch(fn, anchor, name, *args):
    """Entry point `fn` on the anchor's device and current stream, its arguments bound by _ptr.  The CPU check comes
    after every argument is bound, so every check above runs without a GPU."""
    if not anchor.is_cuda:
        raise RuntimeError('%s is a CPU tensor: distributedes_b200 has no CPU path' % name)
    with torch.cuda.device(anchor.device):
        _lib.check(getattr(_lib.load(), fn)(*args, _stream()), fn)


def _rows(t, name):
    """n of a 2-D table t[n, P]."""
    if not isinstance(t, torch.Tensor) or t.dim() != 2:
        raise RuntimeError('%s must be a 2-D tensor [n, P], got shape %r' % (name, tuple(getattr(t, 'shape', ()))))
    return t.shape[0]


def _precision(p):
    if isinstance(p, str):
        if p not in PRECISIONS:
            raise RuntimeError('unknown precision %r (choose from %s)' % (p, sorted(PRECISIONS)))
        return PRECISIONS[p]
    return int(p)


def param_count(state_dim, hidden, action_dim):
    n = _lib.load().des_param_count(state_dim, hidden, action_dim)
    if n < 0:
        raise RuntimeError('invalid MLP dims (%r, %r, %r)' % (state_dim, hidden, action_dim))
    return int(n)


@functools.lru_cache(maxsize=None)
def _mlp(d0, H, A):
    """(P, how a count error about the weights of the (d0, H, A) MLP reads), cached: policy_act runs once per step."""
    return param_count(d0, H, A), 'the (%d,%d,%d) MLP needs' % (d0, H, A)


def new_state(device, generation=0):
    """Device-resident des_state {generation, adam_t, beta1_t, beta2_t} as a 32-byte tensor."""
    st = torch.empty(STATE_BYTES, dtype=U8, device=device)
    _launch('des_state_init', st, 'state', st.data_ptr(), generation)
    return st


def state_advance(state, beta1=0.9, beta2=0.999):
    _launch('des_state_advance', state, 'state', _ptr(state, 'state', U8, STATE_BYTES), beta1, beta2)


def read_state(state):
    raw = bytes(state.cpu().numpy().tobytes())
    s = State.from_buffer_copy(raw)
    return dict(generation=s.generation, adam_t=s.adam_t, beta1_t=s.beta1_t, beta2_t=s.beta2_t)


def noise_fill(n_members, P, seed, generation, member_offset=0, stream_tag=0, device='cuda'):
    """eps[n_members, P] fp32 — debug/parity op (natural_es.py:29)."""
    out = torch.empty((n_members, P), dtype=F32, device=device)
    _launch('des_noise_fill', out, 'out', out.data_ptr(), n_members, P, seed, generation, member_offset, stream_tag)
    return out


def nes_perturb(theta, n_members, sigma, seed, generation, member_offset=0, out=None):
    """theta'[n_members, P] = fp32(theta + sigma*eps) (natural_es.py:28-30): a parity op, and the weight rows of
    host-stepped environments (policy_act).  `out`: an optional [n_members, P] buffer."""
    return _perturb('des_nes_perturb', theta, n_members, sigma, seed, generation, member_offset, out)


def nes_perturb_mirrored(theta, n_members, sigma, seed, generation, member_offset=0, out=None):
    """nes_perturb with mirrored noise: row i = fp32(theta + (-1)^(m & 1) sigma*eps[m >> 1]), m = member_offset + i
    (member_offset and n_members even)."""
    return _perturb('des_nes_perturb_mirrored', theta, n_members, sigma, seed, generation, member_offset, out)


def _perturb(fn, theta, n_members, sigma, seed, generation, member_offset, out):
    P, dev = theta.numel(), theta.device
    if out is None:
        out = torch.empty((n_members, P), dtype=F32, device=dev)
    _launch(fn, theta, 'theta', _ptr(out, 'out', F32, n_members * P, dev), _ptr(theta, 'theta', F32), n_members, P,
            sigma, seed, generation, member_offset)
    return out


def obs_stats_merge(stats, obs, n_feed):
    """SharedStats.merge of one generation's online statistics on the tape env (utils.py:85-96), in place."""
    T, d0 = obs.shape
    _launch('des_obs_stats_merge', obs, 'obs', _ptr(stats, 'stats', F32, 2 * d0 + 1, obs.device), _ptr(obs, 'obs', F32),
            T, d0, float(n_feed))
    return stats


def obs_normalize(obs, stats, out=None):
    """StaticNormalizer.__call__ (utils.py:42-57) over the whole tape: identity while stats are empty."""
    (T, d0), dev = obs.shape, obs.device
    if out is None:
        out = torch.empty((T, d0), dtype=F32, device=dev)
    _launch('des_obs_normalize', obs, 'obs', _ptr(out, 'out', F32, T * d0, dev), _ptr(obs, 'obs', F32),
            _ptr(stats, 'stats', F32, 2 * d0 + 1, dev), T, d0)
    return out


def _env_dims(env):
    """(state_dim, action_dim) of the device environment with library id `env` (envs.DeviceEnv.SPECS)."""
    for spec in DeviceEnv.SPECS.values():
        if spec['env'] == env:
            return spec['state_dim'], spec['action_dim']
    raise RuntimeError('unknown environment id %r' % (env,))


def rollout_eval(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                 generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None, totals_out=None,
                 workspace=None, out=None, episodes_out=None):
    """Closed-loop fitness of members [member_offset, member_offset + n_local): mean return over `repetitions`
    episodes stepped on the device (Evaluator.eval utils.py:116-124 over single_run utils.py:126-139)."""
    return _rollout('des_rollout_eval', theta, 'theta', (sigma, state, noiseless), env, hidden, horizon, repetitions,
                    clip, action_noise_std, seed, generation, member_offset, n_local, obs_stats, totals_out, workspace,
                    out, episodes_out)


def rollout_eval_mirrored(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                          generation=0, state=None, member_offset=0, n_local, noiseless=False, obs_stats=None,
                          totals_out=None, workspace=None, out=None, episodes_out=None):
    """rollout_eval with mirrored noise: member m's weights are theta + (-1)^(m & 1) sigma*eps[m >> 1] (member_offset and
    n_local even; noiseless is rejected: test episodes use rollout_eval).  Episodes stay keyed by the global member."""
    return _rollout('des_rollout_eval_mirrored', theta, 'theta', (sigma, state, noiseless), env, hidden, horizon,
                    repetitions, clip, action_noise_std, seed, generation, member_offset, n_local, obs_stats, totals_out,
                    workspace, out, episodes_out)


def rollout_eval_solutions(solutions, *, env=0, hidden, horizon=200, repetitions=10, clip, action_noise_std=0.0, seed,
                           generation=0, member_offset=0, obs_stats=None, totals_out=None, workspace=None, out=None,
                           episodes_out=None):
    """Closed-loop fitness of explicit solutions[n_local, P] (CMA-ES's ask() rows, cma_es.py:22-29): row i is global
    member member_offset + i, whose episodes reset from the same counter stream as rollout_eval's member."""
    return _rollout('des_rollout_eval_solutions', solutions, 'solutions', None, env, hidden, horizon, repetitions, clip,
                    action_noise_std, seed, generation, member_offset, _rows(solutions, 'solutions'), obs_stats,
                    totals_out, workspace, out, episodes_out)


def _rollout(fn, weights, name, noise, env, hidden, horizon, repetitions, clip, action_noise_std, seed, generation,
             member_offset, n_local, obs_stats, totals_out, workspace, out, episodes_out, record=None, bc_out=None):
    """The launch of rollout_eval[_mirrored] (weights = theta[P], noise = (sigma, state, noiseless)) and of
    rollout_eval_solutions (weights = solutions[n_local, P], noise = None); `record` = (mirrored, states_out, obs_out,
    actions_out, rewards_out) makes it the launch of rollout_record[_solutions], and `bc_out` [n_local, d0] that of
    rollout_eval_bc (ops_novelty)."""
    d0, A = _env_dims(env)
    P, mlp = _mlp(d0, int(hidden), A)
    n_local, reps, w, dev = int(n_local), int(repetitions), 2 * d0 + 1, weights.device
    if out is None:
        out = torch.empty(n_local, dtype=F32, device=dev)
    if totals_out is not None and workspace is None:
        workspace = torch.empty(max(n_local, 1) * w, dtype=F64, device=dev)
    head = (_ptr(out, 'out', F32, n_local, dev), _ptr(episodes_out, 'episodes_out', F32, n_local * reps, dev, True),
            _ptr(totals_out, 'totals_out', F64, w, dev, True),
            _ptr(weights, name, F32, P, need=mlp) if noise else _ptr(weights, name, F32, n_local * P, need=mlp + ' n x P ='),
            _ptr(obs_stats, 'obs_stats', F32, w, dev, True), int(env), Dims(d0, hidden, A, horizon), reps)
    tail = (float(clip), float(action_noise_std), int(seed), int(generation))
    traj = ()
    if record is not None:    # the four trajectories [n_local, reps, horizon, width], after the evaluation's arguments
        steps = n_local * reps * int(horizon)
        traj = tuple(_ptr(t, nm, dt, steps * width, dev, True) for t, (nm, dt, width) in zip(
            record[1:], (('states_out', F64, 2), ('obs_out', F32, d0), ('actions_out', F32, A), ('rewards_out', F64, 1))))
    if noise:     # des_rollout_eval[_mirrored]: sigma before clip, state after the generation, noiseless after n_local
        sigma, state, noiseless = noise
        args = head + (float(sigma),) + tail + (_ptr(state, 'state', U8, STATE_BYTES, dev, True), int(member_offset),
                                                n_local, 1 if noiseless else 0)
        if record is not None:
            args += (1 if record[0] else 0,)
    else:
        args = head + tail + (int(member_offset), n_local)
    args += traj
    if bc_out is not None:
        args += (_ptr(bc_out, 'bc_out', F32, n_local * d0, dev),)
    _launch(fn, weights, name, *args, *_ws(workspace, dev))
    return out


def obs_stats_merge_totals(stats, totals, state_dim):
    """Chan merge of a batch given by fp64 [sum | sum of squares | count] into stats [m|v|n] (utils.py:85-96)."""
    w = 2 * int(state_dim) + 1
    _launch('des_obs_stats_merge_totals', stats, 'stats', _ptr(stats, 'stats', F32, w),
            _ptr(totals, 'totals', F64, w, stats.device), int(state_dim))
    return stats


def policy_act(rows, obs, alive, *, state_dim, hidden, action_dim, repetitions, clip, action_noise_std=0.0, seed,
               generation, member_offset=0, t, obs_stats=None, stat_part=None, out=None):
    """One environment step of host-stepped episodes (Evaluator.single_run utils.py:128-134 minus env.step):
    actions[n_local, repetitions, A] of rows[n_local, P] for raw obs[n_local, repetitions, d0] and alive (uint8) of the
    same leading shape; dead slots get 0.  stat_part (fp64 [n_local, 2*d0+1]) accumulates the raw observation
    statistics of the alive slots."""
    n_local, dev = _rows(rows, 'rows'), rows.device
    d0, A, reps = int(state_dim), int(action_dim), int(repetitions)
    P, mlp = _mlp(d0, int(hidden), A)
    if out is None:
        out = torch.empty((n_local, reps, A), dtype=F32, device=dev)
    _launch('des_policy_act', rows, 'rows', _ptr(out, 'out', F32, n_local * reps * A, dev),
            _ptr(stat_part, 'stat_part', F64, n_local * (2 * d0 + 1), dev, True),
            _ptr(rows, 'rows', F32, n_local * P, need=mlp + ' n x P ='), P, _ptr(obs, 'obs', F32, n_local * reps * d0, dev),
            _ptr(alive, 'alive', U8, n_local * reps, dev), _ptr(obs_stats, 'obs_stats', F32, 2 * d0 + 1, dev, True),
            Dims(d0, int(hidden), A, 0), reps, float(clip), float(action_noise_std), int(seed), int(generation),
            int(member_offset), n_local, int(t))
    return out


def obs_parts_reduce(parts, state_dim, out=None):
    """totals[2*d0+1] fp64 = sum of the stat_part rows [n_local, 2*d0+1] in member order."""
    w, pp = 2 * int(state_dim) + 1, _ptr(parts, 'parts', F64)
    n_local = parts.numel() // w
    if parts.numel() != n_local * w:
        raise RuntimeError('parts has %d entries, not a multiple of 2*d0+1 = %d' % (parts.numel(), w))
    if out is None:
        out = torch.empty(w, dtype=F64, device=parts.device)
    _launch('des_obs_parts_reduce', parts, 'parts', _ptr(out, 'out', F64, w, parts.device), pp, n_local, int(state_dim))
    return out


def eval_workspace(state_dim, hidden, action_dim, tape_len, precision, device):
    """Optional scratch for des_nes_eval (multi-pass tensor-core shapes); None when the shape needs none."""
    with torch.cuda.device(device):
        nbytes = _lib.load().des_nes_eval_workspace_bytes(Dims(state_dim, hidden, action_dim, tape_len), _precision(precision))
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device) if nbytes else None


def nes_eval(theta, obs, target, *, hidden, sigma, clip, seed, generation=0, state=None, member_offset=0,
             n_local, precision='fp32', out=None, workspace=None):
    """Fused sample+forward+fitness for members [member_offset, member_offset+n_local) -> fitness[n_local].

    precision 'f16' / 'f16x3' run the hidden layers on tensor cores with fp16 operands: |obs| and |theta'| must stay
    below 65520, or they overflow to inf.  A NaN action gives a NaN fitness on every path (np.clip keeps NaN): this
    tape, the closed-loop rollouts (whose Pendulum clamps the torque and the speed without dropping NaN either) and
    policy_act, which hands a host environment the NaN."""
    return _nes_eval('des_nes_eval', theta, obs, target, hidden, sigma, clip, seed, generation, state, member_offset,
                     n_local, precision, out, workspace)


def nes_eval_mirrored(theta, obs, target, *, hidden, sigma, clip, seed, generation=0, state=None, member_offset=0,
                      n_local, precision='fp32', out=None, workspace=None):
    """nes_eval with mirrored noise: member m's weights are theta + (-1)^(m & 1) sigma*eps[m >> 1], so member 2p's
    fitness is bit-equal to nes_eval's member p (member_offset and n_local even)."""
    return _nes_eval('des_nes_eval_mirrored', theta, obs, target, hidden, sigma, clip, seed, generation, state,
                     member_offset, n_local, precision, out, workspace)


def _tape(obs, target, dev):
    """(T, d0, A) and the pointers of the tape obs[T, d0], target[T, A] of nes_eval and pop_eval."""
    po, pt = _ptr(obs, 'obs', F32, None, dev), _ptr(target, 'target', F32, None, dev)
    if obs.dim() != 2 or target.dim() != 2 or target.shape[0] != obs.shape[0]:
        raise RuntimeError('the tape is obs[T, d0] and target[T, A]: obs has shape %r, target %r'
                           % (tuple(obs.shape), tuple(target.shape)))
    return obs.shape[0], obs.shape[1], target.shape[1], po, pt


def _nes_eval(fn, theta, obs, target, hidden, sigma, clip, seed, generation, state, member_offset, n_local, precision,
              out, workspace):
    dev = theta.device
    T, d0, A, po, pt = _tape(obs, target, dev)
    P, mlp = _mlp(d0, int(hidden), A)
    if out is None:
        out = torch.empty(n_local, dtype=F32, device=dev)
    _launch(fn, theta, 'theta', _ptr(out, 'out', F32, n_local, dev), _ptr(theta, 'theta', F32, P, need=mlp), po, pt,
            Dims(d0, hidden, A, T), sigma, clip, seed, generation, _ptr(state, 'state', U8, STATE_BYTES, dev, True),
            member_offset, n_local, _precision(precision), *_ws(workspace, dev))
    return out


def pop_eval(solutions, obs, target, *, hidden, clip, out=None):
    """Tape fitness of explicit weight vectors solutions[n, P] (what CMA-ES evaluates, cma_es.py:62-75)."""
    n, dev = _rows(solutions, 'solutions'), solutions.device
    T, d0, A, po, pt = _tape(obs, target, dev)
    P, mlp = _mlp(d0, int(hidden), A)
    if out is None:
        out = torch.empty(n, dtype=F32, device=dev)
    _launch('des_pop_eval', solutions, 'solutions', _ptr(out, 'out', F32, n, dev),
            _ptr(solutions, 'solutions', F32, n * P, need=mlp + ' n x P ='), po, pt, Dims(d0, hidden, A, T), clip, n)
    return out


def rank_workspace(n_local, device, N):
    nbytes = _lib.load().des_rank_workspace_bytes(N, n_local)
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def centered_rank(fitness_all, member_offset=0, n_local=None, *, workspace=None, return_ranks=False, out=None):
    """fitness_shift (utils.py:142-148) for a shard of the global fitness vector."""
    pf = _ptr(fitness_all, 'fitness_all', F32)
    N, dev = fitness_all.numel(), fitness_all.device
    if n_local is None:
        n_local = N - member_offset
    if out is None:
        out = torch.empty(n_local, dtype=F32, device=dev)
    ranks = torch.empty(n_local, dtype=I32, device=dev) if return_ranks else None
    if workspace is None:
        workspace = rank_workspace(n_local, dev, N)
    _launch('des_centered_rank', fitness_all, 'fitness_all', _ptr(out, 'out', F32, n_local, dev),
            _ptr(ranks, 'ranks', I32, n_local, dev, True), pf, N, member_offset, n_local, *_ws(workspace, dev))
    return (out, ranks) if return_ranks else out


def grad_workspace(n_local, P, device):
    nbytes = _lib.load().des_grad_workspace_bytes(n_local, P)
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def nes_grad_partial(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None, out=None):
    """partial[P] = sum_i shaped[i] * eps[member_offset+i] (natural_es.py:91, per shard; eps regenerated)."""
    return _grad_partial('des_nes_grad_partial', shaped_local, P, seed, generation, state, member_offset, workspace, out)


def nes_grad_partial_mirrored(shaped_local, P, *, seed, generation=0, state=None, member_offset=0, workspace=None,
                              out=None):
    """The partial of a mirrored shard: sum_p (shaped[2p] - shaped[2p+1]) * eps[member_offset/2 + p], one eps per pair
    (member_offset and n_local even; grad_workspace(n_local, P) suffices)."""
    return _grad_partial('des_nes_grad_partial_mirrored', shaped_local, P, seed, generation, state, member_offset,
                         workspace, out)


def _grad_partial(fn, shaped_local, P, seed, generation, state, member_offset, workspace, out):
    ps = _ptr(shaped_local, 'shaped_local', F32)
    n_local, dev = shaped_local.numel(), shaped_local.device
    if out is None:
        out = torch.empty(P, dtype=F32, device=dev)
    if workspace is None:
        workspace = grad_workspace(n_local, P, dev)
    _launch(fn, shaped_local, 'shaped_local', _ptr(out, 'out', F32, P, dev), ps, n_local, P, seed, generation,
            _ptr(state, 'state', U8, STATE_BYTES, dev, True), member_offset, *_ws(workspace, dev))
    return out


def nes_apply(theta, adam_m, adam_v, partial_sum, N, state, *, sigma, learning_rate, weight_decay=0.005,
              beta1=0.9, beta2=0.999, epsilon=1e-8, update_out=None, grad_out=None):
    """natural_es.py:92-96 + utils.py:159-166, in place on theta / adam_m / adam_v (fp64 Adam state)."""
    pt = _ptr(theta, 'theta', F32)
    P, dev = theta.numel(), theta.device
    _launch('des_nes_apply', theta, 'theta', pt, _ptr(adam_m, 'adam_m', F64, P, dev), _ptr(adam_v, 'adam_v', F64, P, dev),
            _ptr(update_out, 'update_out', F32, P, dev, True), _ptr(grad_out, 'grad_out', F64, P, dev, True),
            _ptr(partial_sum, 'partial_sum', F32, P, dev), P, N,
            Opt(sigma, learning_rate, weight_decay, beta1, beta2, epsilon), _ptr(state, 'state', U8, STATE_BYTES, dev))


_CMA_WS = {}      # (device, n, lambda) -> workspace tensor of des_cma_rank_mu (tensor-core shapes only)
CMA_TC_MIN_N = 2048      # des_cma_rank_mu runs n >= this on the tensor cores, smaller n on the fp32 FFMA kernel


def _cma_rank_mu(Y, w, out, packed):
    lam, n, dev = _rows(Y, 'Y'), Y.shape[1], Y.device
    size = cma_packed_elems(n) if packed else n * n
    if out is None:
        out = torch.empty(size if packed else (n, n), dtype=F32, device=dev)
    lib = _lib.load()
    key = (str(dev), int(n), int(lam))
    ws = _CMA_WS.get(key)
    if ws is None:
        ws = torch.empty(int(lib.des_cma_rank_mu_workspace_bytes(int(n), int(lam))), dtype=torch.uint8, device=dev)
        if len(_CMA_WS) > 8:
            _CMA_WS.clear()
        _CMA_WS[key] = ws
    _launch('des_cma_rank_mu', Y, 'Y', _ptr(out, 'out', F32, size, dev), _ptr(Y, 'Y', F32), _ptr(w, 'w', F32, lam, dev),
            lam, n, 1 if packed else 0, ws.data_ptr(), ws.numel())
    return out


def cma_rank_mu(Y, w, out=None):
    """dC[n,n] = sum_i w_i y_i y_i^T for Y[lambda_local, n] (rank-mu term of es.tell, cma_es.py:90).
    Tensor cores (split-fp16 wgmma SYRK) for n >= CMA_TC_MIN_N, fp32 FFMA below."""
    return _cma_rank_mu(Y, w, out, False)


def cma_cov_apply(Cmat, dC, pc, *, decay, c1, cmu):
    """C <- decay*C + c1*pc pc^T + cmu*dC, in place."""
    return _cov_apply('des_cma_cov_apply', Cmat, dC, 'dC', False, pc, decay, c1, cmu)


def cma_packed_elems(n):
    return int(_lib.load().des_cma_packed_elems(int(n)))


def cma_rank_mu_packed(Y, w, out=None):
    """The rank-mu partial as packed upper-triangular tiles (the multi-GPU all-reduce payload: half of [n, n])."""
    return _cma_rank_mu(Y, w, out, True)


def cma_cov_apply_packed(Cmat, tiles, pc, *, decay, c1, cmu):
    """C <- decay*C + c1*pc pc^T + cmu*dC with dC as packed upper tiles, in place."""
    return _cov_apply('des_cma_cov_apply_packed', Cmat, tiles, 'tiles', True, pc, decay, c1, cmu)


def _cov_apply(fn, Cmat, dC, name, packed, pc, decay, c1, cmu):
    n, dev = Cmat.shape[0], Cmat.device
    _launch(fn, Cmat, 'Cmat', _ptr(Cmat, 'Cmat', F32, n * n), _ptr(dC, name, F32, cma_packed_elems(n) if packed else n * n, dev),
            _ptr(pc, 'pc', F32, n, dev, True), n, decay, c1, cmu)
    return Cmat


# The recordings of closed-loop episodes: defined in ops_record on this module's launcher, listed here so that ops is
# the whole set of single-population ops.
from .ops_record import rollout_record, rollout_record_solutions  # noqa: E402,F401
# The genetic algorithm's ops (genetic.py): defined in ops_ga on this module's checks.
from .ops_ga import ga_order, ga_order_workspace, ga_rows, rollout_eval_ga  # noqa: E402,F401
# Novelty search's ops (novelty.py): defined in ops_novelty on this module's checks.
from .ops_novelty import novelty, ns_shape, ns_shape_workspace, rollout_eval_bc  # noqa: E402,F401
# The genetic algorithm's novelty search's ops (novelty.NoveltyGA): defined in ops_ga_novelty on this module's checks.
from .ops_ga_novelty import ns_ga_order, ns_ga_order_workspace, rollout_eval_ga_bc  # noqa: E402,F401
