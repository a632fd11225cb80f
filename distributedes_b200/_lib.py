"""ctypes binding of libdes_b200.so (include/des_b200.h).

The library is the product; this module only loads it and declares signatures.  There is no CPU
fallback: if the shared object is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# DES_LIB_PATH selects another build of the same library (kernel experiments: scripts/build_variant.sh)
LIB_PATH = os.environ.get('DES_LIB_PATH') or os.path.join(_PKG, 'libdes_b200.so')

DES_OK = 0
FWD_FP32, FWD_F16, FWD_F16X3 = 0, 1, 2
PRECISIONS = {'fp32': FWD_FP32, 'f16': FWD_F16, 'f16x3': FWD_F16X3}
STREAM_NES_EPS, STREAM_CMA_Z = 0, 1


class Dims(C.Structure):
    _fields_ = [('state_dim', C.c_int32), ('hidden', C.c_int32), ('action_dim', C.c_int32), ('tape_len', C.c_int32)]


class Opt(C.Structure):
    _fields_ = [('sigma', C.c_double), ('learning_rate', C.c_double), ('weight_decay', C.c_double),
                ('beta1', C.c_double), ('beta2', C.c_double), ('epsilon', C.c_double)]


class State(C.Structure):
    _fields_ = [('generation', C.c_uint64), ('adam_t', C.c_uint64), ('beta1_t', C.c_double), ('beta2_t', C.c_double)]


_P, _I64, _U64, _U32, _I32, _D, _SZ = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32, C.c_double, C.c_size_t

# name -> (restype, argtypes); must list every symbol include/des_b200.h declares (tests check this)
SIGNATURES = {
    'des_last_error': (C.c_char_p, []),
    'des_version': (C.c_char_p, []),
    'des_device_count': (C.c_int, []),
    'des_param_count': (_I64, [_I32, _I32, _I32]),
    'des_noise_fill': (C.c_int, [_P, _I64, _I64, _U64, _U64, _I64, _U32, _P]),
    'des_nes_perturb': (C.c_int, [_P, _P, _I64, _I64, _D, _U64, _U64, _I64, _P]),
    'des_nes_perturb_mirrored': (C.c_int, [_P, _P, _I64, _I64, _D, _U64, _U64, _I64, _P]),
    'des_obs_stats_merge': (C.c_int, [_P, _P, _I32, _I32, _D, _P]),
    'des_obs_normalize': (C.c_int, [_P, _P, _P, _I32, _I32, _P]),
    'des_rollout_eval': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, Dims, _I32, _D, _D, _D, _U64, _U64, _P, _I64, _I64, C.c_int,
                                   _P, C.c_size_t, _P]),
    'des_rollout_eval_mirrored': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, Dims, _I32, _D, _D, _D, _U64, _U64, _P, _I64, _I64,
                                            C.c_int, _P, C.c_size_t, _P]),
    'des_rollout_eval_solutions': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, Dims, _I32, _D, _D, _U64, _U64, _I64, _I64, _P,
                                             C.c_size_t, _P]),
    'des_obs_stats_merge_totals': (C.c_int, [_P, _P, _I32, _P]),
    'des_rollout_eval_runs': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, Dims, _I32, _D, _D, _D, _U64, _U64, _P, _I64, _I64,
                                        C.c_int, _P, C.c_size_t, _P]),
    'des_rank_runs_workspace_bytes': (_SZ, [_I64, _I64]),
    'des_centered_rank_runs': (C.c_int, [_P, _P, _P, _I64, _I64, _P, _SZ, _P]),
    'des_grad_runs_workspace_bytes': (_SZ, [_I64, _I64, _I64]),
    'des_nes_grad_partial_runs': (C.c_int, [_P, _P, _I64, _I64, _I64, _U64, _U64, _P, _P, _SZ, _P]),
    'des_nes_apply_runs': (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _I64, _I64, Opt, _P, _P]),
    'des_obs_stats_merge_totals_runs': (C.c_int, [_P, _P, _I32, _I64, _P]),
    'des_policy_act': (C.c_int, [_P, _P, _P, _I64, _P, _P, _P, Dims, _I32, _D, _D, _U64, _U64, _I64, _I64, _I64, _P]),
    'des_obs_parts_reduce': (C.c_int, [_P, _P, _I64, _I32, _P]),
    'des_nes_eval_workspace_bytes': (_SZ, [Dims, C.c_int]),
    'des_nes_eval': (C.c_int, [_P, _P, _P, _P, Dims, _D, _D, _U64, _U64, _P, _I64, _I64, C.c_int, _P, _SZ, _P]),
    'des_nes_eval_mirrored': (C.c_int, [_P, _P, _P, _P, Dims, _D, _D, _U64, _U64, _P, _I64, _I64, C.c_int, _P, _SZ, _P]),
    'des_pop_eval': (C.c_int, [_P, _P, _P, _P, Dims, _D, _I64, _P]),
    'des_rank_workspace_bytes': (_SZ, [_I64, _I64]),
    'des_centered_rank': (C.c_int, [_P, _P, _P, _I64, _I64, _I64, _P, _SZ, _P]),
    'des_grad_workspace_bytes': (_SZ, [_I64, _I64]),
    'des_nes_grad_partial': (C.c_int, [_P, _P, _I64, _I64, _U64, _U64, _P, _I64, _P, _SZ, _P]),
    'des_nes_grad_partial_mirrored': (C.c_int, [_P, _P, _I64, _I64, _U64, _U64, _P, _I64, _P, _SZ, _P]),
    'des_nes_apply': (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _I64, Opt, _P, _P]),
    'des_state_init': (C.c_int, [_P, _U64, _P]),
    'des_state_advance': (C.c_int, [_P, _D, _D, _P]),
    'des_cma_rank_mu_workspace_bytes': (_SZ, [_I64, _I64]),
    'des_cma_rank_mu': (C.c_int, [_P, _P, _P, _I64, _I64, C.c_int, _P, _SZ, _P]),
    'des_cma_cov_apply': (C.c_int, [_P, _P, _P, _I64, _D, _D, _D, _P]),
    'des_cma_packed_elems': (_I64, [_I64]),
    'des_cma_cov_apply_packed': (C.c_int, [_P, _P, _P, _I64, _D, _D, _D, _P]),
    'des_comm_create': (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, _I64, _I64, _P]),
    'des_comm_connect': (C.c_int, [_P, _P]),
    'des_comm_destroy': (None, [_P]),
    'des_comm_fitness_all_dev': (_P, [_P]),
    'des_comm_allgather_fitness': (C.c_int, [_P, _I64, _I64, _P]),
    'des_comm_allreduce_partial': (C.c_int, [_P, _P, _P, _I64, _P]),
    'des_session_create': (C.c_int, [C.POINTER(_P), C.c_int, Dims, _I64, _I64, _I64, Opt, _D, _U64, C.c_int, _P]),
    'des_session_destroy': (None, [_P]),
    'des_session_generation_host': (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    'des_session_upload_tape': (C.c_int, [_P, _P, _P]),
    'des_session_eval': (C.c_int, [_P]),
    'des_session_rank_and_grad': (C.c_int, [_P]),
    'des_session_apply': (C.c_int, [_P]),
    'des_session_fitness_all_dev': (_P, [_P]),
    'des_session_partial_dev': (_P, [_P]),
    'des_session_theta_dev': (_P, [_P]),
    'des_session_stream': (_P, [_P]),
    'des_session_sync': (C.c_int, [_P]),
}

_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises RuntimeError if the .so is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'distributedes_b200: %s is missing. Build it with `python -m distributedes_b200.build` '
            '(needs nvcc). There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)        # AttributeError if the library lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=''):
    if rc != DES_OK:
        msg = load().des_last_error().decode('utf-8', 'replace')
        raise RuntimeError('%s failed (status %d): %s' % (what or 'des_b200 call', rc, msg))
