"""H100-native (sm_90a) Evolution-Strategies hot path (NES population-evaluate-update loop + CMA-ES rank-mu update).

Product code = csrc/*.cu behind the C ABI of include/des_b200.h (libdes_b200.so) + this thin host layer that
keeps the reference's Worker / train() / test() / Evaluator.eval() / fitness_shift / Adam surface.
Importing the package does not need a GPU; calling anything that computes does (no CPU fallback).
"""
from . import _lib  # noqa: F401

__all__ = ['ops', 'engine', 'natural_es', 'cma_es', 'utils', 'model', 'config', 'envs']
