#!/usr/bin/env python
"""Generate the mirrored-sampling goldens by running the REFERENCE's natural_es.train() verbatim:

    tests/golden/train_b64_mirrored.npz           tape (d0 24, H 64, A 4, T 16), N 24, 3 generations, normaliser off
    tests/golden/train_closed_mirrored_pend.npz   closed-loop Pendulum-v0, H 16, N 16, 10 repetitions, 2 generations,
                                                  normaliser on, the reset hook of make_golden.py::golden_train_closed

TEST INFRASTRUCTURE.  Runs only where the reference checkout exists; reuses oracle/make_golden.py's setup (paths,
TapeConfig, RecordingAdam, the gym stand-in and its two train() drivers) without changing it and rewrites no other
fixture.

    python oracle/make_golden_mirrored.py

The one difference from make_golden.py: np.random.randn(P) of worker member m in generation g (natural_es.py:29) returns
the mirrored row (-1)^(m & 1) * noise(seed, g, m >> 1), so the reference trains on explicit +-eps pairs and computes its
own fitness_shift, mean(eps * r) / sigma (natural_es.py:90-92) and Adam step from them.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg             # noqa: E402  (sets up sys.path: gym stand-in, reference, repository)

import numpy as np                    # noqa: E402


def mirrored_noise():
    """make_golden.py's drivers draw member m's row as orc.noise(seed, g, m, 1, P)[0]: serve the mirrored row instead."""
    real_noise = mg.orc.noise

    def row(seed, gen, member, n, P, stream=mg.orc.STREAM_NES_EPS):
        assert n == 1 and stream == mg.orc.STREAM_NES_EPS
        return (-1.0) ** (member & 1) * real_noise(seed, gen, member >> 1, 1, P)
    return real_noise, row


def run(fn, *args, **kw):
    real_noise, row = mirrored_noise()
    mg.orc.noise = row
    try:
        fn(*args, **kw)
    finally:
        mg.orc.noise = real_noise


if __name__ == '__main__':
    run(mg.golden_train_verbatim, 'b64_mirrored', 24, 64, 4, 16, 1.0, 24, seed=6, sigma=0.1, lr=0.1, gens=3)
    run(mg.golden_train_closed, 'mirrored_pend', 16, 16, 10, seed=7, sigma=0.1, lr=0.1, gens=2)
    for name in ('train_b64_mirrored.npz', 'train_closed_mirrored_pend.npz'):
        f = os.path.join(mg.OUT, name)
        print(f, os.path.getsize(f), np.load(f).files)
