"""Minimal stand-in for the third-party ``cma`` package (pycma) so the reference's cma_es.py imports and runs verbatim
where pycma is not installed.  TEST INFRASTRUCTURE ONLY: oracle/make_golden.py puts this directory on sys.path; the
product package never imports it.

Only what cma_es.py:43-49, :62 and :90 touch exists: ``CMAOptions`` (a dict; only 'popsize' is read) and
``CMAEvolutionStrategy(x0, sigma, opts)`` whose ask() / tell() wrap oracle/cma_oracle.CMAState, the fp64 restatement of
the tutorial algorithm (so "the reference's CMA-ES" means the reference's loop around that restatement).

ask() draws z from the counter noise the device's ask() uses: Philox stream tag 1, counter (j/4, member = index,
generation = number of tell() calls so far), key = ``noise_seed`` (module attribute), rounded to fp32 like the device's
samples.  Every instance is appended to ``instances``; each keeps what tell() was handed and the state it left.
"""
import numpy as np

from oracle import cma_oracle
from oracle import nes_oracle as orc

noise_seed = 0
instances = []


class CMAOptions(dict):
    pass


class CMAEvolutionStrategy:
    def __init__(self, x0, sigma0, opts=None):
        opts = opts if opts is not None else CMAOptions()
        self.state = cma_oracle.CMAState(np.asarray(x0, dtype=np.float64), float(sigma0), int(opts['popsize']))
        self.seed = int(noise_seed)
        self.told = []            # per tell(): dict(solutions, cost, m, sigma, pc, ps) after the update
        instances.append(self)

    def ask(self):
        st = self.state
        z = orc.noise(self.seed, st.gen, 0, st.lam, st.n, stream=orc.STREAM_CMA_Z).astype(np.float32).astype(np.float64)
        X = st.ask(z)
        return [X[i].copy() for i in range(st.lam)]

    def tell(self, solutions, cost):
        X = np.asarray(solutions, dtype=np.float64)
        c = np.asarray(cost, dtype=np.float64)
        self.state.tell(X, c)
        st = self.state
        self.told.append(dict(solutions=X.copy(), cost=c.copy(), m=st.m.copy(), sigma=st.sigma, pc=st.pc.copy(),
                              ps=st.ps.copy()))
