"""Build libdes_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m distributedes_b200.build            # build if stale
    python -m distributedes_b200.build --force
"""
from __future__ import annotations

import concurrent.futures
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
OBJ = os.path.join(PKG, 'build')
LIB = os.path.join(PKG, 'libdes_b200.so')
SOURCES = ['des_capi.cu', 'des_noise.cu', 'des_eval_ffma.cu', 'des_eval_tc.cu', 'des_rank.cu', 'des_update.cu',
           'des_cma.cu', 'des_cma_tc.cu', 'des_envs.cu', 'des_envs_sweep.cu', 'des_envs_record.cu', 'des_envs_ga.cu', 'des_ga.cu', 'des_envs_ga_sweep.cu', 'des_ga_sweep.cu', 'des_envs_bc.cu', 'des_envs_bc_sweep.cu', 'des_envs_ga_bc.cu', 'des_novelty.cu', 'des_act.cu', 'des_act_sweep.cu', 'des_obs.cu', 'des_comm.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden']


def _nvcc():
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        raise RuntimeError('nvcc not found: cannot build libdes_b200.so')
    return nvcc


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    headers.append(os.path.join(os.path.dirname(PKG), 'include', 'des_b200.h'))
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + '.o')
        if force or _stale(o, [s] + headers):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', s, '-o', o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (s, r.stdout, r.stderr))
        return r.stderr

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs) or 1)) as ex:
        for log in ex.map(compile_one, jobs):
            if verbose and log:
                print(log)
    objs = [os.path.join(OBJ, src[:-3] + '.o') for src in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [nvcc, '-shared'] + ARCH + ['-o', LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    return LIB


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose='-v' in sys.argv))
