"""The genetic algorithm's kernels compile like the kernels they extend.  ptxas -v: the five GaArgs instantiations of
rollout_pendulum_kernel (des_envs_ga.cu) took 72, 71, 121, 127 and 167 registers at H = 16, 32, 64, 96 and 128, the
counts of their RollArgs twins, and none spills.  The ceilings below are the allocation granules of those counts, not
pins: nvcc 12.9 does not compile this kernel template the same way every time (test_sass_record.py).  Each touches local
memory exactly where its RollArgs twin does (the 40-byte frame of the fp64 sincos argument reduction).  The kernels of
des_ga.cu take at most 32 registers and have no stack frame.

The GaArgs instantiations live in des_envs_ga.cu, so that des_envs.cu compiles exactly the kernels it did.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import CSRC, LIB, _tool

GA = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_6GaArgsEEEvT1_')
GA_REGISTERS = {1: 72, 2: 72, 4: 128, 6: 128, 8: 168}          # R = H/16: ceilings
TABLE_KERNELS = {'ga_rows_kernel': 32, 'ga_negate_kernel': 16, 'ga_scatter_kernel': 16}


def _ptxas(unit, tmp):
    from distributedes_b200.build import NVCC_FLAGS
    nvcc = _tool('nvcc')
    if nvcc is None:
        pytest.skip('nvcc not found')
    r = subprocess.run([nvcc] + NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(CSRC, unit), '-o', str(tmp / 'u.o')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            out[cur] = {}
        m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur and 'frame' not in out[cur]:
            out[cur].update(frame=int(m.group(1)), spill=int(m.group(2)) + int(m.group(3)))
        m = re.search(r'Used (\d+) registers', line)
        if m and cur:
            out[cur]['registers'] = int(m.group(1))
    return out


def test_ga_rollout_instantiations_keep_their_registers_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_envs_ga.cu', tmp_path).items():
        m = GA.search(name)
        assert m, name                                      # the unit compiles the GA kernels only
        R = int(m.group(1))
        seen.add(R)
        assert rep['spill'] == 0 and rep['registers'] <= GA_REGISTERS[R], (name, rep)
    assert seen == set(GA_REGISTERS)


def test_table_kernels_spill_nothing(tmp_path):
    rep = _ptxas('des_ga.cu', tmp_path)
    assert len(rep) == len(TABLE_KERNELS)
    for name, r in rep.items():
        short = next(k for k in TABLE_KERNELS if k in name)
        assert r['spill'] == 0 and r['frame'] == 0 and r['registers'] <= TABLE_KERNELS[short], (name, r)


def test_local_memory_of_the_ga_sass():
    tool = _tool('cuobjdump')
    if tool is None or not os.path.exists(LIB):
        pytest.skip('cuobjdump or the built library missing')
    r = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    local, cur = {}, None
    for line in r.stdout.splitlines():
        if 'Function :' in line:
            cur = line.split('Function :')[1].strip()
            local[cur] = []
        elif cur is not None and re.match(r'\s*/\*[0-9a-f]{4,}\*/', line):
            ins = line.split(';')[0].split('*/', 1)[1].strip()
            if re.search(r'\b(STL|LDL)\b', ins):
                local[cur].append(ins)
    for R in GA_REGISTERS:
        plain = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_8RollArgsEEEvT1_' % R]
        ga = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6GaArgsEEEvT1_' % R]
        assert plain and len(ga) == len(plain), (R, plain, ga)
    for name, ins in local.items():
        if any(k in name for k in TABLE_KERNELS):
            assert not ins, (name, ins)
