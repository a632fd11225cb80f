"""Novelty search's kernels compile clean.  ptxas -v: the five BcArgs instantiations of rollout_pendulum_kernel
(des_envs_bc.cu) spill nothing and take 72, 71, 121, 137 and 167 registers at H = 16, 32, 64, 96 and 128, against 72,
71, 121, 127 and 167 for their RollArgs twins: the twins' allocation granules (8 registers) everywhere but H = 96.  There
the behaviour kernel takes one granule more, as the genetic-algorithm sweep's kernel does (139); this is a deviation from
"within the twins' granules", and a harmless one: shared memory (about 46 KB per CTA at H = 96) already limits an SM to
four 32-thread CTAs, and 144 x 32 registers per CTA does not bind.  The counts are ceilings: nvcc 12.9 does not schedule
this kernel template the same way every time.  Each touches local memory exactly where its twin does (the frame of the
fp64 sincos argument reduction).  The des_novelty kernels spill nothing and have no stack frame, and their SASS has no
local loads or stores.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import CSRC, LIB, _tool

BC = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_6BcArgsEEEvT1_')
BC_REGISTERS = {1: 72, 2: 72, 4: 128, 6: 144, 8: 168}      # R = H/16: ceilings
NOVELTY = re.compile(r'_ZN3des14novelty_kernelILi(\d+)EEEvPfPKflS3_iii')


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
        if m and cur:
            out[cur]['stack'] = int(m.group(1))
            out[cur]['spill'] = int(m.group(2)) + int(m.group(3))
        m = re.search(r'Used (\d+) registers', line)
        if m and cur:
            out[cur]['registers'] = int(m.group(1))
    return out


def test_behaviour_instantiations_keep_their_registers_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_envs_bc.cu', tmp_path).items():
        m = BC.search(name)
        assert m, name                                      # the unit compiles the behaviour kernels only
        seen.add(int(m.group(1)))
        assert rep['spill'] == 0 and rep['registers'] <= BC_REGISTERS[int(m.group(1))], (name, rep)
    assert seen == set(BC_REGISTERS)


def test_novelty_kernels_have_no_stack_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_novelty.cu', tmp_path).items():
        m = NOVELTY.search(name)
        if m:
            seen.add(int(m.group(1)))
        assert rep['spill'] == 0 and rep['stack'] == 0, (name, rep)
    assert seen == {8, 16, 32}


def test_local_memory_of_the_novelty_search_sass():
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
    for R in BC_REGISTERS:
        plain = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_8RollArgsEEEvT1_' % R]
        bc = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6BcArgsEEEvT1_' % R]
        assert plain and len(bc) == len(plain), (R, plain, bc)
    kernels = [name for name in local if NOVELTY.search(name)]
    assert len(kernels) == 3 and all(local[name] == [] for name in kernels)
