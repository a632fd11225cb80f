"""The recording kernels compile like the kernels they extend.  ptxas -v: the ten RecordArgs instantiations of
rollout_pendulum_kernel (des_envs_record.cu) take at most 72, 80, 120, 128 and 168 registers at H = 16, 32, 64, 96 and
128 (the allocation granules of what they have taken), against 72, 71, 121, 127 and 167 for their RollArgs twins, and
none spills.  The counts are ceilings, not pins: nvcc 12.9 does not compile this kernel template the same way every
time.  Between compiles of one source the recording kernels have taken 72 or 79 registers at H = 32, 95 or 119 at
H = 64 and 167 or 168 at H = 128, and des_envs.cu's rollout_pendulum_kernel<8, false, RunArgs> comes out in more than
one schedule too, before recording existed as after.  A recording is not a per-generation path, so the occupancy the
extra registers may cost at H = 32 is not a concern.  Each touches local memory exactly where its RollArgs twin does
(the 40-byte frame of the fp64 sincos argument reduction).

The RecordArgs instantiations live in des_envs_record.cu, so that des_envs.cu compiles exactly the kernels it did.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import CSRC, LIB, _tool

RECORD = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb([01])ENS_10RecordArgsEEEvT1_')
RECORD_REGISTERS = {R: most for R, most in ((1, 72), (2, 80), (4, 120), (6, 128), (8, 168))}      # R = H/16: ceilings


@pytest.fixture(scope='module')
def report(tmp_path_factory):
    from distributedes_b200.build import NVCC_FLAGS
    nvcc = _tool('nvcc')
    if nvcc is None:
        pytest.skip('nvcc not found')
    out, tmp = {}, tmp_path_factory.mktemp('ptxas')
    r = subprocess.run([nvcc] + NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(CSRC, 'des_envs_record.cu'), '-o',
                                              str(tmp / 'des_envs_record.o')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            out[cur] = {}
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur:
            out[cur]['spill'] = int(m.group(1)) + int(m.group(2))
        m = re.search(r'Used (\d+) registers', line)
        if m and cur:
            out[cur]['registers'] = int(m.group(1))
    return out


def test_recording_instantiations_keep_their_registers_and_spill_nothing(report):
    seen = set()
    for name, rep in report.items():
        m = RECORD.search(name)
        assert m, name                                      # the unit compiles the recording kernels only
        key = (int(m.group(1)), m.group(2) == '1')
        seen.add(key)
        assert rep['spill'] == 0 and rep['registers'] <= RECORD_REGISTERS[key[0]], (name, rep)
    assert seen == {(R, rows) for R in RECORD_REGISTERS for rows in (False, True)}


def test_local_memory_of_the_recording_sass():
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
    for R, b in ((R, b) for R in RECORD_REGISTERS for b in (0, 1)):
        plain = local['_ZN3des23rollout_pendulum_kernelILi%dELb%dENS_8RollArgsEEEvT1_' % (R, b)]
        rec = local['_ZN3des23rollout_pendulum_kernelILi%dELb%dENS_10RecordArgsEEEvT1_' % (R, b)]
        assert plain and len(rec) == len(plain), (R, b, plain, rec)
