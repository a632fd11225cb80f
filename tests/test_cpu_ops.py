"""cpu_ops stands in for distributedes_b200.ops in the CPU tests of the host logic, so it must take the arguments the
ops take: a change to an op's signature fails here, not only on a GPU.  ops imports without the library or a GPU."""
import inspect

import cpu_ops
from distributedes_b200 import ops

# ops without a stand-in
ABSENT = {
    'eval_workspace': 'without it the tape evaluation allocates no workspace (fitness.Tape asks with hasattr)',
    'read_state': 'checkpoint I/O on the des_state tensor, never reached through `kernels`',
}
# stand-ins whose signature differs from the op's
OWN_SIGNATURE = {
    'param_count': "(d0, H, A): test_fitness_sources_cpu's digests bind every call's arguments by these names",
    'noise_fill': "the stand-in's default device is the CPU",
}


def _functions(module):
    return {n: f for n, f in vars(module).items()
            if inspect.isfunction(f) and f.__module__ == module.__name__ and not n.startswith('_')}


def test_every_op_has_a_stand_in_with_its_signature():
    ours, theirs = _functions(cpu_ops), _functions(ops)
    assert set(ours) == set(theirs) - set(ABSENT)
    for name in set(ours) - set(OWN_SIGNATURE):
        assert inspect.signature(ours[name]) == inspect.signature(theirs[name]), name
