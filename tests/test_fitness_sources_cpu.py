"""The host logic around the kernels, pinned without a GPU: which device ops every NES and CMA-ES mode launches per
generation, in which order and with which arguments, and which collectives it issues on tensors of which size — one
process and each rank of a 2-rank gloo run.  The kernels are the oracle-backed CPU stand-ins (cpu_ops.py) behind a
recording proxy.  The NES modes a config can describe are pinned a second time through natural_es.build_engine, to the
same records.  Also: the limits each source checks for CMA-ES, and CMA-ES on a host-stepped environment sharded over 2 and 3 gloo ranks against the
single-process run."""
import hashlib
import inspect
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist

import cpu_ops
import host_env_support as hs
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import synth_walk as sw
from ranks import spawn


def _canon(v):
    """Tensors by shape and dtype; numbers by value (the ops cast them to the C types, so 0 and 0.0 are one argument)."""
    if isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool):
        return repr(float(v))
    if isinstance(v, torch.Tensor):
        return 'T%s%s' % (tuple(v.shape), str(v.dtype)[6:])
    if isinstance(v, (list, tuple)):
        return '(%s)' % ','.join(_canon(x) for x in v)
    return repr(v)


class Recorder:
    """Stands in for the kernels module: forwards every attribute, and records each call of a function as its name and
    its arguments bound to the signature (defaults filled in; tensors by shape and dtype).  `hasattr` and `__name__`
    answer as the wrapped module does."""

    def __init__(self, module, log):
        object.__setattr__(self, '_m', module)
        object.__setattr__(self, '_log', log)
        object.__setattr__(self, '__name__', module.__name__)

    def __getattr__(self, name):
        f = getattr(self._m, name)
        if not callable(f):
            return f
        sig = inspect.signature(f)

        def call(*a, **kw):
            b = sig.bind(*a, **kw)
            b.apply_defaults()
            self._log.append((name, tuple((k, _canon(v)) for k, v in b.arguments.items())))
            return f(*a, **kw)
        return call


class record:
    """Records the device ops of `kernels` and the torch.distributed collectives issued inside the block."""
    COLLECTIVES = ('all_reduce', 'all_gather', 'all_gather_into_tensor', 'broadcast', 'reduce_scatter', 'barrier')

    def __init__(self):
        self.log = []
        self.kernels = Recorder(cpu_ops, self.log)

    def __enter__(self):
        self.saved = {n: getattr(dist, n) for n in self.COLLECTIVES}
        for n in self.COLLECTIVES:
            def coll(*a, _n=n, _f=self.saved[n], **kw):
                t = a[0] if a else None
                self.log.append((_n, (('numel', t.numel() if isinstance(t, torch.Tensor) else None),
                                      ('dtype', str(t.dtype)[6:] if isinstance(t, torch.Tensor) else None))))
                return _f(*a, **kw)
            setattr(dist, n, coll)
        return self

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(dist, n, f)

    def trace(self):
        """(the sequence of op and collective names, runs of one name written name*count; a digest of the full
        records)."""
        names = []
        for e in self.log:
            if names and names[-1][0] == e[0]:
                names[-1][1] += 1
            else:
                names.append([e[0], 1])
        return (' '.join(n if k == 1 else '%s*%d' % (n, k) for n, k in names),
                hashlib.sha256(repr(self.log).encode()).hexdigest()[:16])


# ---- the modes ---------------------------------------------------------------------------------------------------------
class Cfg(types.SimpleNamespace):
    """The attributes natural_es.train / cma_es.train read."""

    def __init__(self, **kw):
        super().__init__(**{**dict(state_dim=3, pop_size=6, repetitions=1, test_repetitions=2, max_steps=0,
                                   max_generations=1, seed=7), **kw})


def _nes(mode, kernels):
    from distributedes_b200.engine import HostEnvEngine, NESEngine, RolloutEngine
    mirrored = mode.endswith('mirrored')
    common = dict(pop_size=6, sigma=0.1, learning_rate=0.1, seed=7, device='cpu', kernels=kernels, mirrored=mirrored)
    if mode.startswith('tape'):
        d0, H, A, T = 3, 8, 2, 5
        obs, target = orc.synthetic_tape(T, d0, A)
        return NESEngine(state_dim=d0, hidden=H, action_dim=A, theta0=orc.synthetic_theta(d0, H, A), obs=obs, target=target,
                         clip=1.5, normalize_obs=mode == 'tape_norm', repetitions=2 if mode == 'tape_norm' else 1,
                         **common), Cfg(repetitions=2 if mode == 'tape_norm' else 1)
    if mode.startswith('device'):
        return RolloutEngine(hidden=16, theta0=orc.synthetic_theta(3, 16, 1, seed=2), repetitions=2, horizon=12,
                             action_noise_std=0.1, **common), Cfg(repetitions=2)
    return HostEnvEngine(env_fn=None, state_dim=3, action_dim=1, batch_env_fn=lambda B: po.PendulumBatch(B, 7, horizon=9),
                         hidden=16, theta0=orc.synthetic_theta(3, 16, 1, seed=3), repetitions=2, test_repetitions=3,
                         clip=2.0, **common), Cfg(repetitions=2, test_repetitions=3)


def _nes_config(mode):
    """The config natural_es.build_engine turns into the engine of _nes(mode), for the tape and host-stepped modes (a
    config cannot set the device modes' 12-step horizon)."""
    from distributedes_b200.config import HostEnvConfig, SynthTapeConfig
    if mode.startswith('tape'):         # SynthTapeConfig's tape is orc.synthetic_tape's
        cfg = SynthTapeConfig(hidden_size=8, state_dim=3, action_dim=2, tape_len=5, clip=1.5)
        cfg.initial_weight = orc.synthetic_theta(3, 8, 2)
        cfg.normalize_obs = mode == 'tape_norm'
        cfg.repetitions, cfg.test_repetitions = (2 if cfg.normalize_obs else 1), 2
    else:
        cfg = HostEnvConfig(hs.PendulumProbe, hidden_size=16, clip=2.0,
                            batch_env_fn=lambda B: po.PendulumBatch(B, 7, horizon=9))
        cfg.initial_weight = orc.synthetic_theta(3, 16, 1, seed=3)
        cfg.repetitions, cfg.test_repetitions = 2, 3
    cfg.pop_size, cfg.seed, cfg.max_generations, cfg.mirrored = 6, 7, 1, mode.endswith('mirrored')
    return cfg


def _cma_config(mode, seed=7):
    from distributedes_b200.config import ClosedLoopPendulumConfig, HostEnvConfig, SynthTapeConfig
    from distributedes_b200.envs import GymEnvBatch
    if mode == 'tape':
        cfg = SynthTapeConfig(hidden_size=8, state_dim=3, action_dim=2, tape_len=5)
        cfg.test_repetitions = 2
    elif mode == 'device':
        cfg = ClosedLoopPendulumConfig(16)
        cfg.repetitions = cfg.test_repetitions = 2
    elif mode == 'host':
        cfg = HostEnvConfig(hs.PendulumProbe, hidden_size=16, clip=2.0, task='Pendulum-v0',
                            batch_env_fn=lambda B: po.PendulumBatch(B, seed, horizon=9))
        cfg.repetitions, cfg.test_repetitions = 2, 3
    else:       # episodes of varying length
        cfg = HostEnvConfig(sw.SynthWalkEnv, hidden_size=16, task='SynthWalk-v0',
                            batch_env_fn=lambda B: GymEnvBatch(sw.SynthWalkEnv, B, seed))
        cfg.repetitions, cfg.test_repetitions = 3, 2
    cfg.pop_size, cfg.seed, cfg.max_generations = 6, seed, 2
    return cfg


def _run_nes(mode, from_config=False):
    """natural_es.train over one generation (test, evaluate, rank, gradient, apply; then test and evaluate again), on the
    engine of _nes(mode) or on the one natural_es.build_engine makes of _nes_config(mode)."""
    from distributedes_b200 import natural_es
    rec = record()
    if from_config:
        cfg = _nes_config(mode)
        eng = natural_es.build_engine(cfg, device='cpu', kernels=rec.kernels)
    else:
        eng, cfg = _nes(mode, rec.kernels)
    with rec:
        natural_es.train(cfg, engine=eng)
    return rec.trace()


def _run_cma(mode, cfg=None, kernels=None):
    """cma_es.train over two generations (the second stops before tell); returns its triple and the strategy state."""
    from distributedes_b200 import cma_es
    cfg = cfg if cfg is not None else _cma_config(mode)
    worker = cma_es.Worker(0, None, None, None, None, cfg, device='cpu', kernels=kernels)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, cfg.pop_size, seed=cfg.seed, device='cpu',
                                     kernels=kernels)
    rewards, steps, _ = cma_es.train(cfg, worker=worker, es=es)
    stats = getattr(worker, 'obs_stats', None)
    stats = stats.numpy().copy() if stats is not None else np.zeros(0)
    return dict(rewards=np.asarray(rewards), steps=np.asarray(steps), m=es.m.numpy(), sigma=es.sigma, C=es.C.numpy(),
                stats=stats)


def _trace_cma(mode):
    rec = record()
    with rec:
        _run_cma(mode, kernels=rec.kernels)
    return rec.trace()


def _traces():
    return ({('nes', m): _run_nes(m) for m in NES_MODES} | {('cma', m): _trace_cma(m) for m in CMA_MODES}
            | {('nes_config', m): _run_nes(m, from_config=True) for m in NES_CONFIG_MODES})


NES_MODES = ('tape', 'tape_mirrored', 'tape_norm', 'device', 'device_mirrored', 'host', 'host_mirrored')
CMA_MODES = ('tape', 'device', 'host')
NES_CONFIG_MODES = ('tape', 'tape_mirrored', 'tape_norm', 'host', 'host_mirrored')     # built through build_engine


# per mode, recorded from the host layer as it was before the fitness sources (fitness.py) took over the evaluation:
# (one process, gloo rank 0, gloo rank 1), each as (op and collective names, digest of the full records)
EXPECTED = {('cma', 'device'): (('rollout_eval noise_fill rollout_eval_solutions rollout_eval centered_rank cma_rank_mu '
                                 'cma_cov_apply obs_stats_merge_totals noise_fill rollout_eval_solutions rollout_eval',
                                 '400dab08b1adf49a'),
                                ('rollout_eval noise_fill rollout_eval_solutions all_reduce*2 rollout_eval centered_rank '
                                 'cma_packed_elems cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed all_reduce '
                                 'obs_stats_merge_totals noise_fill rollout_eval_solutions all_reduce*2 rollout_eval',
                                 'cb4e32b88b02638d'),
                                ('rollout_eval noise_fill rollout_eval_solutions all_reduce*2 rollout_eval centered_rank '
                                 'cma_packed_elems cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed all_reduce '
                                 'obs_stats_merge_totals noise_fill rollout_eval_solutions all_reduce*2 rollout_eval',
                                 '8d77cbe688d72a42')),
            ('cma', 'host'): (('policy_act*9 noise_fill policy_act*9 obs_parts_reduce policy_act*9 centered_rank cma_rank_mu '
                               'cma_cov_apply obs_stats_merge_totals noise_fill policy_act*9 obs_parts_reduce policy_act*9',
                               '09a6ac6a3d34a395'),
                              ('policy_act*9 noise_fill policy_act*9 obs_parts_reduce all_reduce*3 policy_act*9 centered_rank '
                               'cma_packed_elems cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed all_reduce '
                               'obs_stats_merge_totals noise_fill policy_act*9 obs_parts_reduce all_reduce*3 policy_act*9',
                               'df39dd3dc9bf694f'),
                              ('policy_act*9 noise_fill policy_act*9 obs_parts_reduce all_reduce*3 policy_act*9 centered_rank '
                               'cma_packed_elems cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed all_reduce '
                               'obs_stats_merge_totals noise_fill policy_act*9 obs_parts_reduce all_reduce*3 policy_act*9',
                               '937282d6d05250a6')),
            ('cma', 'tape'): (('pop_eval*2 noise_fill pop_eval*3 centered_rank cma_rank_mu cma_cov_apply noise_fill pop_eval*3',
                               '401679c3759bf992'),
                              ('pop_eval*2 noise_fill pop_eval all_reduce*2 pop_eval*2 centered_rank cma_packed_elems '
                               'cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed noise_fill pop_eval all_reduce*2 pop_eval*2',
                               '80214682d226b09a'),
                              ('pop_eval*2 noise_fill pop_eval all_reduce*2 pop_eval*2 centered_rank cma_packed_elems '
                               'cma_rank_mu_packed all_reduce*2 cma_cov_apply_packed noise_fill pop_eval all_reduce*2 pop_eval*2',
                               'b454acec8793de43')),
            ('nes', 'device'): (('param_count new_state rank_workspace grad_workspace rollout_eval*2 centered_rank '
                                 'nes_grad_partial nes_apply state_advance obs_stats_merge_totals rollout_eval*2',
                                 '8acc9100499beb9b'),
                                ('param_count new_state rank_workspace grad_workspace rollout_eval*2 all_reduce*2 centered_rank '
                                 'nes_grad_partial all_reduce nes_apply state_advance obs_stats_merge_totals rollout_eval*2 '
                                 'all_reduce*2',
                                 '8230dfdf17129a63'),
                                ('param_count new_state rank_workspace grad_workspace rollout_eval*2 all_reduce*2 centered_rank '
                                 'nes_grad_partial all_reduce nes_apply state_advance obs_stats_merge_totals rollout_eval*2 '
                                 'all_reduce*2',
                                 '912823285ecd2912')),
            ('nes', 'device_mirrored'): (('param_count new_state rank_workspace grad_workspace rollout_eval rollout_eval_mirrored '
                                          'centered_rank nes_grad_partial_mirrored nes_apply state_advance obs_stats_merge_totals '
                                          'rollout_eval rollout_eval_mirrored',
                                          'bc487a509a875d66'),
                                         ('param_count new_state rank_workspace grad_workspace rollout_eval rollout_eval_mirrored '
                                          'all_reduce*2 centered_rank nes_grad_partial_mirrored all_reduce nes_apply '
                                          'state_advance obs_stats_merge_totals rollout_eval rollout_eval_mirrored all_reduce*2',
                                          '3b3e30ecd29efb6c'),
                                         ('param_count new_state rank_workspace grad_workspace rollout_eval rollout_eval_mirrored '
                                          'all_reduce*2 centered_rank nes_grad_partial_mirrored all_reduce nes_apply '
                                          'state_advance obs_stats_merge_totals rollout_eval rollout_eval_mirrored all_reduce*2',
                                          'f686ec8096ab6cb3')),
            ('nes', 'host'): (('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb policy_act*9 '
                               'obs_parts_reduce centered_rank nes_grad_partial nes_apply state_advance obs_stats_merge_totals '
                               'policy_act*9 nes_perturb policy_act*9 obs_parts_reduce',
                               'aae91ee203cf034d'),
                              ('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb policy_act*9 '
                               'obs_parts_reduce all_reduce*3 centered_rank nes_grad_partial all_reduce nes_apply state_advance '
                               'obs_stats_merge_totals policy_act*9 nes_perturb policy_act*9 obs_parts_reduce all_reduce*3',
                               '1b5cdd3614b28620'),
                              ('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb policy_act*9 '
                               'obs_parts_reduce all_reduce*3 centered_rank nes_grad_partial all_reduce nes_apply state_advance '
                               'obs_stats_merge_totals policy_act*9 nes_perturb policy_act*9 obs_parts_reduce all_reduce*3',
                               'f4bdbb9d2cf7bef6')),
            ('nes', 'host_mirrored'): (('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb_mirrored '
                                        'policy_act*9 obs_parts_reduce centered_rank nes_grad_partial_mirrored nes_apply '
                                        'state_advance obs_stats_merge_totals policy_act*9 nes_perturb_mirrored policy_act*9 '
                                        'obs_parts_reduce',
                                        'f1e4fa76059a8a8f'),
                                       ('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb_mirrored '
                                        'policy_act*9 obs_parts_reduce all_reduce*3 centered_rank nes_grad_partial_mirrored '
                                        'all_reduce nes_apply state_advance obs_stats_merge_totals policy_act*9 '
                                        'nes_perturb_mirrored policy_act*9 obs_parts_reduce all_reduce*3',
                                        '7f92a5474511fdab'),
                                       ('param_count new_state rank_workspace grad_workspace policy_act*9 nes_perturb_mirrored '
                                        'policy_act*9 obs_parts_reduce all_reduce*3 centered_rank nes_grad_partial_mirrored '
                                        'all_reduce nes_apply state_advance obs_stats_merge_totals policy_act*9 '
                                        'nes_perturb_mirrored policy_act*9 obs_parts_reduce all_reduce*3',
                                        '8aeb092ba99a102f')),
            ('nes', 'tape'): (('param_count new_state rank_workspace grad_workspace nes_eval*3 centered_rank nes_grad_partial '
                               'nes_apply state_advance nes_eval*3',
                               'f690cd4fabefcfec'),
                              ('param_count new_state rank_workspace grad_workspace nes_eval*3 all_reduce centered_rank '
                               'nes_grad_partial all_reduce nes_apply state_advance nes_eval*3 all_reduce',
                               '776564cfe8f56704'),
                              ('param_count new_state rank_workspace grad_workspace nes_eval*3 all_reduce centered_rank '
                               'nes_grad_partial all_reduce nes_apply state_advance nes_eval*3 all_reduce',
                               '515aa86f8208fae9')),
            ('nes', 'tape_mirrored'): (('param_count new_state rank_workspace grad_workspace nes_eval*2 nes_eval_mirrored '
                                        'centered_rank nes_grad_partial_mirrored nes_apply state_advance nes_eval*2 '
                                        'nes_eval_mirrored',
                                        '7740d8c41a1fbc88'),
                                       ('param_count new_state rank_workspace grad_workspace nes_eval*2 nes_eval_mirrored '
                                        'all_reduce centered_rank nes_grad_partial_mirrored all_reduce nes_apply state_advance '
                                        'nes_eval*2 nes_eval_mirrored all_reduce',
                                        'b9b801d7ba0de48f'),
                                       ('param_count new_state rank_workspace grad_workspace nes_eval*2 nes_eval_mirrored '
                                        'all_reduce centered_rank nes_grad_partial_mirrored all_reduce nes_apply state_advance '
                                        'nes_eval*2 nes_eval_mirrored all_reduce',
                                        'a537587a35e08251')),
            ('nes', 'tape_norm'): (('param_count new_state rank_workspace grad_workspace obs_normalize nes_eval obs_normalize '
                                    'nes_eval obs_normalize nes_eval centered_rank nes_grad_partial nes_apply state_advance '
                                    'obs_stats_merge obs_normalize nes_eval obs_normalize nes_eval obs_normalize nes_eval',
                                    'eef0b1207d01e319'),
                                   ('param_count new_state rank_workspace grad_workspace obs_normalize nes_eval obs_normalize '
                                    'nes_eval obs_normalize nes_eval all_reduce centered_rank nes_grad_partial all_reduce '
                                    'nes_apply state_advance obs_stats_merge obs_normalize nes_eval obs_normalize nes_eval '
                                    'obs_normalize nes_eval all_reduce',
                                    '38299527527bfbb9'),
                                   ('param_count new_state rank_workspace grad_workspace obs_normalize nes_eval obs_normalize '
                                    'nes_eval obs_normalize nes_eval all_reduce centered_rank nes_grad_partial all_reduce '
                                    'nes_apply state_advance obs_stats_merge obs_normalize nes_eval obs_normalize nes_eval '
                                    'obs_normalize nes_eval all_reduce',
                                    'a802077aaf99a0ce'))}


def _expected():
    """EXPECTED, and each NES mode built from a config expects the row of the engine built directly."""
    return list(EXPECTED.items()) + [(('nes_config', m), EXPECTED[('nes', m)]) for m in NES_CONFIG_MODES]


def test_every_mode_issues_the_pinned_ops_and_collectives_in_one_process():
    got = _traces()
    for key, (one, _, _) in _expected():
        assert got[key] == one, key


def test_every_mode_issues_the_pinned_ops_and_collectives_on_each_of_two_gloo_ranks():
    r = spawn(2, _traces)
    for key, (_, r0, r1) in _expected():
        assert (r[0][key], r[1][key]) == (r0, r1), key


@pytest.mark.parametrize('mode,attr,value', [('device', 'repetitions', 11), ('host', 'repetitions', 17),
                                             ('host', 'test_repetitions', 17), ('host', 'state_dim', 33)])
def test_a_cma_worker_is_refused_a_config_its_source_cannot_run(mode, attr, value):
    """Each source checks its own limits when it is built, so CMA-ES meets them when its Worker is made."""
    from distributedes_b200 import cma_es
    cfg = _cma_config(mode)
    setattr(cfg, attr, value)
    with pytest.raises(ValueError, match=attr):
        cma_es.Worker(0, None, None, None, None, cfg, device='cpu', kernels=cpu_ops)


def _walk_cma():
    cfg = _cma_config('walk', seed=5)
    cfg.pop_size, cfg.max_generations = 5, 3
    return _run_cma('walk', cfg=cfg, kernels=cpu_ops)


@pytest.mark.parametrize('world', [2, 3])
def test_host_stepped_cma_sharded_over_gloo_ranks_equals_the_single_process_run(world):
    """cma_es.train on SynthWalk (episodes of 40-160 steps) with ragged shards (3 + 2, 2 + 2 + 1): each rank steps its
    own solutions' environments; the costs, the step counts summed over ranks, the observation totals and the test
    episodes of the best solution give the single-process run's results."""
    one = _walk_cma()
    res = spawn(world, _walk_cma)
    for r in res[1:]:
        for k in one:
            assert np.array_equal(r[k], res[0][k]), k
    r = res[0]
    assert np.array_equal(r['steps'], one['steps']) and len(set(np.diff(one['steps']))) > 1
    # generation 0 is bit-equal; afterwards the strategy state carries the rounding of the per-rank partial sums
    assert np.array_equal(r['rewards'][:2], one['rewards'][:2])
    assert np.allclose(r['rewards'], one['rewards'], rtol=1e-5)
    for k in ('m', 'C', 'stats'):
        assert np.allclose(r[k], one[k], rtol=1e-5, atol=1e-6), k
    assert abs(r['sigma'] - one['sigma']) <= 1e-6 * one['sigma']
