"""Time des_rollout_record (all four trajectories written) against des_rollout_eval on the same arguments, with CUDA
events after a warm-up, the two entry points alternated in one process: the reference's shape (64 members x 10 episodes
x 200 steps) and 2048 members, at H = 16 .. 128.  Each shape also compares the outputs the two share (fitness, episode
returns, observation totals) on the same seed, bit for bit.  Prints one JSON line per shape and the GPU's name and
power limit.

    python scripts/time_record.py [--reps K]
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedes_b200 import ops  # noqa: E402
from distributedes_b200.model import StandardFCNet  # noqa: E402


def gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name()
    return q


def main():
    K = int(sys.argv[sys.argv.index('--reps') + 1]) if '--reps' in sys.argv else 20
    print(json.dumps(dict(gpu=gpu())))
    for N in (64, 2048):
        for H in (16, 32, 64, 96, 128):
            theta = torch.from_numpy(StandardFCNet(3, 1, H, seed=0).get_weight()).cuda()
            stats = torch.tensor([0.1, 0.2, 0.3, 0.5, 0.4, 20.0, 1000.0], dtype=torch.float32, device='cuda')
            kw = dict(hidden=H, horizon=200, repetitions=10, sigma=0.1, clip=2.0, action_noise_std=0.1, seed=7,
                      generation=3, n_local=N, obs_stats=stats)

            def outs():
                return dict(out=torch.empty(N, device='cuda'), episodes_out=torch.empty((N, 10), device='cuda'),
                            totals_out=torch.empty(7, dtype=torch.float64, device='cuda'),
                            workspace=torch.empty(N * 7, dtype=torch.float64, device='cuda'))
            e, r = outs(), outs()
            traj = dict(states_out=torch.empty((N, 10, 200, 2), dtype=torch.float64, device='cuda'),
                        obs_out=torch.empty((N, 10, 200, 3), device='cuda'),
                        actions_out=torch.empty((N, 10, 200, 1), device='cuda'),
                        rewards_out=torch.empty((N, 10, 200), dtype=torch.float64, device='cuda'))
            run_e = lambda: ops.rollout_eval(theta, **kw, **e)                    # noqa: E731
            run_r = lambda: ops.rollout_record(theta, **kw, **r, **traj)          # noqa: E731
            for _ in range(3):
                run_e()
                run_r()
            torch.cuda.synchronize()
            same = all(torch.equal(e[k].view(torch.int32) if e[k].dtype == torch.float32 else e[k].view(torch.int64),
                                   r[k].view(torch.int32) if r[k].dtype == torch.float32 else r[k].view(torch.int64))
                       for k in ('out', 'episodes_out', 'totals_out'))
            te, tr = [], []
            for _ in range(K):
                for fn, acc in ((run_e, te), (run_r, tr)):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    fn()
                    b.record()
                    b.synchronize()
                    acc.append(a.elapsed_time(b))
            me, mr = float(np.median(te)), float(np.median(tr))
            nbytes = sum(t.numel() * t.element_size() for t in traj.values())
            print(json.dumps(dict(members=N, hidden=H, eval_ms=round(me, 4), record_ms=round(mr, 4),
                                  overhead=round(mr / me - 1, 4), trajectory_MB=round(nbytes / 2 ** 20, 1),
                                  shared_outputs_bit_equal=bool(same))))


if __name__ == '__main__':
    main()
