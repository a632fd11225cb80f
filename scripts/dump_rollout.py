"""Dump des_rollout_eval outputs (fitness, episode returns, observation totals) on seeded inputs at H = 32, 64, 96 and 128
into one .npz, for byte comparison of two builds of the library.  The library is called through ctypes directly, with
only the des_rollout_eval signature declared, so a build that predates later entry points loads too.

    python scripts/dump_rollout.py <out.npz> [<libdes_b200.so>]        # default: the in-tree library
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from distributedes_b200 import _lib      # noqa: E402
from oracle import nes_oracle as orc     # noqa: E402


def main(out, path):
    lib = C.CDLL(path)
    fn = lib.des_rollout_eval
    fn.restype, fn.argtypes = _lib.SIGNATURES['des_rollout_eval']
    torch.cuda.set_device(0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for H in (32, 64, 96, 128):
        theta = torch.from_numpy(orc.synthetic_theta(3, H, 1, seed=H)).cuda()
        stats = torch.tensor([-0.2, 0.01, 0.3, 0.5, 0.4, 20.0, 32000.0], dtype=torch.float32, device='cuda')
        for tag, noise, st in (('plain', 0.0, None), ('stats_noise', 0.3, stats)):
            n, reps = 37, 10
            fit = torch.empty(n, dtype=torch.float32, device='cuda')
            ep = torch.empty(n * reps, dtype=torch.float32, device='cuda')
            tot = torch.empty(7, dtype=torch.float64, device='cuda')
            ws = torch.empty(n * 7, dtype=torch.float64, device='cuda')
            rc = fn(C.c_void_p(fit.data_ptr()), C.c_void_p(ep.data_ptr()), C.c_void_p(tot.data_ptr()),
                    C.c_void_p(theta.data_ptr()), C.c_void_p(st.data_ptr() if st is not None else 0), 0,
                    _lib.Dims(3, H, 1, 200), reps, 0.1, 2.0, noise, 19, 5, None, 11, n, 0, C.c_void_p(ws.data_ptr()),
                    ws.numel() * 8, stream)
            assert rc == 0, rc
            torch.cuda.synchronize()
            for k, v in (('fit', fit), ('ep', ep), ('tot', tot)):
                res['%s_%d_%s' % (k, H, tag)] = v.cpu().numpy()
    np.savez(out, **res)
    print('%s: %d arrays from %s' % (out, len(res), path))


if __name__ == '__main__':
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else _lib.LIB_PATH)
