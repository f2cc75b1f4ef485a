"""Output hashes of the one-GEMM kernel (`ops.zgemm`, modes 1 and 3) on host-generated inputs, for
tests/test_gpu_zgemm_bitexact.py.

The kernel promises the same fp32 operations in the same order whatever its pipeline looks like, so its outputs are
compared bit for bit against this fixture: SHA-256 of the raw float32 output (including the 7.0 fill it must overwrite), and a
few sampled values so that a mismatch can say how far off it is.  Inputs come from detfill (counter-based, no RNG library),
so the fixture does not depend on torch's random streams.

    python tests/golden/gen_zgemm_hashes.py [out.json]      # on an H100; default tests/golden/zgemm_hashes.json
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from detfill import det_normal  # noqa: E402

FIXTURE = os.path.join(HERE, 'zgemm_hashes.json')
N_SAMPLES = 8

# (C_in, ncomp, cplus, cminus, Kp): mode 3 weight-set blocks of L = 8, 4 (a K = 32 pair: two sub-segments), 2, 1
MIXED_L = [(96, 3, 2, 0, 16), (16, 5, 3, 1, 32), (40, 7, 4, 2, 16), (12, 3, 2, 0, 16)]
HEADLINE = {1: [(512, 1, 0, 0, 16), (512, 3, 1, 1, 16), (512, 5, 2, 2, 16)],
            3: [(512, 3, 2, 0, 16), (512, 5, 3, 1, 16), (512, 7, 4, 2, 16)]}


def cases():
    """{name: (mode, Co, E, segments, flush)}"""
    out = {}
    for mode in (1, 3):
        for Co in (128, 384, 512):
            for E in (129, 300):
                for flush in (0, 1, 3, 5, 1 << 20):
                    out[f'm{mode}_Co{Co}_E{E}_f{flush}'] = (mode, Co, E, MIXED_L, flush)
        out[f'm{mode}_headline'] = (mode, 512, 512, HEADLINE[mode], 0)
    return out


def run_case(name, mode, Co, E, segs, flush, dev='cuda'):
    """The kernel's output [E, planes, Co] as a float32 numpy array."""
    import torch
    from se3_transformer_pytorch_b200 import ops
    F = 1 if mode == 1 else 2
    segs_k, parts, rowmax = [], [], np.zeros(E)
    for j, (Ci, nc, cp, cm, Kp) in enumerate(segs):
        key = f'zgemm/{name}/{j}'
        U = np.zeros((E, 64), np.float32)
        U[:, :Kp] = det_normal(key + '/U', (E, Kp))
        U[:, Kp - 1] = 1.0                             # the bias slot
        Fp = (det_normal(key + '/F', (Co * Ci * F, Kp)) / np.sqrt(Ci * Kp)).astype(np.float32)
        xp = det_normal(key + '/x', (E, Ci, nc)).astype(np.float32)
        rowmax = np.maximum(rowmax, np.abs(xp).max(axis=(1, 2)))
        tiles = (E + 127) // 128
        X = np.zeros((tiles * 128, Ci, nc), np.float32)
        X[:E] = xp                                     # kernel layout [tiles][Ci][ncomp][128], zero rows past E
        X = np.ascontiguousarray(X.reshape(tiles, 128, Ci, nc).transpose(0, 2, 3, 1)).reshape(-1)
        Ud, Xd = torch.from_numpy(U).to(dev), torch.from_numpy(X).to(dev)
        for kc in range(Kp // 16):
            segs_k.append((Ud[:, 16 * kc:], Xd, Ci, nc, cp, cm))
        parts.append((torch.from_numpy(Fp).to(dev), Ci))
    img, _ = ops.zgemm_image(parts, Co, mode)
    sx = torch.from_numpy(np.exp2(np.floor(9 - np.log2(np.maximum(rowmax, 1e-30)))).astype(np.float32)).to(dev)
    planes = min(mode, 2)
    out = torch.full((E, planes, Co), 7.0, device=dev)
    ops.zgemm(segs_k, img, sx, E, Co, mode, out, planes * Co, [0, Co], flush_stages=flush)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def sample_index(n):
    return [int(i) for i in np.linspace(0, n - 1, N_SAMPLES).round()]


def main(path=FIXTURE):
    res = {}
    for name, (mode, Co, E, segs, flush) in cases().items():
        a = run_case(name, mode, Co, E, segs, flush).reshape(-1)
        res[name] = {'sha256': digest(a), 'samples': [[i, float(a[i])] for i in sample_index(a.size)]}
        print(name, res[name]['sha256'][:16], flush=True)
    with open(path, 'w') as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', path, len(res), 'cases')


if __name__ == '__main__':
    main(*sys.argv[1:])
