"""Dispatch trace of model.conv_forward: which kernel runs, in what order, with which arguments and accumulate flags.

Every CUDA op is replaced by the float64 emulation of tests/dispatch_emulation.py, which records one entry per launch.  For each
case below the trace and fingerprints of the emulated outputs go to tests/golden/dispatch_trace.json; test_dispatch_trace_host.py
checks that conv_forward still produces them exactly.  Runs on CPU:

    python tests/golden/gen_dispatch_trace.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

from dispatch_emulation import Emulation, fingerprint, installed  # noqa: E402

OUT = os.path.join(HERE, 'dispatch_trace.json')

# the switches conv_forward reads; every case starts from none of them set
SWITCHES = ('SE3B200_NO_LOWRANK', 'SE3B200_NO_ALIGNED', 'SE3B200_NO_ZGEMM', 'SE3B200_NO_UTABLE', 'SE3B200_NO_INPUT_SIDE',
            'SE3B200_Z_MODE2', 'SE3B200_FORCE_SIMT', 'SE3B200_LOWRANK_TOL', 'SE3B200_NO_LINEAR_TC')

# C: channels of every degree (the one-GEMM kernel takes multiples of 128).  chunk: the workspace holds two edge tiles of the
# R-first T blocks ('t') or of the rotated gather ('z'), so the 3 tiles of a case run in two edge chunks.
CASES = {
    'zgemm': dict(C=128, chunk='z', deferred=True),
    'aligned': dict(C=32, chunk='t'),
    'global': dict(C=32, chunk='t', env={'SE3B200_NO_ALIGNED': '1'}),
    'global_pooled': dict(C=32, chunk='t', env={'SE3B200_NO_ALIGNED': '1'}, pool=True),
    'zgemm_pooled': dict(C=128, chunk='z', pool=True),
    'zgemm_keep_aligned_kv': dict(C=128, chunk='z', convs=2, keep_aligned=True),
    'ineligible_pair': dict(C=32, chunk='t', ineligible=(2, 2)),
    'plan_miss_direct': dict(C=32, chunk='t', plan_at=0.05, capturing=True),
    'no_lowrank': dict(C=32, chunk='t', env={'SE3B200_NO_LOWRANK': '1'}),
    'force_simt': dict(C=32, chunk='t', env={'SE3B200_FORCE_SIMT': '1'}),
    'free_master': dict(C=128, chunk='z', free_master=True),
}


def _geometry(b, n, k, L, C):
    coors = torch.randn(b, n, 3)
    idx = torch.stack([torch.randperm(n - 1)[:k] for _ in range(b * n)]).reshape(b, n, k)
    idx = idx + (idx >= torch.arange(n).view(1, n, 1)).long()                        # neighbours != self
    rel_pos = (coors[0][:, None, :] - coors[0][idx[0]]).reshape(b, n, k, 3)           # x_i - x_j
    nmask = torch.rand(b, n, k) < 0.9
    inp = {str(d): torch.randn(b, n, C, 2 * d + 1) for d in range(L + 1)}
    return idx, nmask, rel_pos, inp


def run_case(name):
    """Run case `name` under the emulation -> {'trace': [...], 'outputs': [{degree: fingerprint} per conv], 'deferred': int}."""
    from oracle import se3_oracle as O
    from se3_transformer_pytorch_b200 import model as M, ops
    spec = CASES[name]
    C, L, b, n, k = spec['C'], 2, 1, 40, 8
    torch.manual_seed(0)
    fiber = M.Fiber([(d, C) for d in range(L + 1)])
    pool = spec.get('pool', False)
    convs = [M.ConvSE3(fiber, fiber, edge_dim=0, pool=pool, self_interaction=pool) for _ in range(spec.get('convs', 1))]
    idx, nmask, rel_pos, inp = _geometry(b, n, k, L, C)
    rel_dist = rel_pos.norm(dim=-1)
    E = b * n * k
    Bo = O.get_basis(rel_pos.reshape(E, 3).double().numpy(), L)
    bpairs = {(di, do): torch.from_numpy(np.asarray(Bo[f'{di},{do}'])).float().reshape(-1) for di in range(L + 1) for do in range(L + 1)}
    if spec['chunk'] == 'z':
        ws = 2 * sum(C * (2 * d + 1) for d in range(L + 1)) * ops.TILE_E * 4
    else:
        ws = 2 * max(ops.t_numel(1, C, 2 * min(di, do) + 1, 2 * do + 1) * 4 for di in range(L + 1) for do in range(L + 1))

    emu = Emulation()
    env = dict({s: None for s in SWITCHES}, SE3B200_HOST_FRAMES='1', SE3B200_LOWRANK_MIN_EDGES='1', **spec.get('env', {}))
    patches = dict(emu.patches(), basis_pairs=lambda flat, plan, E_: bpairs)
    model_patches = {'T_WORKSPACE_BYTES': ws}
    if 'ineligible' in spec:
        bad = spec['ineligible']
        orig = M.ConvSE3.tc_eligible
        model_patches_cls = {'tc_eligible': lambda self, di, do: (di, do) != bad and orig(self, di, do)}
    else:
        model_patches_cls = {}
    capturing = spec.get('capturing', False)
    saved_env = {key: os.environ.get(key) for key in env}
    try:
        for key, v in env.items():
            if v is None:
                os.environ.pop(key, None)
            else:
                os.environ[key] = v
        with installed(patches, ops), installed(model_patches, M), installed(model_patches_cls, M.ConvSE3), \
                installed({'is_current_stream_capturing': lambda: capturing}, torch.cuda), torch.no_grad():
            if 'plan_at' in spec:
                for conv in convs:
                    conv.lowrank_plan(spec['plan_at'])
            if spec.get('free_master'):
                for conv in convs:
                    conv.pack_weights(free_master=True, max_distance=1.25 * float(rel_dist.max()))
            geom = M.Geometry(rel_pos, L)
            if spec.get('deferred'):
                geom.deferred = []
            outs = M.conv_forward(convs, inp, (idx, nmask, None), rel_dist, (torch.zeros(0), None, geom),
                                  keep_aligned=spec.get('keep_aligned', False))
    finally:
        for key, v in saved_env.items():
            if v is None:
                os.environ.pop(key, None)
            else:
                os.environ[key] = v
    prints = [{d: fingerprint(o.t if isinstance(o, M.AlignedKV) else o) for d, o in out.items()} for out in outs]
    return dict(trace=emu.trace, outputs=prints, deferred=len(geom.deferred or []))


def main():
    res = {name: run_case(name) for name in CASES}
    with open(OUT, 'w') as f:
        json.dump(res, f, indent=0, sort_keys=True)
        f.write('\n')
    for name, r in res.items():
        print(f'{name}: {len(r["trace"])} launches')


if __name__ == '__main__':
    main()
