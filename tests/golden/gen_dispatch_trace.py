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

# C: channels of every degree (the one-GEMM kernel takes multiples of 128).  chunk: the workspace holds two edge tiles of the
# R-first T blocks ('t') or of the rotated gather ('z'), so the 3 tiles of a case run in two edge chunks.
CASES = {
    'zgemm': dict(C=128, chunk='z', deferred=True),
    'aligned': dict(C=32, chunk='t'),
    'global': dict(C=32, chunk='t', switches=dict(no_aligned=True)),
    'global_pooled': dict(C=32, chunk='t', switches=dict(no_aligned=True), pool=True),
    'zgemm_pooled': dict(C=128, chunk='z', pool=True),
    'zgemm_keep_aligned_kv': dict(C=128, chunk='z', convs=2, keep_aligned=True),
    'ineligible_pair': dict(C=32, chunk='t', ineligible=(2, 2)),
    'plan_miss_direct': dict(C=32, chunk='t', plan_at=0.05, capturing=True),
    'no_lowrank': dict(C=32, chunk='t', switches=dict(no_lowrank=True)),
    'force_simt': dict(C=32, chunk='t', switches=dict(force_simt=True)),
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


class Case:
    """The modules, graph and inputs of case `name`; forward() runs conv_forward on them under the emulation."""

    def __init__(self, name):
        from oracle import se3_oracle as O
        from se3_transformer_pytorch_b200 import model as M, ops
        self.spec = spec = CASES[name]
        C, L, b, n, k = spec['C'], 2, 1, 40, 8
        self.L = L
        torch.manual_seed(0)
        fiber = M.Fiber([(d, C) for d in range(L + 1)])
        pool = spec.get('pool', False)
        self.convs = [M.ConvSE3(fiber, fiber, edge_dim=0, pool=pool, self_interaction=pool) for _ in range(spec.get('convs', 1))]
        self.idx, self.nmask, self.rel_pos, self.inp = _geometry(b, n, k, L, C)
        self.rel_dist = self.rel_pos.norm(dim=-1)
        E = b * n * k
        Bo = O.get_basis(self.rel_pos.reshape(E, 3).double().numpy(), L)
        self.bpairs = {(di, do): torch.from_numpy(np.asarray(Bo[f'{di},{do}'])).float().reshape(-1)
                       for di in range(L + 1) for do in range(L + 1)}
        if spec['chunk'] == 'z':
            self.ws = 2 * sum(C * (2 * d + 1) for d in range(L + 1)) * ops.TILE_E * 4
        else:
            self.ws = 2 * max(ops.t_numel(1, C, 2 * min(di, do) + 1, 2 * do + 1) * 4 for di in range(L + 1) for do in range(L + 1))
        self.prepared = False

    def switches(self, **flips):
        """Every switch at its default except the case's own and `flips`, with the float64 host frames and the low-rank path for
        any edge count."""
        from se3_transformer_pytorch_b200 import switches
        return dict(dict.fromkeys(switches.FIELDS), host_frames=True, lowrank_min_edges=1, **dict(self.spec.get('switches', {}), **flips))

    def forward(self, emu, **flips):
        """One conv_forward with every op emulated by `emu`, under self.switches(**flips) -> (fingerprints of the outputs per
        conv, number of deferred plan checks).  The first call first builds what the case asks for (a plan, packed weights)."""
        from se3_transformer_pytorch_b200 import model as M, ops, switches
        spec = self.spec
        patches = dict(emu.patches(), basis_pairs=lambda flat, plan, E_: self.bpairs)
        model_patches = {'T_WORKSPACE_BYTES': self.ws}
        if 'ineligible' in spec:
            bad = spec['ineligible']
            orig = M.ConvSE3.tc_eligible
            model_patches_cls = {'tc_eligible': lambda conv, di, do: (di, do) != bad and orig(conv, di, do)}
        else:
            model_patches_cls = {}
        capturing = spec.get('capturing', False)
        with switches.override(**self.switches(**flips)), installed(patches, ops), installed(model_patches, M), \
                installed(model_patches_cls, M.ConvSE3), installed({'is_current_stream_capturing': lambda: capturing}, torch.cuda), \
                torch.no_grad():
            if not self.prepared:
                self.prepared = True
                if 'plan_at' in spec:
                    for conv in self.convs:
                        conv.lowrank_plan(spec['plan_at'])
                if spec.get('free_master'):
                    for conv in self.convs:
                        conv.pack_weights(free_master=True, max_distance=1.25 * float(self.rel_dist.max()))
            geom = M.Geometry(self.rel_pos, self.L)
            if spec.get('deferred'):
                geom.deferred = []
            outs = M.conv_forward(self.convs, self.inp, (self.idx, self.nmask, None), self.rel_dist, (torch.zeros(0), None, geom),
                                  keep_aligned=spec.get('keep_aligned', False))
        prints = [{d: fingerprint(o.t if isinstance(o, M.AlignedKV) else o) for d, o in out.items()} for out in outs]
        return prints, len(geom.deferred or [])


def run_case(name):
    """Run case `name` under the emulation -> {'trace': [...], 'outputs': [{degree: fingerprint} per conv], 'deferred': int}."""
    emu = Emulation()
    prints, deferred = Case(name).forward(emu)
    return dict(trace=emu.trace, outputs=prints, deferred=deferred)


def main():
    res = {name: run_case(name) for name in CASES}
    with open(OUT, 'w') as f:
        json.dump(res, f, indent=0, sort_keys=True)
        f.write('\n')
    for name, r in res.items():
        print(f'{name}: {len(r["trace"])} launches')


if __name__ == '__main__':
    main()
