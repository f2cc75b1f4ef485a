"""Packed-batch fixtures for SE3Transformer.forward_packed, which has no reference counterpart.  The real reference runs once per
cloud (b = 1, mask of ones, the detfill weights of gen_golden.py) and its outputs are concatenated along the node axis.  Needs a
checkout of the reference on the Python path, as gen_golden.py does:

    PYTHONPATH=<reference checkout> CACHE_PATH=/tmp/se3_cache python tests/golden/gen_golden_varlen.py

Outputs
  tests/golden/model_varlen_<case>.npz     packed inputs ([T, ...] node inputs, per-cloud [n_c, n_c] pair inputs flattened end to
                                           end with cloud c from in/pair_off[c]) and the concatenated reference outputs
  tests/golden/state_keys_varlen.json      state_dict key/shape lists of these models
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gen_golden import HERE, ref_mod, band_adj, to_np, write_split  # noqa: E402
from detfill import fill_state_dict, det_inputs, det_uniform  # noqa: E402

# max_sparse_neighbors >= the bonded count throughout, so the reference's random sub-sampling of bonded neighbours never runs
VARLEN_CASES = [
    dict(name='varlen_cfg1', ctor=dict(dim=64, depth=2, num_degrees=2, num_neighbors=8), lens=[32, 5, 17, 2]),
    dict(name='varlen_type1', ctor=dict(dim=16, dim_in=(16, 4), heads=2, dim_head=8, depth=1, input_degrees=2, num_degrees=2,
                                        output_degrees=2, num_neighbors=6), lens=[12, 3, 9], type1_in=True, fwd=dict(return_type=1)),
    # 2-hop band adjacencies of widths 1, 2, 3: 4, 8, 12 bonded neighbours, so k_c = 7, 8, 11
    dict(name='varlen_edges_sparse', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_edge_tokens=4, edge_dim=8,
                                               attend_sparse_neighbors=True, num_adj_degrees=2, adj_dim=4, num_neighbors=3,
                                               max_sparse_neighbors=16), lens=[16, 9, 12], edges='tokens', adj=[1, 2, 3]),
    dict(name='varlen_rotary_causal', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, rotary_position=True,
                                                rotary_rel_dist=True, causal=True), lens=[10, 3, 14]),
    dict(name='varlen_pooled', ctor=dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, num_neighbors=4,
                                         num_conv_layers=1, norm_out=True, reduce_dim_out=True), lens=[8, 13, 4], fwd=dict(return_pooled=True)),
    dict(name='varlen_z128', ctor=dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=3, output_degrees=2, num_neighbors=6,
                                       valid_radius=10), lens=[20, 9, 14]),
]


def run_varlen_case(case):
    """Writes model_<name>.npz; returns the model's state_dict key/shape list."""
    name, ctor, lens = case['name'], case['ctor'], case['lens']
    T = sum(lens)
    starts = np.cumsum([0] + lens[:-1])
    torch.manual_seed(0)
    model = ref_mod.SE3Transformer(**ctor)
    fill_state_dict(model, seed=11)
    model.eval()
    dim_in = ctor.get('dim_in', ctor['dim'])
    inp = {'seqlens': np.array(lens, dtype=np.int64), 'pair_off': np.cumsum([0] + [n * n for n in lens[:-1]]).astype(np.int64)}
    if case.get('type1_in'):
        inp['feats/0'] = det_inputs(name + '/f0', (T, dim_in[0], 1), 1)
        inp['feats/1'] = det_inputs(name + '/f1', (T, dim_in[1], 3), 1)
    else:
        inp['feats'] = det_inputs(name + '/feats', (T, dim_in), 1)
    inp['coors'] = det_inputs(name + '/coors', (T, 3), 2)
    pair = {}
    if case.get('adj') is not None:
        pair['adj_mat'] = [band_adj(n, w) for n, w in zip(lens, case['adj'])]
    if case.get('edges') == 'tokens':
        pair['edges'] = [(det_uniform(f'edge/{name}/{c}', n * n, 1) * ctor['num_edge_tokens']).astype(np.int64).reshape(n, n)
                         for c, n in enumerate(lens)]
    for k, per_cloud in pair.items():
        inp[k] = np.concatenate([t.reshape(-1) for t in per_cloud])
    outs = []
    for c, (s, n) in enumerate(zip(starts, lens)):
        if 'feats' in inp:
            feats = torch.from_numpy(inp['feats'][s:s + n][None])
        else:
            feats = {d: torch.from_numpy(inp[f'feats/{d}'][s:s + n][None]) for d in ('0', '1')}
        kwargs = dict(case.get('fwd', {}))
        if 'adj_mat' in pair:
            kwargs['adj_mat'] = torch.from_numpy(pair['adj_mat'][c])
        if 'edges' in pair:
            kwargs['edges'] = torch.from_numpy(pair['edges'][c][None])
        with torch.no_grad():
            res = model(feats, torch.from_numpy(inp['coors'][s:s + n][None]), torch.ones(1, n, dtype=torch.bool), **kwargs)
        outs.append({'': res} if torch.is_tensor(res) else res)
    pooled = case.get('fwd', {}).get('return_pooled', False)
    out = {'in/' + k: v for k, v in inp.items()}
    for d in outs[0]:
        key = 'out' if d == '' else f'out/{d}'
        out[key] = np.concatenate([to_np(o[d]) if pooled else to_np(o[d])[0] for o in outs], 0)
    out['config'] = np.array(json.dumps(dict(ctor={k: (list(v) if isinstance(v, tuple) else v) for k, v in ctor.items()},
                                             fwd=case.get('fwd', {}), seqlens=lens)))
    path = os.path.join(HERE, f'model_{name}.npz')
    write_split(path, out)
    print('wrote', path, 'size', os.path.getsize(path))
    return {k: list(v.shape) for k, v in model.state_dict().items()}


if __name__ == '__main__':
    keys = {case['name']: run_varlen_case(case) for case in VARLEN_CASES}
    with open(os.path.join(HERE, 'state_keys_varlen.json'), 'w') as f:
        json.dump(keys, f, indent=0, sort_keys=True)
