"""Packed-batch fixtures (tests/golden/gen_golden_varlen.py): the real reference run once per cloud, outputs concatenated along
the node axis.  No reference import; fixtures only."""
import json
import os

import numpy as np

from helpers import GOLDEN, load_case, rel_err

VARLEN_CASES = ['varlen_cfg1', 'varlen_type1', 'varlen_edges_sparse', 'varlen_rotary_causal', 'varlen_pooled', 'varlen_z128']
PAIR_INPUTS = ('adj_mat', 'edges', 'neighbor_mask')


def varlen_params(name, seed=11):
    """The deterministic weights of a varlen fixture's model as {state_dict key: ndarray} (as helpers.det_params)."""
    from detfill import det_tensor
    with open(os.path.join(GOLDEN, 'state_keys_varlen.json')) as f:
        keys = json.load(f)[name]
    return {k: det_tensor(k, tuple(s), seed).astype(np.float32) for k, s in keys.items() if not k.endswith('inv_freq')}


def load_varlen(name):
    """(z, cfg, feats, coors, seqlens, pairs): feats [T, ...] or {'d': [T, C, 2d+1]}, pairs {name: list of per-cloud [n_c, n_c, ...]}."""
    z, cfg = load_case(name)
    seqlens = [int(n) for n in z['in/seqlens']]
    feats = z['in/feats'] if 'in/feats' in z else {d: z[f'in/feats/{d}'] for d in ('0', '1')}
    pairs = {}
    for key in PAIR_INPUTS:
        if f'in/{key}' in z:
            flat = z[f'in/{key}']
            pairs[key] = [flat[o:o + n * n].reshape(n, n, *flat.shape[1:]) for o, n in zip(z['in/pair_off'], seqlens)]
    return z, cfg, feats, z['in/coors'], seqlens, pairs


def varlen_outputs(z):
    return z['out'] if 'out' in z else {k[4:]: v for k, v in z.items() if k.startswith('out/')}


def cloud_slices(seqlens, pooled):
    """Rows of cloud c in a packed output: its nodes, or row c of a pooled output."""
    starts = np.cumsum([0] + list(seqlens[:-1]))
    return [slice(c, c + 1) if pooled else slice(s, s + n) for c, (s, n) in enumerate(zip(starts, seqlens))]


def per_cloud_errors(res, ref, seqlens, pooled):
    """Worst rel_err over the output degrees, for each cloud on its own (normalised by that cloud's output scale, so that a small
    cloud cannot hide behind a large one)."""
    res = res if isinstance(res, dict) else {'': res}
    ref = ref if isinstance(ref, dict) else {'': ref}
    assert set(res) == set(ref), (set(res), set(ref))
    errs = []
    for sl in cloud_slices(seqlens, pooled):
        errs.append(max(rel_err(np.asarray(res[d])[sl], ref[d][sl]) for d in ref))
    return errs
