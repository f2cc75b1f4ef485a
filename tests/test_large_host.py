"""Clouds of more than 4097 points without a GPU: the numpy oracle against the reference-generated `large` fixtures
(tests/golden/gen_golden_large.py), so that the GPU tests can rely on the oracle at these sizes."""
import json
import os

import numpy as np
import pytest

from helpers import GOLDEN, load_case, rel_err, case_inputs, case_outputs, assert_graph_equal
from oracle import se3_oracle as O

LARGE_CASES = ['large_type1', 'large_bonded_b2']


def large_params(name, seed=11):
    from detfill import det_tensor
    with open(os.path.join(GOLDEN, 'state_keys_large.json')) as f:
        keys = json.load(f)[name]
    return {k: det_tensor(k, tuple(s), seed).astype(np.float32) for k, s in keys.items() if not k.endswith('inv_freq')}


@pytest.mark.parametrize('name', LARGE_CASES)
def test_oracle_matches_large_fixture(name):
    z, cfg = load_case(name)
    assert cfg['n'] > 4097
    feats, coors, mask, extra = case_inputs(z)
    res, inter = O.se3_transformer_forward(large_params(name), cfg['ctor'], feats, coors, mask, return_intermediates=True,
                                           **extra, **cfg['fwd'])
    g = inter['graph']
    assert_graph_equal(g['idx'], g['mask'], g['rel_dist'], z['cap/graph/neighbor_indices'], z['cap/graph/neighbor_mask'],
                       z['cap/graph/rel_dist'])
    assert rel_err(res, case_outputs(z)) < 1e-4
