"""Fixtures for clouds of more than 4097 points, where the neighbour search walks its rows in tiles of 4096 columns.  The real
reference runs on the CPU (dense [b, n, n-1] temporaries: a few GB of host memory per case), with the detfill weights and the
capture hooks of gen_golden.py.  Needs a checkout of the reference on the Python path, as gen_golden.py does:

    PYTHONPATH=<reference checkout> CACHE_PATH=/tmp/se3_cache python tests/golden/gen_golden_large.py

Outputs
  tests/golden/model_large_<case>.npz      inputs, outputs and the captured neighbour graph (split as gen_golden.write_split does)
  tests/golden/state_keys_large.json       state_dict key/shape lists of these models
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from gen_golden import HERE, run_case, write_split  # noqa: E402

KEEP_CAPTURES = ('cap/graph/neighbor_indices', 'cap/graph/neighbor_mask', 'cap/graph/rel_dist')

# max_sparse_neighbors >= the bonded count, so the reference's random sub-sampling of bonded neighbours never runs
LARGE_CASES = [
    dict(name='large_type1', ctor=dict(dim=16, dim_in=4, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2,
                                       reduce_dim_out=True, num_neighbors=8), b=1, n=4500, fwd=dict(return_type=1)),
    # band adjacency of width 2: 4 bonded neighbours, k = 6 + 4; the last 3 / 6 nodes of the two clouds are masked
    dict(name='large_bonded_b2', ctor=dict(dim=16, dim_in=4, heads=2, dim_head=8, depth=1, num_degrees=2, reduce_dim_out=True,
                                           num_neighbors=6, attend_sparse_neighbors=True, max_sparse_neighbors=8),
         b=2, n=4400, adj=2, ragged=True),
]


def run_large_case(case):
    """run_case, keeping of the captured intermediates only the graph (the rest would add megabytes at these sizes)."""
    keys = run_case(case)
    path = os.path.join(HERE, f"model_{case['name']}.npz")
    arrays = {}
    for f in sorted(f for f in os.listdir(HERE) if f.startswith(f"model_{case['name']}.")):
        arrays.update(np.load(os.path.join(HERE, f)))
    write_split(path, {k: v for k, v in arrays.items() if not k.startswith('cap/') or k in KEEP_CAPTURES})
    return keys


if __name__ == '__main__':
    keys = {case['name']: run_large_case(case) for case in LARGE_CASES}
    with open(os.path.join(HERE, 'state_keys_large.json'), 'w') as f:
        json.dump(keys, f, indent=0, sort_keys=True)
