"""The one-GEMM kernel (modes 1 and 3) gives bit-identical outputs to the recorded ones (tests/golden/zgemm_hashes.json,
written by tests/golden/gen_zgemm_hashes.py): mixed weight-set blocks L = 8/4/2/1, drain periods that do and do not divide
L, partly filled last edge tiles, several output tile counts and one headline-width launch.  The bench model amplifies a
one-ulp change of this kernel into a visible change of its outputs, so any change to its pipeline must keep every fp32
operation and its order."""
import json

import numpy as np
import pytest

from gen_zgemm_hashes import FIXTURE, cases, digest, run_case

CASES = cases()
with open(FIXTURE) as _f:
    EXPECTED = json.load(_f)


def test_fixture_covers_every_case():
    assert sorted(EXPECTED) == sorted(CASES)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_zgemm_output_is_bit_identical(name):
    from se3_transformer_pytorch_b200 import ops
    mode, Co, E, segs, flush = CASES[name]
    if not ops.tc_supported('cuda', Co, 1):
        pytest.skip('needs sm_90')
    a = run_case(name, mode, Co, E, segs, flush).reshape(-1)
    exp = EXPECTED[name]
    if digest(a) != exp['sha256']:
        idx = np.array([i for i, _ in exp['samples']])
        want = np.array([v for _, v in exp['samples']], np.float32)
        rel = np.abs(a[idx] - want) / np.maximum(np.abs(want), 1e-30)
        pytest.fail(f'{name}: output differs from the recorded one; at {len(idx)} sampled entries max rel diff '
                    f'{rel.max():.3e}, {int((a[idx] != want).sum())} differ')
