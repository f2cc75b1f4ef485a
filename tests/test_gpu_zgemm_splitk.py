"""Split-K of the one-GEMM kernel (modes 1 and 3): every case of tests/golden/zgemm_hashes.json, run with k_split forced to 2, 3
and the launch's largest value (one split unit per CTA), reproduces the recorded output bit for bit; a split launch is
deterministic; and a k_split above the launch's units is refused."""
import json

import numpy as np
import pytest
import torch

from gen_zgemm_hashes import FIXTURE, cases, digest, run_case
from helpers import zgemm_split_units

CASES = cases()
with open(FIXTURE) as _f:
    EXPECTED = json.load(_f)


def _run(name, k_split):
    from se3_transformer_pytorch_b200 import ops
    orig = ops.zgemm
    used = []

    def forced(*a, **kw):
        kw['k_split'] = k_split(*a, **kw) if callable(k_split) else k_split
        used.append(kw['k_split'])
        return orig(*a, **kw)
    ops.zgemm = forced
    try:
        mode, Co, E, segs, flush = CASES[name]
        return run_case(name, mode, Co, E, segs, flush).reshape(-1), used
    finally:
        ops.zgemm = orig


def _units(segs, w_img, sx, E, Co, mode, out, out_edge_stride, comp_off, flush_stages=0, **_):
    return zgemm_split_units(segs, Co, mode, flush_stages)


def _need_sm90():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported('cuda', 128, 1):
        pytest.skip('needs sm_90')


@pytest.mark.gpu
@pytest.mark.parametrize('split', ['2', '3', 'max'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_split_output_is_bit_identical(name, split):
    _need_sm90()
    want = {'2': 2, '3': 3, 'max': None}[split]
    k = (lambda *a, **kw: min(want, _units(*a, **kw))) if want else _units
    a, used = _run(name, k)
    assert used, 'zgemm was not called'
    assert digest(a) == EXPECTED[name]['sha256'], f'{name} with k_split {used}: output differs from the unsplit kernel'


@pytest.mark.gpu
def test_split_is_deterministic():
    _need_sm90()
    name = 'm3_Co384_E300_f3'
    a, used = _run(name, 3)
    b, _ = _run(name, 3)
    assert used == [3] and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.gpu
def test_k_split_above_units_is_refused():
    _need_sm90()
    with pytest.raises(ValueError, match='k_split'):
        _run('m1_Co128_E129_f1048576', 2)          # mode 1 never drained: one unit


@pytest.mark.gpu
def test_small_grids_choose_a_split():
    """The automatic choice splits launches with fewer tiles than SMs and leaves a full grid alone."""
    _need_sm90()
    from se3_transformer_pytorch_b200 import ops
    sms = ops.sm_count('cuda')
    assert ops.zgemm_k_split(2, 100, sms) > 1
    assert ops.zgemm_k_split(sms, 100, sms) == 1 and ops.zgemm_k_split(4 * sms, 100, sms) == 1
    before = ops.SPLIT_LAUNCHES
    mode, Co, E, segs, flush = CASES['m1_Co128_E129_f0']
    run_case('m1_Co128_E129_f0', mode, Co, E, segs, flush)
    assert ops.SPLIT_LAUNCHES == before + 1
