"""The |m| > 0 GEMM (mode 3, Gauss form) at widths and drain periods the headline shapes do not reach: segments whose weight
sets come in blocks of L = 8, 4, 2 and 1 stages (C_in / 4 = 24, 4, 10, 3 channel groups) in one launch, several output tile
counts, a partly filled last edge tile and drain periods that do and do not divide L.  Each case is checked against float64
and against mode 2 (four real products per complex one, default drain) on the same weights and inputs."""
import pytest

from helpers import rel_err, run_zgemm

pytestmark = pytest.mark.gpu
DEV = 'cuda'

# (C_in, ncomp, cplus, cminus, Kp): L = 8, 4 (a K = 32 pair: two sub-segments), 2, 1
MIXED_L = [(96, 3, 2, 0, 16), (16, 5, 3, 1, 32), (40, 7, 4, 2, 16), (12, 3, 2, 0, 16)]


@pytest.mark.parametrize('Co,E', [(128, 300), (384, 129), (512, 200)])
@pytest.mark.parametrize('flush', [1, 3, 5, 1 << 20])
def test_gauss_blocks_match_fp64_and_mode2(Co, E, flush):
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, Co, 1):
        pytest.skip('needs sm_90')
    out3, ref = run_zgemm(3, Co, E, MIXED_L, flush=flush, seed=Co + flush % 97)
    # mode 2 on the same weights and inputs (same seed), with its default drain: it has no set ends, so without drains its
    # own truncation error would dominate the comparison
    out2, _ = run_zgemm(2, Co, E, MIXED_L, flush=0, seed=Co + flush % 97)
    out3, out2 = out3.cpu().numpy(), out2.cpu().numpy()
    err = rel_err(out3, ref.cpu().numpy())
    assert err < 6e-6, f'mode 3 vs float64: {err:.3e}'
    err2 = rel_err(out3, out2)
    assert err2 < 6e-6, f'mode 3 vs mode 2: {err2:.3e}'
