"""Direct float64 tests of the kernels that the aligned and production routes launch around their GEMMs -- the rotation back
to the global frame, the component-major basis fold, the T blocks of caller-supplied edge blocks, the power-of-two scales --
and of every production kernel at the launch sizes of the decoders (a handful of edges, one node).

Each kernel is called through ops and compared with the float64 statement of its contract in dispatch_emulation.Emulation (the
statement the CPU dispatch tests run against) or in helpers.  Tolerances are elementwise, relative to the same operation applied
to the absolute values of the operands (what fp32 rounding error scales with), so a sign or index slip cannot hide in a
cancellation or behind a larger row.  Layout padding, sentinel rows and the bytes past a launch's output are checked bit for bit."""
import math

import numpy as np
import pytest
import torch

from dispatch_emulation import Emulation, tile_edges
from helpers import attention_reference, decode_T, rel_err, zgemm_problem, zgemm_split_units

pytestmark = pytest.mark.gpu
DEV = 'cuda'

SENTINEL = 7.0
CO = [1, 3, 7, 32, 96, 128, 300]   # 256-thread blocks of (edge, channel) threads start mid-edge unless Co divides 256
EDGES = [1, 37, 201]               # odd: E * Co is a multiple of 256 for none of CO, so every last block is partly filled
STAGING_LIMIT = 48 * 1024          # shared memory the fold / rotate-back kernels may stage a block's per-edge matrices in


def _staging_bytes(Co, nb):
    """Shared memory of a fold / rotate-back launch: the nb floats per edge of every edge a 256-thread block can touch."""
    return (256 // Co + 2) * nb * 4


def _assert_close(got, ref, bound, tol, what=''):
    """|got - ref| <= tol * bound elementwise; got on any device, ref and bound float64 on the host."""
    err = (got.detach().cpu().double() - ref).abs()
    bad = err > tol * bound
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} entries off, worst {float((err / bound.clamp(min=1e-300)).max()):.3e} of the bound'


def _sentinel_buffer(E, shape, pad=3):
    """(buffer of E + 2 pad rows filled with SENTINEL, the view of its rows pad .. pad + E) on the device."""
    buf = torch.full((E + 2 * pad, *shape), SENTINEL, device=DEV)
    return buf, buf[pad:pad + E]


def _assert_sentinel_kept(buf, E, pad=3):
    assert bool((buf[:pad] == SENTINEL).all()) and bool((buf[pad + E:] == SENTINEL).all()), 'rows outside the output were written'


# ------------------------------------------------------------------ rotate_back: out[e, o, :] = D_lo(e) out'[e, o, :]
def _part_patterns(lo):
    full = set(range(lo + 1))
    yield 'all', full
    yield 'no m=0', full - {0}
    for m in range(1, lo + 1):
        yield f'no |m|={m}', full - {m}
    yield 'none', set()


def _rotate_back_case(lo, Co, E, present, g):
    from se3_transformer_pytorch_b200 import ops
    P = 2 * lo + 1
    off = 5                                          # D at an edge offset inside the frames of a larger graph, as _aligned_forward slices them
    Dall = torch.randn(off + E + 4, P, P, generator=g)
    D = Dall[off:off + E]
    parts = [torch.randn(E, Co, generator=g) if 0 in present else None]
    parts += [torch.randn(E, Co, 2, generator=g) if m in present else None for m in range(1, lo + 1)]
    buf, out = _sentinel_buffer(E, (Co, P))
    ops.rotate_back([None if p is None else p.to(DEV) for p in parts], Dall.to(DEV)[off:off + E].reshape(-1), E, Co, lo, out)
    torch.cuda.synchronize()
    em = Emulation()
    ref = torch.empty(E, Co, P, dtype=torch.float64)
    em.rotate_back(parts, D.reshape(-1), E, Co, lo, ref)
    bound = torch.empty(E, Co, P, dtype=torch.float64)
    em.rotate_back([None if p is None else p.abs() for p in parts], D.abs().reshape(-1), E, Co, lo, bound)
    return buf, out, ref, bound


@pytest.mark.parametrize('Co', CO)
@pytest.mark.parametrize('lo', [1, 2, 3])
def test_rotate_back_matches_fp64(lo, Co):
    """Every pattern of present / missing |m| parts, with D a slice at an edge offset and out a slice of a sentinel buffer; no
    parts at all give exact zeros.  A Co whose staging buffer exceeds 48 KiB is refused."""
    g = torch.Generator().manual_seed(100 * lo + Co)
    if _staging_bytes(Co, (2 * lo + 1) ** 2) > STAGING_LIMIT:
        with pytest.raises(RuntimeError, match='staging buffer'):
            _rotate_back_case(lo, Co, 37, set(range(lo + 1)), g)
        return
    for E in EDGES:
        for name, present in _part_patterns(lo):
            buf, out, ref, bound = _rotate_back_case(lo, Co, E, present, g)
            _assert_close(out, ref, bound, 2e-6, f'E={E} parts {name}')
            if not present:
                assert bool((out == 0).all())
            _assert_sentinel_kept(buf, E)


def test_rotate_back_refusals_leave_out_untouched():
    """Co = 1 at degree 3 needs 258 staged 7x7 matrices (> 48 KiB); a part on the host is refused before any launch."""
    from se3_transformer_pytorch_b200 import ops
    E, Co, lo = 37, 1, 3
    D = torch.randn(E * 49, device=DEV)
    buf, out = _sentinel_buffer(E, (Co, 7))
    with pytest.raises(RuntimeError, match='staging buffer'):
        ops.rotate_back([torch.randn(E, Co, device=DEV)], D, E, Co, lo, out)
    buf1, out1 = _sentinel_buffer(E, (2, 3))
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.rotate_back([torch.randn(E, 2)], torch.randn(E * 9, device=DEV), E, 2, 1, out1)
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL).all()) and bool((buf1 == SENTINEL).all())


# ------------------------------------------------------------------ fold_basis(component_major=True)
def _fold_case(P, Q, F, Co, E, basis, accumulate, g):
    """One component-major fold (S [F, E, Q, Co]) into a slice of a sentinel buffer, checked against float64 and against the
    row-major kernel on the transposed S (the same FMAs in the same order: only the load address differs)."""
    from se3_transformer_pytorch_b200 import ops
    S = torch.randn(F, E, Q, Co, generator=g)
    out0 = torch.randn(E, Co, P, generator=g)
    buf, out = _sentinel_buffer(E, (Co, P))
    out.copy_(out0)
    basis_d, S_d = basis.to(DEV), S.to(DEV)
    if _staging_bytes(Co, P * Q * F) > STAGING_LIMIT:
        with pytest.raises(RuntimeError, match='staging buffer'):
            ops.fold_basis(S_d, basis_d, E, Co, P, Q, F, out, accumulate, component_major=True)
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), out0)
        return
    ops.fold_basis(S_d, basis_d, E, Co, P, Q, F, out, accumulate, component_major=True)
    buf_rm, out_rm = _sentinel_buffer(E, (Co, P))
    out_rm.copy_(out0)
    ops.fold_basis(S_d.transpose(-1, -2).contiguous(), basis_d, E, Co, P, Q, F, out_rm, accumulate)
    torch.cuda.synchronize()
    em = Emulation()
    ref, bound = out0.double().clone(), out0.double().abs()
    em.fold_basis(S, basis, E, Co, P, Q, F, ref, accumulate, component_major=True)
    em.fold_basis(S.abs(), basis.abs(), E, Co, P, Q, F, bound, accumulate, component_major=True)
    _assert_close(out, ref, bound, 2e-6, f'P={P} Q={Q} F={F} E={E} accumulate={accumulate}')
    assert torch.equal(out, out_rm), 'component-major and row-major folds differ'
    _assert_sentinel_kept(buf, E)


@pytest.mark.parametrize('Co', CO)
@pytest.mark.parametrize('l', [1, 2, 3])
def test_fold_basis_cm_rotates_back_with_wigner_frames(l, Co):
    """The production shapes (P = Q = 2l+1, F = 1, basis = the real Wigner matrices of ops.frames): the rotate-back of
    _production_forward and Geometry.to_global."""
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(10 * l + Co)
    P = 2 * l + 1
    for E in EDGES:
        D = ops.frames(torch.randn(E, 3, generator=g).to(DEV), 3)[l]
        _fold_case(P, P, 1, Co, E, D.reshape(-1).cpu(), False, g)


@pytest.mark.parametrize('Co', CO)
@pytest.mark.parametrize('P,Q,F', [(2, 3, 2), (3, 3, 3), (3, 7, 3), (5, 3, 3), (6, 4, 2), (7, 5, 5), (7, 7, 7)])
def test_fold_basis_cm_general_shapes(P, Q, F, Co):
    g = torch.Generator().manual_seed(P * 100 + Q * 10 + F + Co)
    for E in EDGES:
        for accumulate in (False, True):
            _fold_case(P, Q, F, Co, E, torch.randn(E * P * Q * F, generator=g), accumulate, g)


@pytest.mark.parametrize('lo', [1, 2, 3])
def test_geometry_to_global(lo):
    """Geometry.to_global materialises an AlignedKV in the global frame: out[e, c, :] = D_lo(e) t[e, :, c] with the frames the
    Geometry built, in float64."""
    from se3_transformer_pytorch_b200.model import AlignedKV, Geometry
    g = torch.Generator().manual_seed(lo)
    b, n, k, C, P = 2, 5, 7, 24, 2 * lo + 1
    geom = Geometry(torch.randn(b, n, k, 3, generator=g).to(DEV), 3)
    t = torch.randn(b, n, k, P, C, generator=g)
    got = geom.to_global(AlignedKV(t.to(DEV), lo))
    assert got.shape == (b, n, k, C, P)
    D = geom.frames().D[lo].cpu().double()
    ref = torch.einsum('epn,enc->ecp', D, t.double().reshape(-1, P, C))
    bound = torch.einsum('epn,enc->ecp', D.abs(), t.double().abs().reshape(-1, P, C))
    _assert_close(got.reshape(-1, C, P), ref, bound, 2e-6)


# ------------------------------------------------------------------ tbuild_blocks as the aligned route uses it
TB_SHAPES = [(1, 1, Q) for Q in (1, 3, 5, 7, 9, 11)] + [(2, 2, Q) for Q in (3, 5, 7, 9, 11)]   # Q = 9, 11: the generic kernel


@pytest.mark.parametrize('Ci', [1, 3, 17, 33, 64])
@pytest.mark.parametrize('P,F,Q', TB_SHAPES)
def test_tbuild_blocks_matches_fp64(P, F, Q, Ci):
    """T of the edge-aligned blocks (EdgeFrames.block: m = 0 -> (P, F) = (1, 1), |m| > 0 -> (2, 2)) and of random blocks, over
    tile windows at the start, in the middle (a partial tile_count) and at the partly filled last tile, into a reused buffer
    pre-filled with NaN: every slot of the window's tiles is written, the layout padding (edges past E, if-slots past Ci F,
    components past P) is exactly 0, and nothing past t_numel changes.  Ci = 33 and 64 run as several channel slabs."""
    from se3_transformer_pytorch_b200 import aligned, ops
    g = torch.Generator().manual_seed(1000 * P + 10 * Q + Ci)
    b, n, k = 2, 23, 9                                   # E = 414: four edge tiles, the last one holding 30 edges
    E = b * n * k
    n_tiles = (E + ops.TILE_E - 1) // ops.TILE_E
    x = torch.randn(b, n, Ci, Q, generator=g)
    idx = torch.randint(0, n, (b, n, k), generator=g)
    blocks = {'random': torch.randn(E * P * Q * F, generator=g)}
    di = (Q - 1) // 2
    if di <= 3:
        frames = aligned.EdgeFrames(torch.randn(E, 3, generator=g), 3)
        for m in ([0] if P == 1 else range(1, di + 1)):
            blocks[f'frames m={m}'] = frames.block(di, m)
    x_d, idx_d = x.to(DEV), idx.to(DEV)
    buf = torch.empty(ops.t_numel(n_tiles, Ci, F, P) + 257, device=DEV)
    em = Emulation()
    for name, blk in blocks.items():
        blk_d = blk.to(DEV)
        for tb, tc in ((0, None), (1, 2), (n_tiles - 1, None)):
            buf.fill_(float('nan'))
            T = ops.tbuild_blocks(x_d, idx_d, blk_d, P, F, tb, tc, out=buf)
            assert T.data_ptr() == buf.data_ptr()
            e0, e1 = tile_edges(E, tb, tc)
            count = (e1 - e0 + ops.TILE_E - 1) // ops.TILE_E
            numel = ops.t_numel(count, Ci, F, P)
            t = decode_T(buf[:numel].cpu().numpy(), count, Ci, F, P, padded=True)
            got = torch.from_numpy(np.ascontiguousarray(t[:e1 - e0, :Ci * F, :P])).reshape(e1 - e0, Ci, F, P)
            ref = em.tbuild_blocks(x, idx, blk, P, F, tb, tc)
            bound = em.tbuild_blocks(x.abs(), idx, blk.abs(), P, F, tb, tc)
            _assert_close(got, ref, bound, 2e-6, f'{name} tiles {tb}+{tc}')
            pad = t.copy()
            pad[:e1 - e0, :Ci * F, :P] = 0.0
            assert np.all(pad == 0.0), f'{name} tiles {tb}+{tc}: layout padding not zero (or not written)'
            assert bool(buf[numel:].isnan().all()), f'{name} tiles {tb}+{tc}: written past t_numel'


# ------------------------------------------------------------------ power-of-two scales
def _scale_feats(g, max_degree, b=2, n=40, C=3):
    """Features of degrees 0..max_degree, per-node magnitudes 1e-5 .. 1e5, and nodes at the edges of the float range: cloud 0
    node 0 all zero, node 1 all -0.0, node 2 subnormal only, node 3 one component near FLT_MAX, node 4 its maximum in a middle
    degree and negative, node 5 the smallest subnormal as its only non-zero, node 6 a maximum of 2e36 (a scale below 2^-100)."""
    mag = torch.pow(10.0, torch.empty(b, n, 1, 1).uniform_(-5, 5, generator=g))
    feats = {str(d): torch.randn(b, n, C, 2 * d + 1, generator=g) * mag for d in range(max_degree + 1)}
    top = str(max_degree)
    mid = str(max_degree // 2)
    for d, t in feats.items():
        t[0, 0] = 0.0
        t[0, 1] = -0.0
        t[0, 2] = torch.randn(C, t.shape[-1], generator=g) * 1e-40
        t[0, 5] = 0.0
    feats[top][0, 3, 0, -1] = 3.3e38
    feats[mid][0, 4, -1, 0] = -1e6
    feats[top][0, 5, -1, 0] = 2.0 ** -149
    feats['0'][0, 6, 0, 0] = 2e36
    return {d: t.to(DEV) for d, t in feats.items()}


def _pow2_scale64(v, target_exp):
    """float64 statement of the power-of-two scale of a float32 magnitude v: 2^j with v 2^j in [2^(target-1), 2^target), j
    clamped to [-100, 100]; 1 where v is 0 or not below 3e38 (inf / NaN included)."""
    v = v.double().cpu()
    _, ex = torch.frexp(v)
    s = torch.exp2((target_exp - ex).clamp(-100, 100).double())
    ok = (v > 0) & (v < float(np.float32(3.0e38)))
    return torch.where(ok, s, torch.ones_like(s)), ok & (target_exp - ex).abs().le(100)


@pytest.mark.parametrize('max_degree', [0, 1, 2, 3, 4, 5])
def test_node_absmax_and_edge_scale(max_degree):
    """node_absmax is the maximum of |x| over every degree, bit for bit (torch.amax); edge_scale from those maxima equals
    edge_scale from the features; both edge_scale and the node scale of linear_tc (se3_pow2_scale_fwd, target 2^14) are the
    power of two their contract states."""
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(max_degree)
    b, n, k = 2, 40, 9
    feats = _scale_feats(g, max_degree, b, n)
    nodemax = ops.node_absmax(feats)
    want = torch.stack([t.abs().amax(dim=(2, 3)) for t in feats.values()]).amax(0).reshape(-1)
    assert torch.equal(nodemax.view(torch.int32), want.view(torch.int32))
    assert int(want[1].view(torch.int32)) == 0 and 0 < float(want[2]) < 1.2e-38 and float(want[5]) == 2.0 ** -149

    idx = torch.randint(0, n, (b, n, k), generator=g)
    idx[0, 0, :7] = torch.arange(7)                      # every special node is some edge's neighbour
    idx = idx.to(DEV)
    sx = ops.edge_scale(feats, idx, max_degree)
    assert torch.equal(sx, ops.edge_scale(None, idx, max_degree, nodemax=nodemax))
    nm = want[(idx + (torch.arange(b, device=DEV) * n)[:, None, None]).reshape(-1)]
    v = nm * torch.tensor(math.sqrt(2 * max_degree + 1), dtype=torch.float32, device=DEV)      # the kernel's float32 product
    for got, mag, target in ((sx, v, 10), (None, want, 14)):
        if got is None:                                  # linear_tc's per-node scale
            got = torch.empty_like(mag)
            assert ops.lib().se3_pow2_scale_fwd(mag.data_ptr(), mag.numel(), target, got.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream) == 0
        exp, in_range = _pow2_scale64(mag, target)
        got = got.cpu().double()
        assert torch.equal(got, exp), f'target 2^{target}'
        scaled = mag.cpu().double() * got
        assert bool(((scaled >= 2.0 ** (target - 1)) & (scaled < 2.0 ** target))[in_range].all())
        assert bool((got[mag.cpu() == 0] == 1).all())


# ------------------------------------------------------------------ decoder-sized launches
ZGEMM_MIXES = {                    # the segment mixes of test_gpu_zgemm.test_zgemm_matches_fp64: (C_in, ncomp, cplus, cminus, Kp)
    1: [[(8, 1, 0, 0, 16)], [(4, 3, 1, 1, 16), (12, 5, 2, 2, 16)], [(16, 1, 0, 0, 16), (8, 3, 1, 1, 32), (4, 7, 3, 3, 16)]],
    2: [[(6, 3, 2, 0, 16)], [(4, 3, 2, 0, 16), (10, 5, 3, 1, 32), (2, 7, 4, 2, 16)], [(32, 7, 6, 0, 16)]],
    3: [[(8, 3, 2, 0, 16)], [(4, 3, 2, 0, 16), (12, 5, 3, 1, 32), (4, 7, 4, 2, 16)], [(32, 7, 6, 0, 16)]],
}


@pytest.mark.parametrize('flush', [0, 1])
@pytest.mark.parametrize('Co', [128, 512])
@pytest.mark.parametrize('mix', [0, 1, 2])
@pytest.mark.parametrize('mode', [1, 2, 3])
def test_zgemm_at_decode_sizes(mode, mix, Co, flush):
    """E = 1, 16, 127, 128 edges (a decode step: one or a few nodes): against float64; forced split-K (2, 3 and the launch's
    split units; mode 2 has one unit) bit-identical to the unsplit launch; rows of the output buffer past E keep their fill on
    both paths; and the automatic choice splits exactly when the launch has more than one unit (its grid has at most four output
    tiles, far fewer than SMs).  torch.equal compares values, so it does not see a -0.0 that the split reduction (a sum that
    starts from +0.0) returns as +0.0; the hash tests of test_gpu_zgemm_splitk.py compare bits."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, Co, 1):
        pytest.skip('needs sm_90')
    planes = min(mode, 2)
    for E in (1, 16, 127, 128):
        segs, img, sx, ref = zgemm_problem(mode, Co, E, ZGEMM_MIXES[mode][mix], seed=E + flush)
        units = zgemm_split_units(segs, Co, mode, flush)
        assert units >= 1 and (mode != 2 or units == 1)

        def launch(k_split):
            buf = torch.full((E + 9, planes, Co), SENTINEL, device=DEV)
            ops.zgemm(segs, img, sx, E, Co, mode, buf[:E], planes * Co, [0, Co], flush_stages=flush, k_split=k_split)
            torch.cuda.synchronize()
            assert bool((buf[E:] == SENTINEL).all()), f'E={E} k_split={k_split}: rows past E written'
            return buf[:E]

        whole = launch(1)
        err = rel_err(whole.cpu().numpy(), ref.cpu().numpy())
        # the error is the tensor cores' accumulation rounding and does not depend on E.  Measured on an H100 80GB HBM3 (700 W)
        # over 25 seeds per (mode, mix, Co) at E = 16, 127 and 300: at most 3.9e-6 (mode 2, second mix; 3.4e-6 at E = 300), 3.0e-6
        # for mode 1, 2.9e-6 for mode 3.  test_zgemm_matches_fp64's 3e-6 for modes 1 and 2 lies inside that spread and holds
        # there only for its seeds, so modes 1 and 2 get 5e-6 here, not 3e-6.
        assert err < (6e-6 if mode == 3 else 5e-6), f'E={E}: {err:.3e}'
        for k_split in sorted({min(2, units), min(3, units), units} - {1}):
            assert torch.equal(launch(k_split), whole), f'E={E}: k_split={k_split} of {units} differs from the unsplit launch'
        before = ops.SPLIT_LAUNCHES
        assert torch.equal(launch(None), whole)
        assert ops.SPLIT_LAUNCHES - before == (1 if units > 1 else 0), f'E={E}: {units} units'


@pytest.mark.parametrize('K', [1, 16])
@pytest.mark.parametrize('li', [0, 1, 3, 5])
def test_rotgather_one_node(li, K):
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(10 * li + K)
    Ci, Q = 10, 2 * li + 1
    x = torch.randn(1, 1, Ci, Q, generator=g)
    idx = torch.zeros(1, 1, K, dtype=torch.int64)
    D = torch.randn(K, Q, Q, generator=g) if li else None
    X = ops.rotgather(x.to(DEV), idx.to(DEV), None if D is None else D.to(DEV))
    got = X[:Ci * Q * 128].reshape(Ci, Q, 128).permute(2, 0, 1).cpu()
    em = Emulation()
    ref = em.rotgather(x, idx, D)
    bound = em.rotgather(x.abs(), idx, None if D is None else D.abs())
    _assert_close(got[:K], ref, bound, 2e-6)
    assert bool((got[K:] == 0).all())


@pytest.mark.parametrize('K', [1, 16])
@pytest.mark.parametrize('lo', [0, 1, 2, 3])
def test_rotate_pool_one_node(lo, K):
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(10 * lo + K)
    Co, P = 96, 2 * lo + 1
    Op = torch.randn(K, P, Co, generator=g)
    D = torch.randn(K, P, P, generator=g) if lo else None
    em = Emulation()
    for mask in (None, torch.rand(K, generator=g) > 0.5, torch.zeros(K, dtype=torch.bool)):
        sa = torch.randn(1, Co, P, generator=g)
        out = torch.empty(1, Co, P, device=DEV)
        ops.rotate_pool(Op.to(DEV), None if D is None else D.to(DEV), None if mask is None else mask.to(DEV), sa.to(DEV), 1, K, Co, lo, out)
        ref, bound = torch.empty(1, Co, P, dtype=torch.float64), torch.empty(1, Co, P, dtype=torch.float64)
        em.rotate_pool(Op, D, mask, sa, 1, K, Co, lo, ref)
        em.rotate_pool(Op.abs(), None if D is None else D.abs(), mask, sa.abs(), 1, K, Co, lo, bound)
        _assert_close(out, ref, bound, 2e-6, f'mask {mask}')


@pytest.mark.parametrize('M', [1, 3, 5, 7])
def test_linear_tc_one_node(M):
    from se3_transformer_pytorch_b200 import ops
    D, Eo = 64, 128
    if not ops.linear_supported(D, Eo, DEV):
        pytest.skip('needs sm_90')
    g = torch.Generator().manual_seed(M)
    x = torch.randn(1, 1, D, M, generator=g) * 1e-3
    W = torch.randn(D, Eo, generator=g) / D ** 0.5
    img = ops.linear_image(W.to(DEV))
    for res in (None, torch.randn(1, 1, Eo, M, generator=g) * 1e-3):
        out = ops.linear_tc(x.to(DEV), img, Eo, res=None if res is None else res.to(DEV))
        ref = torch.einsum('bndm,de->bnem', x.double(), W.double()) + (0 if res is None else res.double())
        # 3-pass fp16 split (~2^-21 per product) + fp32 partial sums, as test_gpu_zgemm.test_linear_tc_matches_fp64
        assert float((out.cpu().double() - ref).abs().max() / ref.abs().max()) < 6e-6


@pytest.mark.parametrize('K', [1, 16])
@pytest.mark.parametrize('M', [1, 3, 7])
def test_attention_one_node(M, K):
    """One query node attending over itself and K neighbours; with D (M > 1) the keys and values arrive edge-aligned and
    component major and the kernel rotates them back."""
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(10 * M + K)
    H, Dh = 2, 16
    Ckv = H * Dh
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    q, sk, sv = f(1, 1, H * Dh, M), f(1, 1, Ckv, M), f(1, 1, Ckv, M)
    kw = dict(heads=H, dim_head=Dh, scale=Dh ** -0.5, self_k=cu(sk), self_v=cu(sv))
    k, v = f(1, 1, K, Ckv, M), f(1, 1, K, Ckv, M)
    with_self = lambda s, t: np.concatenate([s[:, :, None], t], 2)
    ref = attention_reference(q, with_self(sk, k), with_self(sv, v), None, H, Dh, H, Dh ** -0.5)
    assert rel_err(ops.attention(cu(q), cu(k), cu(v), **kw).cpu().numpy(), ref) < 5e-6
    if M == 1:
        return
    Dm = np.linalg.qr(rng.standard_normal((K, M, M)))[0].astype(np.float32)
    kp, vp = f(1, 1, K, M, Ckv), f(1, 1, K, M, Ckv)
    rot = lambda t: np.einsum('epn,enc->ecp', Dm.astype(np.float64), t.reshape(K, M, Ckv).astype(np.float64)).reshape(1, 1, K, Ckv, M)
    ref = attention_reference(q, with_self(sk, rot(kp)), with_self(sv, rot(vp)), None, H, Dh, H, Dh ** -0.5)
    got = ops.attention(cu(q), cu(kp), cu(vp), D=cu(Dm), k_aligned=True, **kw)
    assert rel_err(got.cpu().numpy(), ref) < 5e-6
