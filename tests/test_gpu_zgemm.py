"""Kernel-level parity of the production path's kernels (csrc/zgemm.cu, aligned.cu, radial_trunk_u) through the C ABI against
float64 restatements of what each computes (DESIGN.md 4.5); the whole-model / oracle comparisons at the benchmarked shape are
in test_gpu_headline.py.  Tolerances are written next to each assert (north_star: 1e-4 relative on outputs)."""
import numpy as np
import pytest
import torch

from helpers import rel_err, run_zgemm

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.mark.parametrize('mode,Co,E,segs', [
    (1, 256, 300, [(8, 1, 0, 0, 16)]),                                     # N = 256, 3 edge tiles (the last one partly filled)
    (1, 128, 128, [(4, 3, 1, 1, 16), (12, 5, 2, 2, 16)]),                  # N = 128 tile, two input degrees
    (1, 512, 257, [(16, 1, 0, 0, 16), (8, 3, 1, 1, 32), (4, 7, 3, 3, 16)]),  # a K = 32 pair (two sub-segments)
    (2, 128, 300, [(6, 3, 2, 0, 16)]),                                     # (+m, -m) = components 2, 0 of an l = 1 input
    (2, 256, 200, [(4, 3, 2, 0, 16), (10, 5, 3, 1, 32), (2, 7, 4, 2, 16)]),
    (2, 512, 129, [(32, 7, 6, 0, 16)]),
    (3, 128, 300, [(8, 3, 2, 0, 16)]),
    (3, 256, 200, [(4, 3, 2, 0, 16), (12, 5, 3, 1, 32), (4, 7, 4, 2, 16)]),
    (3, 512, 129, [(32, 7, 6, 0, 16)]),
])
@pytest.mark.parametrize('flush', [0, 1, 2, 3, 7])
def test_zgemm_matches_fp64(mode, Co, E, segs, flush):
    """One launch against float64, with the fp32 drain of the accumulators every `flush` stages (0: the default schedule)."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, Co, 1):
        pytest.skip('needs sm_90')
    out, ref = run_zgemm(mode, Co, E, segs, flush=flush, seed=flush)
    err = rel_err(out.cpu().numpy(), ref.cpu().numpy())
    assert err < (6e-6 if mode == 3 else 3e-6), f'flush={flush}: {err:.3e}'


@pytest.mark.parametrize('x_scale', [1e-6, 1.0, 3e4])
def test_zgemm_is_scale_invariant(x_scale):
    """The per-edge power-of-two scale keeps the fp16 operands in range whatever the magnitude of the features."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    for mode in (2, 3):
        out, ref = run_zgemm(mode, 128, 200, [(8, 3, 2, 0, 16)], x_scale=x_scale)
        assert rel_err(out.cpu().numpy(), ref.cpu().numpy()) < 6e-6


@pytest.mark.parametrize('mode', [1, 2, 3])
def test_zgemm_headline_width_long_k(mode):
    """cfg2 widths (C_in = C_out = 512, four input degrees: K = 32768 / 65536 per output) with all-positive operands, the
    worst case for the round-toward-zero accumulation of the tensor cores: the periodic drain into fp32 registers keeps the
    result within 1e-5 of float64 (the error without it is recorded next to it)."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 512, 1):
        pytest.skip('needs sm_90')
    segs = [(512, 2 * l + 1, l + (1 if mode >= 2 and l else 0), l - (1 if mode >= 2 and l else 0), 16) for l in ((0, 1, 2, 3) if mode == 1 else (1, 2, 3))]
    out, ref = run_zgemm(mode, 512, 512, segs, flush=0, positive=True)
    err = rel_err(out.cpu().numpy(), ref.cpu().numpy())
    out2, _ = run_zgemm(mode, 512, 512, segs, flush=1 << 20, positive=True)
    err_nodrain = rel_err(out2.cpu().numpy(), ref.cpu().numpy())
    print(f'zgemm mode {mode} long-K positive operands: rel err {err:.3e} (default drain), {err_nodrain:.3e} (never drained)')
    import json, os
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/zgemm_accumulation.jsonl', 'a') as f:
        f.write(json.dumps(dict(mode=mode, rel_err_default_drain=err, rel_err_never_drained=err_nodrain)) + '\n')
    assert err < 1e-5


def test_frames_match_float64_host_math():
    """se3_frames_fwd vs the float64 torch restatement (aligned.EdgeFrames: Rodrigues rotation, Wigner matrices from the
    harmonics at rotated sample points), including coincident points (r = 0), the axis itself and its antipode."""
    from se3_transformer_pytorch_b200 import ops, aligned
    g = torch.Generator().manual_seed(0)
    rel = torch.randn(500, 3, generator=g)
    rel[0] = 0.0
    rel[1] = torch.tensor([0.0, 2.0, 0.0])
    rel[2] = torch.tensor([0.0, -3.0, 0.0])
    rel[3] = torch.tensor([1e-4, -1.0, 0.0])
    rel[4] = torch.tensor([0.5, 0.0, 0.0])
    rel = rel.to(DEV)
    for lmax in (1, 3, 5):
        D = ops.frames(rel, lmax)
        ref = aligned.EdgeFrames(rel, lmax).D
        for l in range(1, lmax + 1):
            assert float((D[l] - ref[l]).abs().max()) < 2e-6, l
            eye = torch.eye(2 * l + 1, device=DEV)
            assert float((D[l] @ D[l].transpose(1, 2) - eye).abs().max()) < 1e-5          # orthogonal


@pytest.mark.parametrize('li,Ci,b,n,k', [(0, 10, 1, 20, 7), (1, 6, 2, 30, 9), (3, 5, 1, 40, 16), (5, 3, 1, 12, 5)])
def test_rotgather(li, Ci, b, n, k):
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(li)
    Q = 2 * li + 1
    x = torch.randn(b, n, Ci, Q, generator=g).to(DEV)
    idx = torch.randint(0, n, (b, n, k), generator=g).to(DEV)
    E = b * n * k
    D = torch.randn(E, Q, Q, generator=g).to(DEV) if li else None
    X = ops.rotgather(x, idx, D)
    tiles = (E + 127) // 128
    got = X[:tiles * Ci * Q * 128].reshape(tiles, Ci, Q, 128).permute(0, 3, 1, 2).reshape(tiles * 128, Ci, Q)
    xg = x.reshape(b * n, Ci, Q)[(idx + (torch.arange(b, device=DEV) * n)[:, None, None]).reshape(-1)]
    ref = xg if D is None else torch.einsum('eqn,eiq->ein', D.double(), xg.double()).float()
    assert float((got[:E] - ref).abs().max()) < 1e-5
    assert float(got[E:].abs().max()) == 0.0 if tiles * 128 > E else True


def test_edge_scale():
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(0)
    b, n, k = 2, 16, 5
    feats = {'0': torch.randn(b, n, 4, 1, generator=g).to(DEV) * 1e-3, '1': torch.randn(b, n, 4, 3, generator=g).to(DEV) * 50}
    feats['1'][0, 3] = 0.0
    feats['0'][0, 3] = 0.0
    idx = torch.randint(0, n, (b, n, k), generator=g).to(DEV)
    sx = ops.edge_scale(feats, idx, 1)
    nodemax = torch.maximum(feats['0'].abs().amax(dim=(2, 3)), feats['1'].abs().amax(dim=(2, 3))).reshape(-1)
    nm = nodemax[(idx + (torch.arange(b, device=DEV) * n)[:, None, None]).reshape(-1)]
    v = nm * 3 ** 0.5 * sx
    assert bool(((v < 1024) & (v >= 512))[nm > 0].all())
    assert bool((sx[nm == 0] == 1).all())
    assert bool((torch.log2(sx) == torch.log2(sx).round()).all())


def test_radial_trunk_u():
    """Fused trunk + radial coordinates: g identical to se3_radial_trunk_fwd, U = g V (ones column at r), residual statistics."""
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(0)
    E, in_dim, pairs = 200, 1, 3
    feat = (torch.rand(E, in_dim, generator=g) * 3).to(DEV)
    stride = ops.trunk_param_stride(in_dim)
    params = (torch.randn(pairs, stride, generator=g) * 0.3).to(DEV)
    g_ref = ops.radial_trunk(feat, params, pairs)
    r = [15, 31, 20]
    V = torch.zeros(pairs, 128, 64, device=DEV)
    for p in range(pairs):
        q, _ = torch.linalg.qr(torch.randn(128, r[p], generator=g))
        V[p, :, :r[p]] = q.to(DEV)
    ones_col = torch.tensor(r, dtype=torch.int32, device=DEV)
    gmean = g_ref.mean(dim=1).contiguous()                   # the centre of the affine model
    stats = torch.zeros(pairs, 2, device=DEV)
    U, g_out = ops.radial_trunk_u(feat, params, V, gmean, ones_col, stats, want_g=True)
    assert torch.equal(g_out, g_ref)
    for p in range(pairs):
        gc = g_ref[p].double() - gmean[p].double()
        ref = gc @ V[p].double()
        assert float((U[p, :, :r[p]] - ref[:, :r[p]]).abs().max()) < 1e-5
        assert bool((U[p, :, r[p]] == 1).all()) and float(U[p, :, r[p] + 1:].abs().max()) == 0.0
        resid = (gc - ref @ V[p].double().t()).abs().max()
        assert abs(float(stats[p, 0]) - float(resid)) < 1e-5 * max(1.0, float(resid))
        assert abs(float(stats[p, 1]) - float(g_ref[p].abs().max())) < 1e-6
    U2, none = ops.radial_trunk_u(feat, params, V, gmean, ones_col, stats)
    assert none is None and torch.equal(U2, U)


@pytest.mark.parametrize('M,Dh,H,K,opts', [
    (3, 16, 2, 5, dict(self_kv=True)),
    (7, 64, 8, 16, dict(self_kv=True, mask=True)),
    (5, 24, 3, 9, dict(self_kv=True, null=True, one_headed=True, mask=True)),
    (3, 8, 2, 4, dict(self_kv=True, linear_keys=True)),
    (7, 40, 2, 6, dict(mask=True, all_masked_row=True, self_kv=False)),
])
def test_attention_with_fused_rotate_back(M, Dh, H, K, opts):
    """se3_attn_aligned_fwd (keys / values in the edge frame, rotated inside the kernel) == se3_attn_fwd on the rotated tensors."""
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(M * 100 + K)
    b, n = 2, 11
    hk = 1 if opts.get('one_headed') else H
    Ckv = hk * Dh
    rn = lambda *s: torch.randn(*s, generator=g).to(DEV)
    q = rn(b, n, H * Dh, M)
    kp, vp = rn(b, n, K, M, Ckv), rn(b, n, K, M, Ckv)              # aligned, component major
    Dm, _ = torch.linalg.qr(torch.randn(b * n * K, M, M, generator=g))
    Dm = Dm.to(DEV).contiguous()
    rot = lambda t: torch.einsum('epn,enc->ecp', Dm.double(), t.reshape(-1, M, Ckv).double()).float().reshape(b, n, K, Ckv, M)
    kw = dict(heads=H, dim_head=Dh, scale=Dh ** -0.5, kv_heads=hk)
    if opts.get('self_kv'):
        kw.update(self_k=rn(b, n, Ckv, M), self_v=rn(b, n, Ckv, M))
    if opts.get('null'):
        kw.update(null_k=rn(Ckv, M), null_v=rn(Ckv, M))
    if opts.get('mask'):
        m = torch.rand(b, n, K, generator=g) > 0.3
        if opts.get('all_masked_row'):
            m[0, 0] = False
        kw.update(nmask=m.to(DEV))
    if opts.get('linear_keys'):
        k_node = rn(b, n, Ckv, M)
        idx = torch.randint(0, n, (b, n, K), generator=g).to(DEV)
        ref = ops.attention(q, k_node, rot(vp), k_idx=idx, **kw)
        out = ops.attention(q, k_node, vp, k_idx=idx, D=Dm, k_aligned=False, **kw)
    else:
        ref = ops.attention(q, rot(kp), rot(vp), **kw)
        out = ops.attention(q, kp, vp, D=Dm, k_aligned=True, **kw)
    assert rel_err(out.cpu().numpy(), ref.cpu().numpy()) < 3e-6


@pytest.mark.parametrize('lo,K,Co,masked,self_add', [(0, 8, 128, True, True), (1, 5, 96, True, False), (3, 16, 256, True, True), (2, 40, 300, False, True)])
def test_rotate_pool(lo, K, Co, masked, self_add):
    """Fused rotate-back + masked mean over the neighbours + self-interaction (S:256-266, utils.py:72-80)."""
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(lo)
    nodes, P = 23, 2 * lo + 1
    Op = torch.randn(nodes * K, P, Co, generator=g).to(DEV)
    D = torch.randn(nodes * K, P, P, generator=g).to(DEV) if lo else None
    mask = (torch.rand(nodes * K, generator=g) > 0.4).to(DEV) if masked else None
    if masked:
        mask[:K] = False                                           # a node with no valid neighbour -> zero (+ self term)
    sa = torch.randn(nodes, Co, P, generator=g).to(DEV) if self_add else None
    out = torch.empty(nodes, Co, P, device=DEV)
    ops.rotate_pool(Op, D, mask, sa, nodes, K, Co, lo, out)
    rot = Op.double().transpose(1, 2) if D is None else torch.einsum('epn,enc->ecp', D.double(), Op.double())       # [E, Co, P]
    rot = rot.reshape(nodes, K, Co, P)
    if mask is None:
        ref = rot.mean(1)
    else:
        mk = mask.reshape(nodes, K, 1, 1).double()
        cnt = mk.sum(1)
        ref = (rot * mk).sum(1) / cnt.clamp(min=1.0)
        ref = torch.where(cnt == 0, torch.zeros_like(ref), ref)
    if sa is not None:
        ref = ref + sa.double()
    assert float((out.double() - ref).abs().max()) < 1e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('D,Eo,M,nodes,with_res', [(64, 128, 1, 37, False), (512, 512, 7, 50, True), (2048, 512, 3, 33, True),
                                                   (512, 2048, 5, 29, False), (128, 256, 1, 300, True)])
def test_linear_tc_matches_fp64(D, Eo, M, nodes, with_res):
    """LinearSE3 on the tensor cores (reference S:78-95, A operand read in place from [b,n,D,M]) vs float64, also with the
    fused residual and with features of very different magnitude per node (the per-node power-of-two scale)."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.linear_supported(D, Eo, DEV):
        pytest.skip('needs sm_90')
    g = torch.Generator().manual_seed(D + M)
    x = torch.randn(1, nodes, D, M, generator=g)
    x = x * torch.logspace(-6, 4, nodes).view(1, nodes, 1, 1)          # per-node magnitudes 1e-6 .. 1e4
    x[0, 3] = 0.0
    x = x.to(DEV)
    W = (torch.randn(D, Eo, generator=g) / D ** 0.5).to(DEV)
    res = torch.randn(1, nodes, Eo, M, generator=g).to(DEV) * x.abs().amax(dim=(2, 3), keepdim=True) if with_res else None
    out = ops.linear_tc(x, ops.linear_image(W), Eo, res=res)
    ref = torch.einsum('bndm,de->bnem', x.double(), W.double())
    if res is not None:
        ref = ref + res.double()
    # relative to each node's own output scale (rows differ by 10 orders of magnitude)
    scale = ref.abs().amax(dim=(2, 3), keepdim=True).clamp(min=1e-30)
    # 3-pass fp16 split (~2^-21 per product) + fp32 partial sums: a few 1e-6 of the row's scale
    assert float(((out.double() - ref).abs() / scale).max()) < 6e-6
    assert float(out[0, 3].abs().max()) == 0.0 or with_res


def test_radial_table_matches_trunk_kernel():
    """Radial coordinates by table lookup (se3_radial_table_fwd, 4-point Lagrange on the plan's float64 grid) vs the per-edge
    radial MLP + projection (se3_radial_trunk_u_fwd) on the same distances; out-of-range distances raise the flag."""
    from se3_transformer_pytorch_b200 import ops
    from se3_transformer_pytorch_b200.model import ConvSE3, Fiber
    torch.manual_seed(0)
    conv = ConvSE3(Fiber.create(2, 128), Fiber.create(2, 128), pool=False, self_interaction=False).to(DEV)
    plan = conv.lowrank_plan(4.0)
    assert plan['utab'] is not None and conv.utable_error < 2e-7, conv.utable_error
    pairs = len(conv.pairs)
    Vs = torch.stack([plan['pairs'][p]['V'] for p in conv.pairs]).contiguous()
    gm = torch.stack([plan['pairs'][p]['gmean'] for p in conv.pairs]).contiguous()
    ones = torch.tensor([plan['pairs'][p]['r'] for p in conv.pairs], dtype=torch.int32, device=DEV)
    d = torch.cat([torch.rand(5000, device=DEV) * 4.0, torch.tensor([0.0, 4.0, plan['D']], device=DEV)])
    stats_t, stats_k = torch.zeros(pairs, 2, device=DEV), torch.zeros(pairs, 2, device=DEV)
    Ut = ops.radial_table(d, plan['utab'], plan['D'], ones, stats_t)
    Uk, _ = ops.radial_trunk_u(d.unsqueeze(-1).contiguous(), conv.packed()['trunk'], Vs, gm, ones, stats_k)
    assert float((Ut - Uk).abs().max()) < 3e-6 * max(1.0, float(Uk.abs().max()))     # the fp32 MLP itself is ~1e-6 off float64
    assert float(stats_t.abs().max()) == 0.0
    ops.radial_table(torch.tensor([1.0, plan['D'] * 1.01], device=DEV), plan['utab'], plan['D'], ones, stats_t)
    assert bool((stats_t == 1).all())
    ops.radial_table(torch.tensor([float('nan')], device=DEV), plan['utab'], plan['D'], ones, stats_k.zero_())
    assert bool((stats_k == 1).all())
