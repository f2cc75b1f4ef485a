"""GPU parity tests, kernel by kernel, through the C ABI (ctypes) against the numpy oracle and the committed
reference-generated fixtures.  Tolerances: indices/masks bit exact; fp32 values within the relative bound written
next to each assert (north_star: 1e-4 relative)."""
import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_case, rel_err, decode_T, assert_graph_equal
from oracle import se3_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def cu(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


# ------------------------------------------------------------------ K1
@pytest.mark.parametrize('case', [
    dict(b=2, n=33, k=8), dict(b=1, n=17, k=16), dict(b=2, n=64, k=5, radius=1.2, ragged=True),
    dict(b=1, n=40, k=6, causal=True), dict(b=2, n=24, k=7, nbr=True), dict(b=1, n=32, k=10, sparse=4, knn0=True),
    dict(b=1, n=300, k=16), dict(b=1, n=1024, k=16),
])
def test_knn_matches_oracle(case):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(1)
    b, n, k = case['b'], case['n'], case['k']
    coors = rng.standard_normal((b, n, 3)).astype(np.float32)
    mask = np.ones((b, n), dtype=bool)
    if case.get('ragged'):
        mask[0, -5:] = False
        mask[1, -11:] = False
    nbr = (rng.random((b, n, n)) < 0.5) if case.get('nbr') else None
    sparse = None
    num_neighbors = k
    if case.get('sparse'):
        i = np.arange(n)
        sparse = np.broadcast_to((np.abs(i[:, None] - i[None]) <= case['sparse']) & (i[:, None] != i[None]), (b, n, n)).copy()
    radius = case.get('radius', 1e5)
    g = O.neighbor_graph(coors, mask, num_neighbors=0 if case.get('knn0') else num_neighbors, valid_radius=radius,
                         causal=case.get('causal', False), sparse_adj=sparse, neighbor_mask=nbr)
    kk = g['idx'].shape[-1]
    idx, nm, rel_pos, rel_dist = ops.knn(cu(coors), kk, 0 if case.get('knn0') else radius, node_mask=cu(mask),
                                         neighbor_mask=None if nbr is None else cu(nbr),
                                         sparse_adj=None if sparse is None else cu(sparse), causal=case.get('causal', False))
    idx, nm, rel_pos, rel_dist = (t.cpu().numpy() for t in (idx, nm, rel_pos, rel_dist))
    assert_graph_equal(idx, nm, rel_dist, g['idx'], g['mask'], g['rel_dist'])
    if not (case.get('causal') or case.get('nbr') or case.get('sparse')):
        # no engineered ties: the full ordered lists agree bit for bit
        assert np.array_equal(idx, g['idx'])
        assert np.array_equal(nm, g['mask'])
        assert np.array_equal(rel_pos, g['rel_pos'])
    # rel_pos / rel_dist are consistent with idx everywhere
    bi = np.arange(b)[:, None, None]
    assert np.array_equal(rel_pos, coors[:, :, None, :] - coors[bi, idx])
    assert np.allclose(rel_dist, np.sqrt((rel_pos.astype(np.float64) ** 2).sum(-1)), rtol=1e-6)


def test_gather_pairs_and_pool():
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(2)
    b, n, k, e = 2, 19, 5, 7
    pf = rng.standard_normal((b, n, n, e)).astype(np.float32)
    idx = rng.integers(0, n, (b, n, k))
    out = ops.gather_pairs(cu(pf), cu(idx)).cpu().numpy()
    assert np.array_equal(out, np.take_along_axis(pf, idx[..., None], 2))
    x = rng.standard_normal((b, n, k, 6, 3)).astype(np.float32)
    m = rng.random((b, n, k)) < 0.6
    m[0, 0] = False                                            # an all-masked row -> zeros (utils.py:79)
    got = ops.pool(cu(x), cu(m)).cpu().numpy()
    assert rel_err(got, O.masked_mean(x, m, 2)) < 1e-6
    assert np.all(got[0, 0] == 0)


# ------------------------------------------------------------------ K2
def test_basis_matches_reference_fixture_and_oracle():
    from se3_transformer_pytorch_b200 import ops
    z = np.load(f'{GOLDEN}/sh_basis.npz')
    r = z['r_ij']
    basis = ops.get_basis(cu(r), 3)
    assert len(basis) == 16
    for key, v in basis.items():
        li, lo = key.split(',')
        got = v.cpu().numpy().reshape(r.shape[0], 2 * int(lo) + 1, 2 * int(li) + 1, -1)
        ref = z[f'basis_{li}_{lo}']
        assert np.abs(got - ref)[:-1].max() < 3e-5, key                     # reference fp32 path
        # last fixture vector is 1e-4 off the pole: the reference's fp32 (1 - cos^2)^(m/2) cancels to 0 there, the
        # Cartesian evaluation keeps the true 3.5e-5 -- inside the 1e-4 parity bound, and closer to the fp64 value
        assert np.abs(got - ref).max() < 1e-4, key
    rng = np.random.default_rng(3)
    r2 = rng.standard_normal((2, 50, 4, 3)).astype(np.float32)
    ref = O.get_basis(r2.astype(np.float64), 3)
    got = ops.get_basis(cu(r2), 3)
    for key in ref:
        li, lo = key.split(',')
        assert got[key].shape == (2, 50, 4, 1, 2 * int(lo) + 1, 1, 2 * int(li) + 1, 2 * min(int(li), int(lo)) + 1)
        assert np.abs(got[key].cpu().numpy().reshape(ref[key].shape) - ref[key]).max() < 2e-6, key
    # higher degrees (tables shipped to degree 5)
    ref5 = O.get_basis(r2[:1, :8].astype(np.float64), 5)
    got5 = ops.get_basis(cu(r2[:1, :8]), 5)
    for key in ref5:
        assert np.abs(got5[key].cpu().numpy().reshape(ref5[key].shape) - ref5[key]).max() < 5e-6, key


# ------------------------------------------------------------------ K3
@pytest.mark.parametrize('in_dim,E', [(1, 300), (9, 129), (35, 64)])
def test_radial_trunk(in_dim, E):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(4)
    pairs = 3
    feat = np.abs(rng.standard_normal((E, in_dim))).astype(np.float32)
    Ps, packs = [], []
    for p in range(pairs):
        P = {'net.0.weight': rng.standard_normal((128, in_dim)) / np.sqrt(in_dim), 'net.0.bias': 0.1 * rng.standard_normal(128),
             'net.1.weight': 1 + 0.1 * rng.standard_normal(128), 'net.1.bias': 0.1 * rng.standard_normal(128),
             'net.3.weight': rng.standard_normal((128, 128)) / np.sqrt(128), 'net.3.bias': 0.1 * rng.standard_normal(128),
             'net.4.weight': 1 + 0.1 * rng.standard_normal(128), 'net.4.bias': 0.1 * rng.standard_normal(128)}
        P = {k: v.astype(np.float32) for k, v in P.items()}
        Ps.append(P)
        packs.append(np.concatenate([P['net.0.weight'].T.ravel(), P['net.0.bias'], P['net.1.weight'], P['net.1.bias'],
                                     P['net.3.weight'].T.ravel(), P['net.3.bias'], P['net.4.weight'], P['net.4.bias']]))
    params = cu(np.stack(packs))
    assert params.shape[1] == ops.trunk_param_stride(in_dim)
    g = ops.radial_trunk(cu(feat), params, pairs).cpu().numpy()
    for p in range(pairs):
        ref = O.radial_trunk(feat.astype(np.float64), {k: v.astype(np.float64) for k, v in Ps[p].items()}, '')
        assert rel_err(g[p], ref) < 5e-6


# ------------------------------------------------------------------ K4
def _pair_problem(rng, b, n, k, Ci, Co, di, do):
    Q, P, F = 2 * di + 1, 2 * do + 1, 2 * min(di, do) + 1
    E = b * n * k
    x = rng.standard_normal((b, n, Ci, Q)).astype(np.float32)
    idx = rng.integers(0, n, (b, n, k))
    Bm = rng.standard_normal((E, P, Q, F)).astype(np.float32)
    g = np.abs(rng.standard_normal((E, 128))).astype(np.float32)
    W3 = (rng.standard_normal((Co * Ci * F, 128)) / np.sqrt(128)).astype(np.float32)
    b3 = (0.1 * rng.standard_normal(Co * Ci * F)).astype(np.float32)
    xj = x[np.arange(b)[:, None, None], idx].reshape(E, Ci, Q)
    T = np.einsum('epqf,eiq->eifp', Bm.astype(np.float64), xj.astype(np.float64))
    R = (g.astype(np.float64) @ W3.astype(np.float64).T + b3).reshape(E, Co, Ci, F)
    out = np.einsum('eoif,eifp->eop', R, T)
    return dict(x=x, idx=idx, B=Bm, g=g, W3=W3, b3=b3, T=T.reshape(E, Ci * F, P), R=R, out=out, E=E, P=P, Q=Q, F=F)


@pytest.mark.parametrize('di,do,Ci', [(0, 0, 5), (1, 2, 6), (3, 3, 4), (2, 1, 7), (4, 5, 3)])
def test_tbuild(di, do, Ci):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(5)
    pr = _pair_problem(rng, 2, 11, 7, Ci, 4, di, do)
    n_tiles = (pr['E'] + 127) // 128
    T = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do)
    got = decode_T(T.cpu().numpy(), n_tiles, Ci, pr['F'], pr['P'])
    assert rel_err(got[:pr['E']], pr['T']) < 2e-6
    assert np.all(got[pr['E']:] == 0)
    # tile sub-range (edge chunking) gives the same tiles
    if n_tiles > 1:
        T1 = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do, tile_begin=1, tile_count=1)
        got1 = decode_T(T1.cpu().numpy(), 1, Ci, pr['F'], pr['P'])
        assert np.array_equal(got1, got[128:256])


@pytest.mark.parametrize('di,do,Ci,Co', [(0, 0, 8, 16), (1, 1, 5, 7), (2, 3, 6, 33), (3, 3, 4, 16), (1, 0, 9, 4)])
def test_pairwise_simt(di, do, Ci, Co):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(6)
    pr = _pair_problem(rng, 1, 13, 11, Ci, Co, di, do)
    E, P, F = pr['E'], pr['P'], pr['F']
    T = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do)
    out = torch.full((E, Co, P), 7.0, device=DEV)
    ops.pairwise_simt(cu(pr['g']), cu(pr['W3']), cu(pr['b3']), T, E, Co, Ci, F, P, out, accumulate=False)
    assert rel_err(out.cpu().numpy(), pr['out']) < 5e-6
    ops.pairwise_simt(cu(pr['g']), cu(pr['W3']), cu(pr['b3']), T, E, Co, Ci, F, P, out, accumulate=True)
    assert rel_err(out.cpu().numpy(), 2 * pr['out']) < 5e-6


@pytest.mark.parametrize('di,do,Ci,Co,n,k', [(0, 0, 8, 32, 16, 8), (1, 1, 5, 32, 16, 9), (3, 3, 4, 64, 20, 13), (2, 3, 6, 32, 32, 8),
                                             (1, 0, 33, 96, 16, 8), (3, 2, 16, 32, 7, 5)])
def test_pairwise_tc_matches_fp64(di, do, Ci, Co, n, k):
    """tcgen05 kernel (3-pass bf16 split) vs float64 numpy: 2e-5 relative; also the raw R tile of step 0."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, Co, 2 * do + 1):
        pytest.skip('tensor-core path needs sm_90')
    rng = np.random.default_rng(7)
    pr = _pair_problem(rng, 1, n, k, Ci, Co, di, do)
    E, P, F = pr['E'], pr['P'], pr['F']
    T = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do)
    w_img = ops.pack_w3(cu(pr['W3']), cu(pr['b3']), Co, Ci, F)
    g_dev = cu(pr['g'])
    n_tiles = (E + 127) // 128
    out = torch.full((E, Co, P), 3.0, device=DEV)
    dump = torch.zeros((n_tiles, Co // 32, 128, 128), device=DEV)
    ops.pairwise_tc(g_dev, w_img, T, E, Co, Ci, F, P, out, accumulate=False, dump=dump)
    torch.cuda.synchronize()
    # R of step 0: column = if_local*32 + o_local for (i,f) 0..3 of each 32-channel block
    R = pr['R'].reshape(E, Co, Ci * F)
    d = dump.cpu().numpy()
    for ob in range(Co // 32):
        for ifl in range(min(4, Ci * F)):
            got = d[:, ob, :, ifl * 32:(ifl + 1) * 32].reshape(n_tiles * 128, 32)[:E]
            assert rel_err(got, R[:, ob * 32:(ob + 1) * 32, ifl]) < 2e-5, (ob, ifl)
    assert rel_err(out.cpu().numpy(), pr['out']) < 2e-5
    ops.pairwise_tc(g_dev, w_img, T, E, Co, Ci, F, P, out, accumulate=True)
    assert rel_err(out.cpu().numpy(), 2 * pr['out']) < 2e-5


@pytest.mark.parametrize('csz', [1, 2, 4])
def test_pairwise_tc_cluster_sizes(csz, monkeypatch):
    """W-multicast cluster sizes 1/2/4 (incl. a padded last cluster: 5 edge tiles) give the same result."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 64, 5):
        pytest.skip('tensor-core path needs sm_90')
    monkeypatch.setenv('SE3B200_TC_CLUSTER', str(csz))
    rng = np.random.default_rng(9)
    di, do, Ci, Co = 2, 2, 12, 64
    pr = _pair_problem(rng, 1, 40, 15, Ci, Co, di, do)         # E = 600 -> 5 edge tiles
    E, P, F = pr['E'], pr['P'], pr['F']
    T = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do)
    out = torch.zeros((E, Co, P), device=DEV)
    ops.pairwise_tc(cu(pr['g']), ops.pack_w3(cu(pr['W3']), cu(pr['b3']), Co, Ci, F), T, E, Co, Ci, F, P, out, accumulate=False)
    assert rel_err(out.cpu().numpy(), pr['out']) < 2e-5


@pytest.mark.parametrize('r,P,di,do', [(15, 7, 3, 3), (31, 3, 1, 1), (20, 5, 2, 2), (63, 1, 0, 0)])
def test_pairwise_lowrank_matches_fp64(r, P, di, do):
    """Low-rank radial kernel: G = U V^T exactly of rank r; result vs float64 of the original (K = 128) contraction."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 64, P):
        pytest.skip('tensor-core path needs sm_90')
    rng = np.random.default_rng(11)
    Ci, Co = 10, 64
    pr = _pair_problem(rng, 1, 30, 9, Ci, Co, di, do)             # E = 270 -> 3 edge tiles (one padding CTA in a 2-cluster)
    E, F = pr['E'], pr['F']
    Vq, _ = np.linalg.qr(rng.standard_normal((128, r)))
    Ur = rng.standard_normal((E, r))
    G = (Ur @ Vq.T)                                                # exactly rank r
    W3, b3 = pr['W3'].astype(np.float64), pr['b3'].astype(np.float64)
    R = (G @ W3.T + b3).reshape(E, Co, Ci, F)
    ref = np.einsum('eoif,eifp->eop', R, pr['T'].reshape(E, Ci, F, P))
    Kp = 16 * ((r + 1 + 15) // 16)
    U = np.zeros((E, 64), dtype=np.float32); U[:, :r] = Ur; U[:, r] = 1.0
    Fp = np.zeros((Co * Ci * F, Kp), dtype=np.float32); Fp[:, :r] = W3 @ Vq; Fp[:, r] = b3
    T = ops.tbuild(cu(pr['x']), cu(pr['idx']), cu(pr['B']).reshape(-1), di, do)
    img = ops.pack_lowrank(cu(Fp), Co, Ci, F, Kp)
    out = torch.full((E, Co, P), 5.0, device=DEV)
    ops.pairwise_lr(cu(U), img, T, E, Co, Ci, F, P, Kp, out, accumulate=False)
    assert rel_err(out.cpu().numpy(), ref) < 3e-6
    ops.pairwise_lr(cu(U), img, T, E, Co, Ci, F, P, Kp, out, accumulate=True)
    assert rel_err(out.cpu().numpy(), 2 * ref) < 3e-6


@pytest.mark.parametrize('r,di,do', [(15, 0, 3), (15, 1, 3), (31, 1, 2), (15, 0, 1)])
def test_input_side_contraction_matches_fp64(r, di, do):
    """Pairs with l_in < l_out on the low-rank path: S = R x (Q FMAs per radial weight), then the basis fold; result vs
    float64 of the reference order (kernel = R . B first, S:336-343)."""
    from se3_transformer_pytorch_b200 import ops
    P, Q = 2 * do + 1, 2 * di + 1
    if not ops.tc_supported(DEV, 64, P):
        pytest.skip('tensor-core path needs sm_90')
    rng = np.random.default_rng(17)
    Ci, Co = 12, 64
    pr = _pair_problem(rng, 1, 30, 9, Ci, Co, di, do)
    E, F = pr['E'], pr['F']
    Vq, _ = np.linalg.qr(rng.standard_normal((128, r)))
    Ur = rng.standard_normal((E, r))
    G = Ur @ Vq.T
    W3, b3 = pr['W3'].astype(np.float64), pr['b3'].astype(np.float64)
    R = (G @ W3.T + b3).reshape(E, Co, Ci, F)
    ref = np.einsum('eoif,eifp->eop', R, pr['T'].reshape(E, Ci, F, P))
    Kp = 16 * ((r + 1 + 15) // 16)
    U = np.zeros((E, 64), dtype=np.float32); U[:, :r] = Ur; U[:, r] = 1.0
    Fp = np.zeros((Co * Ci * F, Kp), dtype=np.float32); Fp[:, :r] = W3 @ Vq; Fp[:, r] = b3
    X = ops.gather_tiles(cu(pr['x']), cu(pr['idx']))
    Xd = decode_T(X.cpu().numpy(), (E + 127) // 128, Ci, 1, Q)[:E]   # [E, Ci, Q] == gathered neighbour features
    xg = pr['x'].reshape(-1, Ci, Q)[pr['idx'].reshape(-1)]
    assert np.array_equal(Xd, xg)
    S = torch.empty((F, E, Co, Q), device=DEV)
    Fv = Fp.reshape(Co, Ci, F, Kp)
    for f in range(F):
        img = ops.pack_lowrank(cu(np.ascontiguousarray(Fv[:, :, f, :]).reshape(-1, Kp)), Co, Ci, 1, Kp)
        ops.pairwise_lr(cu(U), img, X, E, Co, Ci, 1, Q, Kp, S[f], accumulate=False, alg_P=P)
    out = torch.full((E, Co, P), 5.0, device=DEV)
    Bp = cu(pr['B']).reshape(-1)
    ops.fold_basis(S, Bp, E, Co, P, Q, F, out, accumulate=False)
    assert rel_err(out.cpu().numpy(), ref) < 3e-6
    ops.fold_basis(S, Bp, E, Co, P, Q, F, out, accumulate=True)
    assert rel_err(out.cpu().numpy(), 2 * ref) < 3e-6


def test_lowrank_basis_of_radial_trunk():
    """Distance-only radial trunks are numerically low rank: a basis of rank <= 31 reproduces the float64 curve to 1e-6 (ops.LOWRANK_TOL),
    and the fp32 kernel outputs at unseen distances stay within fp32 noise of that subspace."""
    from se3_transformer_pytorch_b200 import ops
    from se3_transformer_pytorch_b200.model import RadialFunc
    torch.manual_seed(0)
    rp = RadialFunc(1, 4, 4, edge_dim=0).to(DEV)
    grid = torch.linspace(0, 4, 16384, device=DEV, dtype=torch.float64).unsqueeze(-1)
    basis = ops.lowrank_basis(rp.trunk64(grid))
    assert basis is not None and basis[0] <= 31
    r, V, mean = basis
    d = torch.rand(30000, 1, device=DEV) * 3.9
    g = ops.radial_trunk(d.contiguous(), rp.trunk_params()[None].contiguous(), 1)[0]
    Vf = V.float()
    gc = g - mean.float()
    res = (gc - (gc @ Vf) @ Vf.t()).abs().max() / g.abs().max()
    assert float(res) < 5e-6
    # unstructured samples do not factor: the caller falls back to the direct kernel
    assert ops.lowrank_basis(torch.randn(4096, 128, device=DEV, dtype=torch.float64)) is None


def test_pairwise_tc_headline_width_matches_simt():
    """BASELINE cfg2 widths (C_in = C_out = 512, degree 3 -> 3) on a small edge set: tensor-core vs SIMT fp32."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 512, 7):
        pytest.skip('tensor-core path needs sm_90')
    torch.manual_seed(0)
    b, n, k, C, di, do = 1, 24, 8, 512, 3, 3
    E, P, Q, F = b * n * k, 7, 7, 7
    x = torch.randn(b, n, C, Q, device=DEV)
    idx = torch.randint(0, n, (b, n, k), device=DEV)
    Bm = torch.randn(E * P * Q * F, device=DEV)
    g = torch.randn(E, 128, device=DEV).abs()
    W3 = torch.randn(C * C * F, 128, device=DEV) / 128 ** 0.5
    b3 = 0.1 * torch.randn(C * C * F, device=DEV)
    T = ops.tbuild(x, idx, Bm, di, do)
    ref = torch.empty(E, C, P, device=DEV)
    ops.pairwise_simt(g, W3, b3, T, E, C, C, F, P, ref, accumulate=False)
    out = torch.empty(E, C, P, device=DEV)
    ops.pairwise_tc(g, ops.pack_w3(W3, b3, C, C, F), T, E, C, C, F, P, out, accumulate=False)
    assert rel_err(out.cpu().numpy(), ref.cpu().numpy()) < 2e-5
    # linearity in T (size independent property): out(2T) == 2 out(T)
    out2 = torch.empty(E, C, P, device=DEV)
    ops.pairwise_tc(g, ops.pack_w3(W3, b3, C, C, F), 2 * T, E, C, C, F, P, out2, accumulate=False)
    assert rel_err(out2.cpu().numpy(), 2 * out.cpu().numpy()) < 1e-6


# ------------------------------------------------------------------ K5
@pytest.mark.parametrize('M,Dh,H,K,opts', [
    (1, 8, 2, 5, dict(self_kv=True)), (3, 24, 8, 8, dict(self_kv=True, mask=True)), (7, 64, 8, 16, dict(self_kv=True, mask=True)),
    (5, 16, 4, 33, dict()), (1, 8, 2, 4, dict(self_kv=True, null=True, G=3, mask=True)), (3, 8, 4, 6, dict(one_headed=True, self_kv=True, null=True)),
    (3, 8, 2, 6, dict(lin_keys=True, self_kv=True, mask=True)),
])
def test_attention(M, Dh, H, K, opts):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(8)
    b, n = 2, 9
    kvh = 1 if opts.get('one_headed') else H
    Ckv = kvh * Dh
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    q = f(b, n, H * Dh, M)
    v = f(b, n, K, Ckv, M)
    idx = rng.integers(0, n, (b, n, K))
    if opts.get('lin_keys'):
        k_nodes = f(b, n, Ckv, M)
        k = k_nodes[np.arange(b)[:, None, None], idx]
    else:
        k = f(b, n, K, Ckv, M)
    nmask = (rng.random((b, n, K)) < 0.6) if opts.get('mask') else None
    kd, vd = k, v
    kw = {}
    if opts.get('self_kv'):
        sk, sv = f(b, n, Ckv, M), f(b, n, Ckv, M)
        kd = np.concatenate([sk[:, :, None], kd], 2); vd = np.concatenate([sv[:, :, None], vd], 2)
        kw.update(self_k=cu(sk), self_v=cu(sv))
    if opts.get('null'):
        nk, nv = f(Ckv, M), f(Ckv, M)
        kd = np.concatenate([np.broadcast_to(nk, (b, n, 1, Ckv, M)), kd], 2)
        vd = np.concatenate([np.broadcast_to(nv, (b, n, 1, Ckv, M)), vd], 2)
        kw.update(null_k=cu(nk), null_v=cu(nv))
    if opts.get('G'):
        gk, gv = f(b, opts['G'], Ckv, M), f(b, opts['G'], Ckv, M)
        kd = np.concatenate([np.broadcast_to(gk[:, None], (b, n, opts['G'], Ckv, M)), kd], 2)
        vd = np.concatenate([np.broadcast_to(gv[:, None], (b, n, opts['G'], Ckv, M)), vd], 2)
        kw.update(global_k=cu(gk), global_v=cu(gv))
    J = kd.shape[2]
    scale = Dh ** -0.5
    qh = q.reshape(b, n, H, Dh, M).astype(np.float64)
    kh = np.broadcast_to(kd.reshape(b, n, J, kvh, Dh, M), (b, n, J, H, Dh, M)) if kvh == 1 else kd.reshape(b, n, J, H, Dh, M)
    vh = np.broadcast_to(vd.reshape(b, n, J, kvh, Dh, M), (b, n, J, H, Dh, M)) if kvh == 1 else vd.reshape(b, n, J, H, Dh, M)
    sim = np.einsum('bihdm,bijhdm->bihj', qh, kh.astype(np.float64)) * scale
    if nmask is not None:
        mk = np.concatenate([np.ones((b, n, J - K), dtype=bool), nmask], -1)[:, :, None]
        sim = np.where(mk, sim, -np.finfo(np.float32).max)
    sim = sim - sim.max(-1, keepdims=True)
    a = np.exp(sim); a /= a.sum(-1, keepdims=True)
    ref = np.einsum('bihj,bijhdm->bihdm', a, vh.astype(np.float64)).reshape(b, n, H * Dh, M)
    got = ops.attention(cu(q), cu(k_nodes) if opts.get('lin_keys') else cu(k), cu(v), heads=H, dim_head=Dh, scale=scale,
                        nmask=None if nmask is None else cu(nmask), k_idx=cu(idx) if opts.get('lin_keys') else None,
                        kv_heads=kvh, **kw).cpu().numpy()
    assert rel_err(got, ref) < 5e-6


@pytest.mark.parametrize('M,gelu', [(1, True), (3, True), (7, True), (5, False)])
def test_norm_se3(M, gelu):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(10)
    x = rng.standard_normal((2, 9, 12, M)).astype(np.float32)
    x[0, 0, 0] = 0.0                                            # zero vector: norm clamps to eps, output 0
    scale = (1 + 0.1 * rng.standard_normal((1, 1, 12))).astype(np.float32)
    P = {'transform.0.scale': scale.astype(np.float64)}
    ref = O.norm_se3({'0': x.astype(np.float64)}, P, '', nonlin=O.gelu if gelu else (lambda t: t))['0']
    got = ops.norm_se3(cu(x), cu(scale), 1e-12, gelu).cpu().numpy()
    assert rel_err(got, ref) < 2e-6
    assert np.all(got[0, 0, 0] == 0)


def test_errors_are_loud():
    from se3_transformer_pytorch_b200 import ops
    with pytest.raises(RuntimeError, match='k must be'):
        ops.knn(torch.randn(1, 4, 3, device=DEV), 9, 1e5)
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.knn(torch.randn(1, 4, 3), 2, 1e5)
    # mask shapes (ADVICE r1): [n, n] / [1, n, n] broadcast over the batch, anything else is refused (not read out of bounds)
    c = torch.randn(2, 6, 3, device=DEV)
    nm = torch.rand(6, 6, device=DEV) > 0.3
    a = ops.knn(c, 3, 1e5, neighbor_mask=nm)
    b_ = ops.knn(c, 3, 1e5, neighbor_mask=nm.unsqueeze(0).expand(2, 6, 6).contiguous())
    assert all(torch.equal(x, y) for x, y in zip(a, b_))
    with pytest.raises(ValueError, match='neighbor_mask'):
        ops.knn(c, 3, 1e5, neighbor_mask=torch.ones(3, 6, 6, dtype=torch.bool, device=DEV))
    with pytest.raises(ValueError, match='node_mask'):
        ops.knn(c, 3, 1e5, node_mask=torch.ones(6, dtype=torch.bool, device=DEV))
