"""Every kernel at the limits INTEGRATION.md documents: degrees up to 5 (2l+1 = 11 components), up to 4096 neighbours, and
dim_head * (2l+1) up to 1024.  Kernels are checked against the float64 restatements of test_gpu_kernels.py / test_gpu_zgemm.py;
attention is compared per (node, head) row, relative to that row's own scale.  The models of 5 and 6 degrees run against
reference-generated fixtures, and one production-path model attends over ~1000 neighbours."""
import numpy as np
import pytest
import torch

from helpers import DEG_CASES, GOLDEN, attention_reference, load_case, rel_err, run_zgemm
from test_gpu_kernels import (test_norm_se3 as _norm_case, test_pairwise_lowrank_matches_fp64 as _pairwise_lr_case,
                              test_pairwise_simt as _pairwise_simt_case, test_pairwise_tc_matches_fp64 as _pairwise_tc_case)
from test_gpu_model import build_model, check_outputs, run_model
from test_gpu_zgemm import (DEV, test_linear_tc_matches_fp64 as _linear_tc_case, test_rotate_pool as _rotate_pool_case,
                            test_rotgather as _rotgather_case)

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _row_err(got, ref, H):
    """max over (node, head) of max |got - ref| / max |ref| within that row; got, ref [b, n, H*Dh, M]."""
    b, n = ref.shape[:2]
    d = np.abs(np.asarray(got, np.float64) - ref).reshape(b, n, H, -1).max(-1)
    s = np.abs(ref).reshape(b, n, H, -1).max(-1)
    return float((d / np.maximum(s, 1e-30)).max())


def _keys(rng, b, n, M, Ckv, k, v, opts):
    """Prefix keys of opts as kernel kwargs, and keys / values [b,n,J,Ckv,M] in the kernel's order (global, null, self, edges)."""
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    kw, kd, vd = {}, k, v
    if opts.get('self_kv'):
        sk, sv = f(b, n, Ckv, M), f(b, n, Ckv, M)
        kd = np.concatenate([sk[:, :, None], kd], 2); vd = np.concatenate([sv[:, :, None], vd], 2)
        kw.update(self_k=sk, self_v=sv)
    if opts.get('null'):
        nk, nv = f(Ckv, M), f(Ckv, M)
        kd = np.concatenate([np.broadcast_to(nk, (b, n, 1, Ckv, M)), kd], 2)
        vd = np.concatenate([np.broadcast_to(nv, (b, n, 1, Ckv, M)), vd], 2)
        kw.update(null_k=nk, null_v=nv)
    if opts.get('G'):
        gk, gv = f(b, opts['G'], Ckv, M), f(b, opts['G'], Ckv, M)
        kd = np.concatenate([np.broadcast_to(gk[:, None], (b, n, opts['G'], Ckv, M)), kd], 2)
        vd = np.concatenate([np.broadcast_to(gv[:, None], (b, n, opts['G'], Ckv, M)), vd], 2)
        kw.update(global_k=gk, global_v=gv)
    return kw, kd, vd


def _mask(rng, b, n, K, opts):
    if not opts.get('mask'):
        return None
    m = rng.random((b, n, K)) < 0.6
    if opts.get('all_masked_row'):
        m[0, 0] = False                                        # no valid neighbour: prefix keys only, or uniform weights
    return m


# ------------------------------------------------------------------ se3_attn_fwd: one case per register template NL = ceil(L / 32)
ATTN_CASES = [
    # (dim_head, M, H, K, b, n, opts)                                                        L = dim_head * M -> NL template
    (32, 1, 2, 7, 2, 5, dict(self_kv=True)),                                                  # 32 -> 1
    (64, 1, 3, 9, 2, 5, dict(mask=True, all_masked_row=True)),                                # 64 -> 2
    (24, 5, 2, 6, 2, 5, dict(self_kv=True, null=True, G=2)),                                  # 120 -> 4
    (64, 3, 4, 10, 2, 5, dict(one_headed=True, self_kv=True, mask=True)),                     # 192 -> 6
    (32, 7, 2, 8, 2, 5, dict(G=3, mask=True)),                                                # 224 -> 8
    (64, 5, 2, 12, 2, 5, dict(self_kv=True, null=True, mask=True, all_masked_row=True)),      # 320 -> 10
    (64, 7, 5, 6, 2, 5, dict(one_headed=True, null=True)),                                    # 448 -> 14 (5 heads: a partial block)
    (64, 9, 2, 5, 2, 5, dict(self_kv=True, mask=True)),                                       # 576 -> 18
    (64, 11, 2, 7, 2, 5, dict(self_kv=True, null=True, mask=True, all_masked_row=True)),      # 704 -> 22
    (93, 11, 2, 5, 2, 5, dict(self_kv=True, G=2, mask=True)),                                 # 1023 -> 32
    (8, 3, 2, 4096, 1, 2, dict(self_kv=True, null=True, mask=True)),                          # 4098 keys: 64 KB of logits
]


@pytest.mark.parametrize('Dh,M,H,K,b,n,opts', ATTN_CASES, ids=lambda v: str(v) if not isinstance(v, dict) else '-'.join(v))
def test_attention_templates_match_fp64(Dh, M, H, K, b, n, opts):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(Dh * 1000 + M * 10 + K)
    kvh = 1 if opts.get('one_headed') else H
    Ckv = kvh * Dh
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    q, k, v = f(b, n, H * Dh, M), f(b, n, K, Ckv, M), f(b, n, K, Ckv, M)
    nmask = _mask(rng, b, n, K, opts)
    kw, kd, vd = _keys(rng, b, n, M, Ckv, k, v, opts)
    scale = Dh ** -0.5
    ref = attention_reference(q, kd, vd, nmask, H, Dh, kvh, scale)
    got = ops.attention(cu(q), cu(k), cu(v), heads=H, dim_head=Dh, scale=scale, kv_heads=kvh,
                        nmask=None if nmask is None else cu(nmask), **{key: cu(t) for key, t in kw.items()}).cpu().numpy()
    err = _row_err(got, ref, H)
    assert err < 1e-5, f'rel err per row {err:.3e}'


# ------------------------------------------------------------------ se3_attn_aligned_fwd: every degree and register width, long lists
def _aligned_case(M, Dh, H, K, b, n, k_aligned, opts, seed):
    """Keys / values in the edge frames (component major, as zgemm writes them) against float64: rotate to the global frame in
    float64, then attend as attention_reference does."""
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(seed)
    kvh = 1 if opts.get('one_headed') else H
    Ckv = kvh * Dh
    E = b * n * K
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    q, kp, vp = f(b, n, H * Dh, M), f(b, n, K, M, Ckv), f(b, n, K, M, Ckv)
    Dm = np.linalg.qr(rng.standard_normal((E, M, M)))[0].astype(np.float32)
    rot = lambda t: np.einsum('epn,enc->ecp', Dm.astype(np.float64), t.reshape(E, M, Ckv).astype(np.float64)).reshape(b, n, K, Ckv, M)
    vg = rot(vp)
    kg = rot(kp) if k_aligned else f(b, n, K, Ckv, M)          # k_aligned = False: keys already in the global frame
    nmask = _mask(rng, b, n, K, opts)
    kw, kd, vd = _keys(rng, b, n, M, Ckv, kg, vg, opts)
    scale = Dh ** -0.5
    ref = attention_reference(q, kd, vd, nmask, H, Dh, kvh, scale)
    got = ops.attention(cu(q), cu(kp if k_aligned else kg.astype(np.float32)), cu(vp), heads=H, dim_head=Dh, scale=scale,
                        kv_heads=kvh, nmask=None if nmask is None else cu(nmask), D=cu(Dm), k_aligned=k_aligned,
                        **{key: cu(t) for key, t in kw.items()}).cpu().numpy()
    err = _row_err(got, ref, H)
    assert err < 1e-5, f'rel err per row {err:.3e}'


@pytest.mark.parametrize('M', [3, 5, 7, 9, 11])
@pytest.mark.parametrize('Dh', [8, 64, 100, 128])               # register slots per lane ND = 1, 2, 4, 4
def test_aligned_attention_degrees_and_widths(M, Dh):
    k_aligned = (M // 2 + Dh // 8) % 2 == 0                       # both ways for every M and every dim_head
    opts = [dict(self_kv=True), dict(mask=True, all_masked_row=True), dict(self_kv=True, null=True, mask=True),
            dict(one_headed=True, self_kv=True, mask=True)][(M // 2 + Dh) % 4]
    _aligned_case(M, Dh, 3, 5, 2, 4, k_aligned, opts, seed=M * 1000 + Dh)


ALIGNED_LONG = [
    # (M, Dh, H, K, b, n, k_aligned, opts)
    (11, 100, 2, 33, 1, 3, True, dict(self_kv=True, mask=True)),                 # one edge past the first D tile
    (5, 64, 2, 64, 1, 3, False, dict(mask=True, all_masked_row=True)),            # two whole tiles
    (7, 16, 6, 300, 1, 3, True, dict(self_kv=True, null=True, mask=True)),        # 6 heads: a block with two idle warps
    (7, 8, 2, 1000, 1, 2, True, dict(self_kv=True, mask=True)),
    (7, 8, 2, 1000, 1, 2, False, dict(self_kv=True)),
    (3, 8, 6, 4096, 1, 2, True, dict(self_kv=True, null=True, mask=True)),        # 4098 keys: 64 KB of logits
]


@pytest.mark.parametrize('M,Dh,H,K,b,n,k_aligned,opts', ALIGNED_LONG,
                         ids=lambda v: str(v) if not isinstance(v, dict) else '-'.join(v))
def test_aligned_attention_long_neighbour_lists(M, Dh, H, K, b, n, k_aligned, opts):
    _aligned_case(M, Dh, H, K, b, n, k_aligned, opts, seed=K + M)


# ------------------------------------------------------------------ per-node kernels at 9 and 11 components
@pytest.mark.parametrize('M,gelu', [(9, True), (11, False)])
def test_norm_se3_high_degree(M, gelu):
    _norm_case(M, gelu)


@pytest.mark.parametrize('D,Eo,M,nodes,with_res', [(512, 128, 9, 31, True), (64, 256, 11, 40, False)])
def test_linear_tc_high_degree(D, Eo, M, nodes, with_res):
    _linear_tc_case(D, Eo, M, nodes, with_res)


# ------------------------------------------------------------------ pairwise kernels with degree 4 and 5 on either side
@pytest.mark.parametrize('di,do,Ci,Co', [(4, 4, 3, 6), (5, 5, 2, 5), (2, 5, 4, 7), (5, 1, 3, 9), (4, 0, 5, 4)])
def test_pairwise_simt_high_degree(di, do, Ci, Co):
    _pairwise_simt_case(di, do, Ci, Co)


@pytest.mark.parametrize('di,do,Ci,Co,n,k', [(4, 3, 4, 32, 12, 9), (5, 2, 3, 64, 16, 8), (5, 3, 2, 32, 11, 13), (4, 1, 5, 32, 9, 7)])
def test_pairwise_tc_high_degree_input(di, do, Ci, Co, n, k):
    _pairwise_tc_case(di, do, Ci, Co, n, k)


@pytest.mark.parametrize('r,P,di,do', [(15, 7, 4, 3), (31, 5, 5, 2), (20, 3, 4, 1), (15, 7, 5, 3)])
def test_pairwise_lowrank_high_degree_input(r, P, di, do):
    _pairwise_lr_case(r, P, di, do)


# ------------------------------------------------------------------ production-path kernels at degrees 4 and 5
@pytest.mark.parametrize('lo,K,Co,masked,self_add', [(4, 7, 128, True, True), (5, 33, 96, True, False)])
def test_rotate_pool_high_degree(lo, K, Co, masked, self_add):
    _rotate_pool_case(lo, K, Co, masked, self_add)


def test_rotgather_nine_components():
    _rotgather_case(4, 7, 2, 15, 11)


@pytest.mark.parametrize('mode,Co,E,segs', [
    (1, 128, 300, [(8, 9, 4, 4, 16), (4, 11, 5, 5, 32)]),                           # m = 0 components of l = 4 and l = 5
    (3, 256, 200, [(8, 11, 6, 4, 16), (12, 11, 10, 0, 16), (4, 11, 8, 2, 32)]),     # (+m, -m) of l = 5 for m = 1, 5, 3
])
def test_zgemm_high_degree_segments(mode, Co, E, segs):
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, Co, 1):
        pytest.skip('needs sm_90')
    out, ref = run_zgemm(mode, Co, E, segs, seed=Co + mode)
    err = rel_err(out.cpu().numpy(), ref.cpu().numpy())
    assert err < (6e-6 if mode == 3 else 3e-6), f'{err:.3e}'


# ------------------------------------------------------------------ models of 5 and 6 degrees against the reference
_MODELS = {}        # one model per fixture for its three routes (z128_deg6 has 680 M parameters, filled on the host)


@pytest.mark.parametrize('route', ['default', 'force_simt', 'lowrank'])
@pytest.mark.parametrize('name', DEG_CASES)
def test_high_degree_model_matches_reference_golden(name, route):
    """Default dispatch, fp32 SIMT only, and the low-rank dispatch forced on for these few edges.  On the low-rank route the
    pairs with degree_out <= 3 run on the tensor cores (pairwise_lr, where the widths allow it) and those with degree_out >= 4 on
    SIMT; z128_deg6's conv_out (outputs of degree <= 1, 128 channels) runs on the one-GEMM path with inputs up to degree 5."""
    from se3_transformer_pytorch_b200 import ops, switches
    z, cfg = load_case(name)
    if name not in _MODELS:
        _MODELS.clear()
        _MODELS[name] = build_model(cfg)
    model = _MODELS[name]
    sw = dict(default={}, force_simt=dict(force_simt=True), lowrank=dict(lowrank_min_edges=0))[route]
    ops.PROFILE = []
    try:
        with switches.override(**sw):
            res = run_model(model, z, cfg)
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    kinds = {p[0] for p in prof}
    check_outputs(res, z)
    if route == 'force_simt':
        assert not kinds & {'pairwise_tc', 'pairwise_lr', 'zgemm'}, kinds
    if route == 'lowrank':
        assert 'pairwise_simt' in kinds, kinds
        if name != 'deg6':                                     # (16-channel fibers: no tensor-core tile fits)
            assert 'pairwise_lr' in kinds, kinds
        if name == 'z128_deg6':
            assert {'zgemm', 'rotgather', 'rotate_pool'} <= kinds, kinds


# ------------------------------------------------------------------ the production path at ~1000 neighbours and at dim_head 256
def _count_fused(monkeypatch):
    """Counts calls of se3_attn_aligned_fwd (attention with the rotate-back fused)."""
    from se3_transformer_pytorch_b200 import ops
    lib, calls = ops.lib(), []
    fn = lib.se3_attn_aligned_fwd
    monkeypatch.setattr(lib, 'se3_attn_aligned_fwd', lambda *a: calls.append(a[16]) or fn(*a))    # a[16]: K
    return calls


def test_production_path_attends_over_a_thousand_neighbours(monkeypatch):
    """num_neighbors = inf on 1000 points: 999 keys per query, more than the fused attention kernel took when it kept the D of
    all edges in shared memory (965 at degree 3).  Fused == rotate-back + se3_attn_fwd within 1e-5 per degree, and the output is
    rotation-equivariant."""
    from se3_transformer_pytorch_b200 import SE3Transformer, ops, switches
    torch.manual_seed(0)
    with torch.device(DEV):
        model = SE3Transformer(dim=128, heads=2, dim_head=64, depth=1, num_degrees=4, output_degrees=2,
                               num_neighbors=float('inf')).eval()
    n = 1000
    feats = torch.randn(1, n, 128, device=DEV)
    coors = torch.randn(1, n, 3, device=DEV) * 3
    mask = torch.ones(1, n, dtype=torch.bool, device=DEV)
    calls = _count_fused(monkeypatch)
    ops.PROFILE = []
    torch.cuda.reset_peak_memory_stats()
    try:
        with torch.no_grad():
            out = model(feats, coors, mask)
        torch.cuda.synchronize()
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    peak = torch.cuda.max_memory_allocated()
    print(f'1000 points, 999 neighbours, dim 128, 4 degrees: peak {peak / 1e9:.2f} GB')
    kinds = {p[0] for p in prof}
    assert 'zgemm' in kinds, kinds
    assert calls and set(calls) == {n - 1}, calls
    # measured 54-59 GB on an H100 80GB HBM3 (700 W): well above the ~16 GB of edge-level K / V alone; the bound keeps it on the card
    assert peak < 64e9
    fused = len(calls)
    with torch.no_grad(), switches.override(no_attn_rotate=True):
        ref = model(feats, coors, mask)
    assert len(calls) == fused
    for d in ('0', '1'):
        err = rel_err(out[d].cpu().numpy(), ref[d].cpu().numpy())
        assert err < 1e-5, f'degree {d}: fused vs separate rotate-back {err:.3e}'
    R = torch.from_numpy(np.load(f'{GOLDEN}/rot_15_0_45.npz')['R']).float().to(DEV)
    with torch.no_grad():
        out_rot = model(feats, coors @ R, mask)
    assert (out_rot['1'] - out['1'] @ R).abs().max().item() / out['1'].abs().max().item() < 2e-5
    assert (out_rot['0'] - out['0']).abs().max().item() / out['0'].abs().max().item() < 2e-5


def test_production_path_with_wide_heads(monkeypatch):
    """dim_head = 256 (L = 768 at degree 1, inside the documented dim_head * (2l+1) <= 1024): wider than the fused attention
    kernel takes, so the production path rotates back separately and runs se3_attn_fwd; the result matches the oracle."""
    from se3_transformer_pytorch_b200 import SE3Transformer, ops, switches
    from detfill import fill_state_dict, det_inputs
    from oracle import se3_oracle as O
    cfg = dict(dim=128, heads=1, dim_head=256, depth=1, num_degrees=2, output_degrees=2, num_neighbors=6)
    model = SE3Transformer(**cfg)
    fill_state_dict(model, seed=3)
    feats = det_inputs('wide_heads/feats', (1, 20, 128), 1)
    coors = det_inputs('wide_heads/coors', (1, 20, 3), 2)
    mask = np.ones((1, 20), dtype=bool)
    ref = O.se3_transformer_forward({k: v.numpy() for k, v in model.state_dict().items()}, cfg, feats, coors, mask)
    model = model.to(DEV).eval()
    calls = _count_fused(monkeypatch)
    ops.PROFILE = []
    try:
        with torch.no_grad(), switches.override(lowrank_min_edges=0):
            out = model(cu(feats), cu(coors), cu(mask))
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    assert 'zgemm' in {p[0] for p in prof} and not calls
    for d in ref:
        err = rel_err(out[d].cpu().numpy(), ref[d])
        assert err < 1e-4, f'degree {d}: {err:.3e}'
