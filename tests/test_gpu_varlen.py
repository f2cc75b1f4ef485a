"""Packed batches of clouds of different sizes on the GPU (SE3Transformer.forward_packed, ops.knn with seqlens): the segmented neighbour
search against the padded one per cloud (bit for bit), the whole model against the real reference run once per cloud and against a
per-cloud loop of forward(), equivariance per cloud, independence of the clouds and the edge count."""
import numpy as np
import pytest
import torch

from helpers import GOLDEN, rel_err
from detfill import fill_state_dict
from varlen_helpers import VARLEN_CASES, load_varlen, varlen_outputs, per_cloud_errors, cloud_slices

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items()} if isinstance(res, dict) else res.cpu().numpy()


def _band(n, w):
    i = torch.arange(n)
    return ((i[:, None] - i[None]).abs() <= w) & (i[:, None] != i[None])


# ------------------------------------------------------------------ segmented neighbour search
KNN_CASES = [
    dict(lens=[33, 5, 17, 2], k=8),                                   # n_c - 1 < k, and a cloud of 2
    dict(lens=[2, 4097, 3], k=16),                                    # the largest cloud the sort takes
    dict(lens=[40, 12, 25], k=6, causal=True),
    dict(lens=[30, 9, 21], k=5, radius=1.0),
    dict(lens=[24, 7, 16], k=6, nbr=True),
    dict(lens=[20, 11, 16], k=3, sparse=[1, 3, 2]),                   # bonded counts 2, 6, 4: k_c differs per cloud
    dict(lens=[300], k=16),                                           # B = 1
    dict(lens=[2048] * 40, k=16),                                     # T = 81920 > 65535 CTAs in one grid dimension
]


@pytest.mark.parametrize('case', KNN_CASES, ids=lambda c: ','.join(f'{k}={v if k != "lens" else len(v)}' for k, v in c.items()))
def test_knn_packed_matches_padded_knn_per_cloud(case):
    from se3_transformer_pytorch_b200 import ops
    lens, k = case['lens'], case['k']
    g = torch.Generator().manual_seed(5)
    coors = torch.randn(sum(lens), 3, generator=g).to(DEV)
    radius, causal = case.get('radius', 1e5), case.get('causal', False)
    nbr = [torch.rand(n, n, generator=g) < 0.5 for n in lens] if case.get('nbr') else None
    adj = [_band(n, w) for n, w in zip(lens, case['sparse'])] if case.get('sparse') else None
    ks = [min(k + (int(a.sum(-1).max()) if adj else 0), n - 1) for n, a in zip(lens, adj or [None] * len(lens))]
    flat = lambda ms: None if ms is None else torch.cat([m.reshape(-1) for m in ms]).to(DEV)
    K = max(ks)
    idx, mask, rel_pos, rel_dist = ops.knn(coors, ks, radius, neighbor_mask=flat(nbr), sparse_adj=flat(adj), causal=causal, seqlens=lens,
                                           K=K)
    assert idx.shape == (sum(lens), K) and rel_pos.shape == (sum(lens), K, 3)
    s = 0
    for c, (n, kc) in enumerate(zip(lens, ks)):
        ref = ops.knn(coors[s:s + n][None], kc, radius, neighbor_mask=None if nbr is None else nbr[c][None].to(DEV),
                      sparse_adj=None if adj is None else adj[c][None].to(DEV), causal=causal)
        rows = slice(s, s + n)
        got = (idx[rows, :kc] - s, mask[rows, :kc], rel_pos[rows, :kc], rel_dist[rows, :kc])
        for name, a, b in zip(('idx', 'mask', 'rel_pos', 'rel_dist'), got, ref):
            assert torch.equal(a, b[0]), (c, name)
        # empty slots: masked copies of slot k_c - 1 (finite values inside the cloud's distance range)
        for t in (idx, rel_pos, rel_dist):
            assert torch.equal(t[rows, kc:], t[rows, kc - 1:kc].expand_as(t[rows, kc:])), c
        assert not mask[rows, kc:].any(), c
        s += n


# ------------------------------------------------------------------ against the reference, once per cloud
def _reference_model(cfg):
    from se3_transformer_pytorch_b200 import SE3Transformer
    model = SE3Transformer(**cfg['ctor'])
    fill_state_dict(model, seed=11)
    return model.to(DEV).eval()


def _run_packed(model, feats, coors, seqlens, pairs, fwd):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    feats = {k: t(v) for k, v in feats.items()} if isinstance(feats, dict) else t(feats)
    return model.forward_packed(feats, t(coors), seqlens, **{k: [t(x) for x in v] for k, v in pairs.items()}, **fwd)


@pytest.mark.parametrize('name', VARLEN_CASES)
def test_forward_packed_matches_reference(name):
    z, cfg, feats, coors, seqlens, pairs = load_varlen(name)
    res = _run_packed(_reference_model(cfg), feats, coors, seqlens, pairs, cfg['fwd'])
    errs = per_cloud_errors(_np(res), varlen_outputs(z), seqlens, cfg['fwd'].get('return_pooled', False))
    assert max(errs) < 1e-4, errs


def test_forward_packed_production_path_matches_reference(monkeypatch):
    """varlen_z128 with the one-GEMM production path forced on for these few edges and the fp32 masters released."""
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    monkeypatch.setenv('SE3B200_LOWRANK_MIN_EDGES', '0')
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_z128')
    d_max = max(float(np.linalg.norm(c[:, None] - c[None], axis=-1).max()) for c in np.split(coors, np.cumsum(seqlens)[:-1]))
    model = _reference_model(cfg)
    model.pack_weights(free_master=True, max_distance=1.1 * d_max)
    ops.PROFILE = []
    try:
        res = _run_packed(model, feats, coors, seqlens, pairs, cfg['fwd'])
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    kinds = {p[0] for p in prof}
    assert 'zgemm' in kinds and 'knn_varlen' in kinds, kinds
    errs = per_cloud_errors(_np(res), varlen_outputs(z), seqlens, False)
    assert max(errs) < 1e-4, errs


# ------------------------------------------------------------------ against forward(), one cloud at a time
LENS = [23, 5, 2, 14]
SMALL = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4)
LOOP_CASES = {
    'tokens_pos': (dict(SMALL, num_tokens=7, num_positions=32), dict(tokens=7)),
    'rotary': (dict(SMALL, rotary_position=True, rotary_rel_dist=True, fourier_encode_dist=True), {}),
    'linkeys': (dict(SMALL, linear_proj_keys=True), {}),
    'onehead_nullkv': (dict(SMALL, one_headed_key_values=True, use_null_kv=True), {}),
    'tiekv': (dict(SMALL, tie_key_values=True), {}),
    'contedges': (dict(SMALL, output_degrees=2, edge_dim=6), dict(edges=6, fwd=dict(return_type=1))),
    'nbrmask': (dict(SMALL, valid_radius=10), dict(neighbor_mask=True)),
    'pooled': (dict(SMALL, output_degrees=2, num_conv_layers=1), dict(fwd=dict(return_pooled=True))),
}


def _random_inputs(ctor, lens, opts, seed=0):
    g = torch.Generator().manual_seed(seed)
    T = sum(lens)
    if opts.get('tokens'):
        feats = torch.randint(0, opts['tokens'], (T,), generator=g)
    else:
        feats = torch.randn(T, ctor['dim'], generator=g)
    coors = torch.randn(T, 3, generator=g)
    pairs = {}
    if opts.get('edges'):
        pairs['edges'] = [torch.randn(n, n, opts['edges'], generator=g) for n in lens]
    if opts.get('neighbor_mask'):
        pairs['neighbor_mask'] = [torch.rand(n, n, generator=g) < 0.6 for n in lens]
    to = lambda t: t.to(DEV)
    return to(feats), to(coors), {k: [to(t) for t in v] for k, v in pairs.items()}


def _per_cloud_forward(model, feats, coors, lens, pairs, fwd):
    """forward() on each cloud alone (batch 1, no mask), outputs concatenated along the node axis (pooled: stacked)."""
    outs, s = [], 0
    for c, n in enumerate(lens):
        kw = {k: v[c][None] for k, v in pairs.items()}
        outs.append(model(feats[s:s + n][None], coors[s:s + n][None], **kw, **fwd))
        s += n
    pooled = fwd.get('return_pooled', False)
    cat = lambda ts: torch.cat([t if pooled else t[0] for t in ts], 0)
    return {d: cat([o[d] for o in outs]) for d in outs[0]} if isinstance(outs[0], dict) else cat(outs)


@pytest.mark.parametrize('name', list(LOOP_CASES))
def test_forward_packed_matches_per_cloud_forward(name):
    from se3_transformer_pytorch_b200 import SE3Transformer
    ctor, opts = LOOP_CASES[name]
    torch.manual_seed(0)
    model = SE3Transformer(**ctor).to(DEV).eval()
    feats, coors, pairs = _random_inputs(ctor, LENS, opts)
    fwd = opts.get('fwd', {})
    packed = model.forward_packed(feats, coors, LENS, **pairs, **fwd)
    loop = _per_cloud_forward(model, feats, coors, LENS, pairs, fwd)
    errs = per_cloud_errors(_np(packed), _np(loop), LENS, fwd.get('return_pooled', False))
    assert max(errs) < 2e-5, errs


HEADLINE_LENS = [1024, 832, 640, 448]


def test_forward_packed_matches_per_cloud_forward_at_headline_width(monkeypatch):
    """Headline widths, depth 1, a protein-like batch.  Both sides run the production path (the low-rank switch-over is forced to
    0 edges so that the 448-node cloud alone takes it too); the packed forward runs first and builds the radial plan over every
    cloud's distances, which the per-cloud forwards then reuse."""
    from se3_transformer_pytorch_b200 import SE3Transformer, ops
    if not ops.tc_supported(DEV, 512, 7):
        pytest.skip('needs sm_90')
    monkeypatch.setenv('SE3B200_LOWRANK_MIN_EDGES', '0')
    torch.manual_seed(0)
    with torch.device(DEV):
        model = SE3Transformer(dim=512, heads=8, dim_head=64, depth=1, num_degrees=4, output_degrees=2, num_neighbors=16).eval()
    feats, coors, _ = _random_inputs(dict(dim=512), HEADLINE_LENS, {}, seed=1)
    ops.PROFILE = []
    try:
        packed = model.forward_packed(feats, coors, HEADLINE_LENS)
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    kinds = {p[0] for p in prof}
    assert 'zgemm' in kinds, kinds
    loop = _per_cloud_forward(model, feats, coors, HEADLINE_LENS, {}, {})
    errs = per_cloud_errors(_np(packed), _np(loop), HEADLINE_LENS, False)
    assert max(errs) < 2e-5, errs


# ------------------------------------------------------------------ equivariance, one rotation per cloud
def _rotation(g):
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q.float()


def test_forward_packed_is_equivariant_per_cloud():
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    model = SE3Transformer(dim=64, depth=1, attend_self=True, num_neighbors=4, num_degrees=2, output_degrees=2).to(DEV).eval()
    lens = [20, 7, 13]
    g = torch.Generator().manual_seed(2)
    R = [torch.from_numpy(np.load(f'{GOLDEN}/rot_15_0_45.npz')['R']).float()] + [_rotation(g) for _ in lens[1:]]
    feats, coors, _ = _random_inputs(dict(dim=64), lens, {}, seed=3)
    per_node_R = torch.cat([r.expand(n, 3, 3) for r, n in zip(R, lens)]).to(DEV)          # [T, 3, 3]
    rotated = model.forward_packed(feats, torch.einsum('ti,tij->tj', coors, per_node_R), lens)
    plain = model.forward_packed(feats, coors, lens)
    expect1 = torch.einsum('tci,tij->tcj', plain['1'], per_node_R)
    for sl in cloud_slices(lens, False):
        for got, want in ((rotated['1'][sl], expect1[sl]), (rotated['0'][sl], plain['0'][sl])):
            scale = want.abs().max().item()
            assert (got - want).abs().max().item() / scale < 1e-5


# ------------------------------------------------------------------ independence of the clouds
def test_clouds_are_independent_and_order_free():
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    model = SE3Transformer(**dict(SMALL, output_degrees=2)).to(DEV).eval()
    lens = [23, 5, 17, 9]
    feats, coors, _ = _random_inputs(SMALL, lens, {}, seed=4)
    base = model.forward_packed(feats, coors, lens)
    # change cloud 1 (nodes 23 .. 27): coordinates and features
    feats2, coors2 = feats.clone(), coors.clone()
    feats2[23:28] = torch.randn(5, SMALL['dim'], device=DEV)
    coors2[23:28] = 3 * torch.randn(5, 3, device=DEV)
    changed = model.forward_packed(feats2, coors2, lens)
    slices = cloud_slices(lens, False)
    identical = []
    for c, sl in enumerate(slices):
        if c == 1:
            assert rel_err(changed['0'][sl].cpu().numpy(), base['0'][sl].cpu().numpy()) > 1e-3
            continue
        for d in base:
            assert rel_err(changed[d][sl].cpu().numpy(), base[d][sl].cpu().numpy()) < 1e-6, (c, d)
            identical.append(torch.equal(changed[d][sl], base[d][sl]))
    print(f'other clouds bit-identical after changing cloud 1: {all(identical)}')
    # permuting the clouds permutes the outputs
    order = [2, 0, 3, 1]
    perm = torch.cat([torch.arange(sl.start, sl.stop) for sl in (slices[c] for c in order)]).to(DEV)
    permuted = model.forward_packed(feats[perm], coors[perm], [lens[c] for c in order])
    for d in base:
        assert rel_err(permuted[d].cpu().numpy(), base[d][perm].cpu().numpy()) < 1e-6, d


def test_packed_forward_builds_only_the_real_edges():
    """sum_c n_c K edges (K = max k_c), not B max(n_c) K as a padded batch would."""
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    model = SE3Transformer(**dict(SMALL, num_neighbors=16)).to(DEV).eval()
    feats, coors, _ = _random_inputs(SMALL, HEADLINE_LENS, {}, seed=5)
    seen = {}
    hook = model.conv_in.register_forward_pre_hook(lambda m, a: seen.update(idx=a[1][0]))
    try:
        model.forward_packed(feats, coors, HEADLINE_LENS)
    finally:
        hook.remove()
    assert tuple(seen['idx'].shape) == (1, sum(HEADLINE_LENS), 16)
    assert seen['idx'].numel() == 47104 < len(HEADLINE_LENS) * max(HEADLINE_LENS) * 16 == 65536
