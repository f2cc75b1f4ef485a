"""Clouds of more than 4097 points through SE3Transformer.forward, where the neighbour search walks each row in tiles of 4096
columns and merges every tile into a running list of the best next_pow2(k) keys.

  * the search against the numpy oracle, bit for bit (indices, masks, rel_pos, rel_dist), with node masks, valid_radius, causal,
    neighbor_mask, bonded neighbours and lattice ties across tile boundaries; at n = 70 000 against a chunked torch restatement;
  * the model against reference fixtures at n ~ 4500 (tests/golden/gen_golden_large.py);
  * a cloud made of far-apart parts of <= 4097 points against forward() on each part alone, which runs the whole-row search:
    at headline widths on the production path, and with every dense pair input of the reference API at n ~ 10^4;
  * rotation and permutation equivariance, and the errors for k > 4096 and for forward_packed beyond its cap.
"""

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_case, rel_err, case_inputs, case_outputs, assert_graph_equal
from oracle import se3_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def lattice(n, rng):
    """n distinct points of an integer lattice in random order: every distance repeats, and equal distances land in
    different tiles and around the k-th slot."""
    side = int(np.ceil(n ** (1 / 3))) + 1
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3)
    return g[rng.permutation(len(g))[:n]].astype(np.float32)


# ------------------------------------------------------------------ the tiled search
KNN_CASES = [
    dict(n=4097, k=16),                                   # the longest row that is sorted whole
    dict(n=4098, k=1),                                    # two tiles, the second holding one column
    dict(n=4098, k=4096),                                 # the longest running list
    dict(n=4099, k=16, causal=True),
    dict(n=5000, k=4096, lattice=True),
    dict(b=2, n=5000, k=16, ragged=True, radius=0.05),
    dict(n=5000, k=16, nbr=True),
    dict(n=8193, k=10, sparse=3),                         # banded bonded neighbours: k = 10 + 6
    dict(n=8193, k=16, lattice=True),
    dict(n=12289, k=64, lattice=True),
]


@pytest.mark.parametrize('case', KNN_CASES, ids=lambda c: '-'.join(f'{k}{v}' for k, v in c.items()))
def test_tiled_knn_matches_oracle_bit_for_bit(case):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(case['n'] + case['k'])
    b, n, k = case.get('b', 1), case['n'], case['k']
    if case.get('lattice'):
        coors = np.stack([lattice(n, rng) for _ in range(b)])
    else:
        coors = rng.standard_normal((b, n, 3)).astype(np.float32)
    mask = np.ones((b, n), dtype=bool)
    if case.get('ragged'):
        mask[0, -5:] = False
        mask[1, -4200:] = False                            # masked nodes in both tiles of every row
    nbr = (rng.random((b, n, n)) < 0.5) if case.get('nbr') else None
    sparse = None
    if case.get('sparse'):
        i = np.arange(n)
        sparse = ((np.abs(i[:, None] - i[None]) <= case['sparse']) & (i[:, None] != i[None]))[None]
    radius = case.get('radius', 1e5)
    g = O.neighbor_graph(coors, mask, num_neighbors=k, valid_radius=radius, causal=case.get('causal', False), sparse_adj=sparse,
                         neighbor_mask=nbr)
    kk = g['idx'].shape[-1]
    assert kk == k + (2 * case['sparse'] if sparse is not None else 0)
    idx, nm, rel_pos, rel_dist = ops.knn(cu(coors), kk, radius, node_mask=cu(mask), neighbor_mask=None if nbr is None else cu(nbr),
                                         sparse_adj=None if sparse is None else cu(sparse), causal=case.get('causal', False))
    assert np.array_equal(idx.cpu().numpy(), g['idx'])
    assert np.array_equal(nm.cpu().numpy(), g['mask'])
    assert np.array_equal(rel_pos.cpu().numpy(), g['rel_pos'])
    assert np.array_equal(rel_dist.cpu().numpy(), g['rel_dist'])


def torch_knn(coors, k, chunk=512):
    """The search restated with torch on the GPU for one cloud coors [n, 3]: explicit dx, dy, dz, one op per multiply and add
    (no contraction into FMA), keys (bits(distance) << 32) | column on the self-removed grid, sorted.  Returns idx, rel_pos,
    rel_dist as ops.knn does for b = 1."""
    n = coors.shape[0]
    cols = torch.arange(n, device=coors.device)
    out = []
    for s in range(0, n, chunk):
        rows = cols[s:s + chunk]
        dx = coors[rows, 0:1] - coors[None, :, 0]
        dy = coors[rows, 1:2] - coors[None, :, 1]
        dz = coors[rows, 2:3] - coors[None, :, 2]
        d = torch.sqrt(dx * dx + dy * dy + dz * dz)
        jc = cols[None, :] - (cols[None, :] > rows[:, None]).long()
        key = (d.view(torch.int32).long() << 32) | jc
        key = key.masked_fill(cols[None, :] == rows[:, None], torch.iinfo(torch.int64).max)
        top = key.sort(dim=1).values[:, :k]
        jc = top & 0xffffffff
        j = jc + (jc >= rows[:, None]).long()
        g = lambda t: t.gather(1, j)
        out.append((j, torch.stack((g(dx), g(dy), g(dz)), -1), g(d)))
    return tuple(torch.cat(t)[None] for t in zip(*out))


def test_tiled_knn_at_70000_points_matches_torch_restatement():
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(70)
    n, k = 70000, 16
    coors = torch.randn(1, n, 3, generator=g).to(DEV)
    idx, nm, rel_pos, rel_dist = ops.knn(coors, k, 1e5)
    ref_idx, ref_pos, ref_dist = torch_knn(coors[0], k)
    assert torch.equal(idx, ref_idx)
    assert bool(nm.all())
    assert torch.equal(rel_pos, ref_pos)
    assert torch.equal(rel_dist, ref_dist)


# ------------------------------------------------------------------ the model at n > 4097
def _run(model, feats, coors, mask=None, **kw):
    """model(...) under the launch profile: (output, the set of kernel kinds launched)."""
    from se3_transformer_pytorch_b200 import ops
    ops.PROFILE = []
    try:
        out = model(feats, coors, mask, **kw)
        torch.cuda.synchronize()
    finally:
        prof, ops.PROFILE = ops.PROFILE, None
    return out, {p[0] for p in prof}


@pytest.mark.parametrize('name', ['large_type1', 'large_bonded_b2'])
def test_model_matches_large_reference_fixture(name):
    from se3_transformer_pytorch_b200 import SE3Transformer
    from detfill import fill_state_dict
    z, cfg = load_case(name)
    model = SE3Transformer(**cfg['ctor'])
    fill_state_dict(model, seed=11)
    model = model.to(DEV).eval()
    feats, coors, mask, extra = case_inputs(z)
    cap = {}
    hook = model.conv_in.register_forward_pre_hook(lambda m, a, k: cap.update(edge_info=a[1], rel_dist=k['rel_dist']), with_kwargs=True)
    try:
        res = model(cu(feats), cu(coors), cu(mask), **{k: cu(v) for k, v in extra.items()}, **cfg['fwd'])
    finally:
        hook.remove()
    idx, nmask, _ = cap['edge_info']
    assert_graph_equal(idx.cpu().numpy(), nmask.cpu().numpy(), cap['rel_dist'].cpu().numpy(), z['cap/graph/neighbor_indices'],
                       z['cap/graph/neighbor_mask'], z['cap/graph/rel_dist'])
    err = rel_err(res.cpu().numpy(), case_outputs(z))
    assert err < 1e-4, f'rel err {err:.3e}'


def _rot():
    return torch.from_numpy(np.load(f'{GOLDEN}/rot_15_0_45.npz')['R']).float()


def _assert_parts_match(out, parts, bounds, tol=0.0):
    """out[:, s:e] against each part's own output: bit-identical (tol = 0), or within tol relative."""
    for d in out:
        for part, (s, e) in zip(parts, bounds):
            err = rel_err(out[d][:, s:e].cpu().numpy(), part[d].cpu().numpy())
            assert (torch.equal(out[d][:, s:e], part[d]) if tol == 0 else err < tol), f'degree {d}, nodes {s}:{e}: rel err {err:.3e}'


def test_two_far_apart_clouds_match_each_alone_at_headline_width():
    """One cloud of 2 x 2100 points (a cloud and a rotated, permuted copy of it, 1e4 apart): with k = 16 no neighbour crosses
    between the halves, so each half's output is forward() on that half alone (same coordinates), whose rows are sorted whole."""
    from se3_transformer_pytorch_b200 import SE3Transformer, ops
    if not ops.tc_supported(DEV, 512, 7):
        pytest.skip('needs sm_90')
    m = 2100
    g = torch.Generator().manual_seed(11)
    a = torch.randn(m, 3, generator=g)
    b = (a @ _rot())[torch.randperm(m, generator=g)] + torch.tensor([1e4, 0., 0.])
    coors = torch.cat((a, b))[None].to(DEV)
    feats = torch.randn(1, 2 * m, 512, generator=g).to(DEV)
    torch.manual_seed(0)
    with torch.device(DEV):
        model = SE3Transformer(dim=512, heads=8, dim_head=64, depth=1, num_degrees=4, output_degrees=2, num_neighbors=16).eval()
    model.pack_weights(free_master=True, max_distance=16.0)
    out, kinds = _run(model, feats, coors)
    assert kinds & {'zgemm', 'pairwise_lr'} and 'rotgather' in kinds, kinds          # the production dispatch
    assert not kinds & {'pairwise_tc', 'pairwise_simt'}, kinds
    parts = []
    for s, e in ((0, m), (m, 2 * m)):
        part, kinds = _run(model, feats[:, s:e].contiguous(), coors[:, s:e].contiguous())
        assert kinds & {'zgemm', 'pairwise_lr'} and 'rotgather' in kinds, kinds
        parts.append(part)
    _assert_parts_match(out, parts, ((0, m), (m, 2 * m)))


def test_dense_pair_inputs_at_10k_points_match_each_part_alone():
    """The torch glue that stays dense [b, n, n] as in the reference (bonded neighbours and their 2-hop adjacency, hop-count
    embeddings, edge-token gather, neighbor_mask) at n = 10 200: three parts of 3400 points 1e4 apart, every pair input block
    diagonal, so each part's output is forward() on that part alone.  The graph is the same; the outputs agree to 1e-6 and not
    bit for bit because at width 16 LinearSE3 runs on torch.matmul, whose cuBLAS kernel depends on the row count.  The peak
    device memory of the forward is printed."""
    from se3_transformer_pytorch_b200 import SE3Transformer
    m, P = 3400, 3
    n = m * P
    g = torch.Generator(device=DEV).manual_seed(12)
    coors = torch.cat([torch.randn(m, 3, generator=g, device=DEV) * 10 + torch.tensor([1e4 * p, 0., 0.], device=DEV)
                       for p in range(P)])[None]
    feats = torch.randn(1, n, 16, generator=g, device=DEV)
    block = torch.zeros(n, n, dtype=torch.bool, device=DEV)
    for p in range(P):
        block[p * m:(p + 1) * m, p * m:(p + 1) * m] = True
    i = torch.arange(n, device=DEV)
    adj = block & ((i[:, None] - i[None]).abs() == 1)                                 # chains: 4 bonded within 2 hops
    nbr = (block & (torch.rand(n, n, generator=g, device=DEV) < 0.7))[None]
    edges = torch.randint(0, 4, (1, n, n), generator=g, device=DEV)
    torch.manual_seed(0)
    model = SE3Transformer(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, num_neighbors=8,
                           attend_sparse_neighbors=True, max_sparse_neighbors=8, num_adj_degrees=2, adj_dim=4, num_edge_tokens=4,
                           edge_dim=4).to(DEV).eval()
    kw = lambda s, e: dict(adj_mat=adj[s:e, s:e].contiguous(), edges=edges[:, s:e, s:e].contiguous(),
                           neighbor_mask=nbr[:, s:e, s:e].contiguous())
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = model(feats, coors, **kw(0, n))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bounds = [(p * m, (p + 1) * m) for p in range(P)]
    parts = [model(feats[:, s:e].contiguous(), coors[:, s:e].contiguous(), **kw(s, e)) for s, e in bounds]
    _assert_parts_match(out, parts, bounds, tol=1e-6)
    pair_bytes = sum(t.numel() * t.element_size() for t in (adj, nbr, edges))
    print(f'n = {n} on {torch.cuda.get_device_name()}: forward peak {peak / 1e9:.2f} GB above {pair_bytes / 1e9:.2f} GB of pair inputs')


def _small_model(**kw):
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    return SE3Transformer(**{**dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, output_degrees=2, num_neighbors=16),
                             **kw}).to(DEV).eval()


def test_equivariance_at_5000_points():
    """f(x R) == f(x) R for the type-1 output, R = rot(15, 0, 45), within 1e-5 relative to the output scale."""
    model = _small_model()
    g = torch.Generator().manual_seed(13)
    n = 5000
    feats = torch.randn(1, n, 16, generator=g).to(DEV)
    coors = torch.randn(1, n, 3, generator=g).to(DEV)
    R = _rot().to(DEV)
    out1 = model(feats, coors @ R, return_type=1)
    out2 = model(feats, coors, return_type=1) @ R
    scale = out2.abs().max().item()
    assert (out1 - out2).abs().max().item() / scale < 1e-5


def test_permutation_equivariance_at_5000_points():
    model = _small_model()
    g = torch.Generator().manual_seed(14)
    n = 5000
    feats = torch.randn(1, n, 16, generator=g).to(DEV)
    coors = torch.randn(1, n, 3, generator=g).to(DEV)
    perm = torch.randperm(n, generator=g).to(DEV)
    out = model(feats, coors)
    outp = model(feats[:, perm], coors[:, perm])
    for d in out:
        assert rel_err(outp[d].cpu().numpy(), out[d][:, perm].cpu().numpy()) < 1e-6, d


def test_more_than_4096_neighbours_is_refused():
    from se3_transformer_pytorch_b200 import ops
    coors = torch.randn(1, 5000, 3, device=DEV)
    with pytest.raises(RuntimeError, match='k = 4097 neighbours exceeds 4096'):
        ops.knn(coors, 4097, 1e5)
    # the default num_neighbors = inf asks for n - 1 neighbours
    with pytest.raises(RuntimeError, match='k = 4999 neighbours exceeds 4096'):
        _small_model(num_neighbors=float('inf'))(torch.randn(1, 5000, 16, device=DEV), coors)


def test_forward_packed_keeps_its_cap():
    model = _small_model()
    with pytest.raises(ValueError, match='4097'):
        model.forward_packed(torch.randn(4098, 16, device=DEV), torch.randn(4098, 3, device=DEV), [4098])
