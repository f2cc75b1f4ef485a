"""Sparse pair inputs of SE3Transformer.forward on the GPU:

  * ops.knn reading sorted column lists (ops.PairRows) against ops.knn on the densified masks, bit for bit, on the
    cases of the tiled-search test plus empty rows, an empty neighbour list and a batch-shared 2-D adjacency;
  * ops.pair_lookup against the dense gathers, -1 for absent pairs;
  * every reference fixture with pair inputs, run with them as torch.sparse_coo (also uncoalesced, with stored zeros): bit for bit
    the dense forward on to_dense(), and within 1e-4 of the fixture;
  * a bonded cloud of 100 000 points (30 parts 1e4 apart) against forward() on each part alone with dense inputs;
  * peak device memory linear in n with sparse pair inputs and with none.
"""
import numpy as np
import pytest
import torch

from helpers import load_case, rel_err, case_inputs, case_outputs
from detfill import fill_state_dict
from test_gpu_large_clouds import KNN_CASES, lattice
from bench_bonded import CTOR, bonded_parts

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------ the search
CSR_CASES = KNN_CASES + [
    dict(b=2, n=3000, k=16, nbr=True, sparse=2, empty_rows=True),     # rows with no allowed and no bonded column
    dict(n=300, k=4, nbr='none', sparse=1),                           # nothing allowed anywhere: an empty neighbour list
    dict(b=3, n=6000, k=8, sparse=4, shared=True, causal=True),       # one [n, n] adjacency for the batch, two tiles
]


@pytest.mark.parametrize('case', CSR_CASES, ids=lambda c: '-'.join(f'{k}{v}' for k, v in c.items()))
def test_knn_column_lists_match_dense_masks_bit_for_bit(case):
    from se3_transformer_pytorch_b200 import ops
    rng = np.random.default_rng(case['n'] + case['k'])
    b, n = case.get('b', 1), case['n']
    if case.get('lattice'):
        coors = np.stack([lattice(n, rng) for _ in range(b)])
    else:
        coors = rng.standard_normal((b, n, 3)).astype(np.float32)
    mask = np.ones((b, n), dtype=bool)
    if case.get('ragged'):
        mask[0, -5:] = False
        mask[1, -4200:] = False
    nbr = None
    if case.get('nbr'):
        nbr = np.zeros((b, n, n), dtype=bool) if case['nbr'] == 'none' else rng.random((b, n, n)) < 0.5
    adj = None
    if case.get('sparse'):
        i = np.arange(n)
        adj = ((np.abs(i[:, None] - i[None]) <= case['sparse']) & (i[:, None] != i[None]))
        adj = adj if case.get('shared') else np.broadcast_to(adj, (b, n, n)).copy()
    if case.get('empty_rows'):
        nbr[:, ::7] = False
        adj[:, ::5] = False
    k = case['k'] + (2 * case['sparse'] if adj is not None else 0)
    k = min(k, n - 1)
    nbr_t = None if nbr is None else cu(nbr)
    adj_t = None if adj is None else cu(adj)
    kw = dict(node_mask=cu(mask), causal=case.get('causal', False))
    radius = case.get('radius', 1e5)
    dense = ops.knn(cu(coors), k, radius, neighbor_mask=nbr_t, sparse_adj=adj_t, **kw)
    rows = lambda t: None if t is None else ops.coo_to_rows(t.to_sparse(), n)
    if adj is not None and case.get('shared'):
        assert rows(adj_t).shared
    sparse = ops.knn(cu(coors), k, radius, neighbor_mask=rows(nbr_t), sparse_adj=rows(adj_t), **kw)
    for a, s in zip(dense, sparse):
        assert torch.equal(a, s)


@pytest.mark.parametrize('shared', [False, True])
def test_pair_lookup_matches_dense_gathers(shared):
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(5)
    b, n, k, e = 2, 700, 24, 3
    shape = (n, n) if shared else (b, n, n)
    nnz = 20000
    ind = torch.stack([torch.randint(0, s, (nnz,), generator=g, device=DEV) for s in shape])
    tokens = torch.sparse_coo_tensor(ind, torch.randint(0, 5, (nnz,), generator=g, device=DEV), shape)
    feats = torch.sparse_coo_tensor(ind, torch.randn(nnz, e, generator=g, device=DEV), (*shape, e))
    idx, *_ = ops.knn(torch.randn(b, n, 3, generator=g, device=DEV), k, 1e5)
    present = torch.sparse_coo_tensor(ind, torch.ones(nnz, dtype=torch.bool, device=DEV), shape).to_dense().expand(b, n, n)
    for t in (tokens, feats):
        rows = ops.coo_to_rows(t, n)
        pos = ops.pair_lookup(rows, idx)
        assert torch.equal(pos == -1, ~present.gather(2, idx))
        v = torch.cat((rows.values, rows.values.new_zeros((1, *rows.values.shape[1:]))))[pos]
        dense = t.to_dense().expand(b, n, n, *t.shape[len(shape):])
        ref = dense.gather(2, idx) if t is tokens else ops.gather_pairs(dense.contiguous(), idx)
        assert torch.equal(v, ref)


# ------------------------------------------------------------------ the model on the reference fixtures
PAIR_CASES = ['edges_sparse', 'adjdeg', 'nbrmask', 'contedges', 'cfg4_b2', 'large_bonded_b2']   # (af2 has no pair inputs)


def messy(t, seed):
    """t as an uncoalesced torch.sparse_coo tensor: every entry split in two summands (bool: repeated), and stored zeros at
    random pairs and on the diagonal."""
    g = torch.Generator().manual_seed(seed)
    dense_dims = 1 if t.dim() == 4 else 0
    s = t.to_sparse(t.dim() - dense_dims).coalesce()
    ind, val = s.indices(), s.values()
    if val.dtype == torch.bool:
        parts = (val, val)
    elif val.is_floating_point():
        parts = (val * 0.5, val - val * 0.5)
    else:
        parts = (val // 2, val - val // 2)
    n = t.shape[1]
    zi = torch.stack([torch.randint(0, sz, (max(ind.shape[1] // 10, 1),), generator=g) for sz in t.shape[:t.dim() - dense_dims]])
    diag = torch.arange(n).expand(ind.shape[0], n).clone()
    if ind.shape[0] == 3:
        diag[0] = 0
    zeros = torch.zeros((zi.shape[1] + n, *val.shape[1:]), dtype=val.dtype)
    ind = torch.cat((ind, ind, zi, diag), 1)
    return torch.sparse_coo_tensor(ind, torch.cat((*parts, zeros)), t.shape)


def _as_dict(o):
    return o if isinstance(o, dict) else {'0': o}


@pytest.mark.parametrize('name', PAIR_CASES)
def test_fixture_with_sparse_pair_inputs_is_bit_identical_to_dense(name):
    from se3_transformer_pytorch_b200 import SE3Transformer
    z, cfg = load_case(name)
    model = SE3Transformer(**cfg['ctor'])
    fill_state_dict(model, seed=11)
    model = model.to(DEV).eval()
    feats, coors, mask, extra = case_inputs(z)
    feats = {k: cu(v) for k, v in feats.items()} if isinstance(feats, dict) else cu(feats)
    args = (feats, cu(coors), cu(mask))
    dense = {k: torch.from_numpy(v) for k, v in extra.items()}
    ref = _as_dict(model(*args, **{k: v.to(DEV) for k, v in dense.items()}, **cfg['fwd']))
    sparse = _as_dict(model(*args, **{k: v.to_sparse(v.dim() - (k == 'edges' and v.dim() == 4)).to(DEV) for k, v in dense.items()},
                            **cfg['fwd']))
    want = _as_dict(case_outputs(z))
    for d in ref:
        assert torch.equal(sparse[d], ref[d]), d
        assert rel_err(sparse[d].cpu().numpy(), want[d]) < 1e-4, d
    # uncoalesced, with stored zeros: against the dense forward on its to_dense(), one pair input sparse at a time and all at once
    for which in [[k] for k in dense] + ([list(dense)] if len(dense) > 1 else []):
        ms = {k: messy(v, seed=len(k)) for k, v in dense.items() if k in which}
        kw_sparse = {k: ms[k].to(DEV) if k in ms else v.to(DEV) for k, v in dense.items()}
        kw_dense = {k: ms[k].to_dense().to(DEV) if k in ms else v.to(DEV) for k, v in dense.items()}
        a = _as_dict(model(*args, **kw_sparse, **cfg['fwd']))
        b = _as_dict(model(*args, **kw_dense, **cfg['fwd']))
        for d in a:
            assert torch.equal(a[d], b[d]), (which, d)


# ------------------------------------------------------------------ large bonded clouds
def _model():
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    return SE3Transformer(**CTOR).to(DEV).eval()


def _block(t, s, e):
    """The dense [.., e - s, e - s] block of the sparse pair input t (last two sparse dims)."""
    t = t.coalesce()
    ind, val = t.indices(), t.values()
    sel = (ind[-2] >= s) & (ind[-2] < e) & (ind[-1] >= s) & (ind[-1] < e)
    ind = ind[:, sel].clone()
    ind[-2:] -= s
    return torch.sparse_coo_tensor(ind, val[sel], (*t.shape[:-2], e - s, e - s)).to_dense()


def test_bonded_cloud_of_100000_points_matches_each_part_alone():
    """30 parts 1e4 apart, sparse bonds, edge tokens, 2-hop embeddings and neighbor_mask: each part's output is forward() on
    that part alone with dense inputs, to 1e-6 (not bit for bit: at width 16 LinearSE3 runs on torch.matmul, whose cuBLAS kernel
    depends on the row count)."""
    n, P = 100000, 30
    model = _model()
    feats, coors, adj, edges, nbr, bounds = bonded_parts(n, P, DEV, seed=3)
    out = model(feats, coors, adj_mat=adj, edges=edges, neighbor_mask=nbr)
    for s, e in bounds:
        part = model(feats[:, s:e].contiguous(), coors[:, s:e].contiguous(), adj_mat=_block(adj, s, e), edges=_block(edges, s, e),
                     neighbor_mask=_block(nbr, s, e))
        for d in out:
            err = rel_err(out[d][:, s:e].cpu().numpy(), part[d].cpu().numpy())
            assert err < 1e-6, f'degree {d}, nodes {s}:{e}: rel err {err:.3e}'


def _peak(model, feats, coors, **kw):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    model(feats, coors, **kw)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_peak_memory_is_linear_in_nodes():
    """The forward's peak device memory above what was allocated before it: from n = 50 000 to 100 000 it grows by less than
    2.3x with sparse pair inputs and with none.  At n = 10 200 the sparse pair inputs cost less than a tenth of what the dense
    ones cost on top of the forward without pair inputs (H100: 114 MB against 1721 MB), and the whole sparse forward less than
    0.3 of the dense one (0.26: the forward without pair inputs alone is 0.21 of it)."""
    from se3_transformer_pytorch_b200 import SE3Transformer
    model = _model()
    torch.manual_seed(0)
    plain = SE3Transformer(**{k: v for k, v in CTOR.items() if k not in ('attend_sparse_neighbors', 'max_sparse_neighbors',
                                                                          'num_adj_degrees', 'adj_dim', 'num_edge_tokens',
                                                                          'edge_dim')}).to(DEV).eval()
    peaks = {}
    for n, P in ((10200, 3), (50000, 15), (100000, 30)):
        feats, coors, adj, edges, nbr, _ = bonded_parts(n, P, DEV, seed=n)
        sparse = dict(adj_mat=adj, edges=edges, neighbor_mask=nbr)
        peaks[n, 'sparse'] = _peak(model, feats, coors, **sparse)
        peaks[n, 'none'] = _peak(plain, feats, coors)
        if n == 10200:
            dense = {k: v.to_dense() for k, v in sparse.items()}
            peaks[n, 'dense'] = _peak(model, feats, coors, **dense)
            del dense
    print('peak MB on', torch.cuda.get_device_name(), {f'{n}/{kind}': round(p / 2 ** 20, 1) for (n, kind), p in peaks.items()})
    for kind in ('sparse', 'none'):
        assert peaks[100000, kind] < 2.3 * peaks[50000, kind], kind
    assert peaks[10200, 'sparse'] - peaks[10200, 'none'] < (peaks[10200, 'dense'] - peaks[10200, 'none']) / 10
    assert peaks[10200, 'sparse'] < 0.3 * peaks[10200, 'dense']
