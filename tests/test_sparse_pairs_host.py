"""Sparse pair inputs of SE3Transformer.forward without a GPU: the refusals (checked before any device work), the conversion of
a torch.sparse_coo input into sorted column lists, and the sparse N-hop expansion and bonded selection against the dense
_bonded on the densified adjacency."""
import pytest
import torch

from se3_transformer_pytorch_b200 import ops


def _model(**kw):
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    return SE3Transformer(**{**dict(dim=8, heads=2, dim_head=4, depth=1, num_degrees=2, num_neighbors=4), **kw})


def densify(rows, b, n):
    """PairRows -> dense [b, n, n, ...] of its values (zero where absent)."""
    R = rows.ptr.numel() - 1
    r = torch.repeat_interleave(torch.arange(R), rows.ptr.diff())
    out = torch.zeros((R // n, n, n, *rows.values.shape[1:]), dtype=rows.values.dtype)
    out[r // n, r % n, rows.cols.long()] = rows.values
    return out.expand(b, *out.shape[1:]) if rows.shared else out


def chain(n):
    i = torch.arange(n)
    return (i[:, None] - i[None]).abs() == 1


def ring(n):
    i = torch.arange(n)
    d = (i[:, None] - i[None]) % n
    return (d == 1) | (d == n - 1)


def random_graph(n, p, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(n, n, generator=g) < p
    return a | a.T


# ------------------------------------------------------------------ refusals
def _sp(*shape, dtype=torch.bool, dense_dims=0):
    i = torch.zeros((len(shape) - dense_dims, 1), dtype=torch.long)
    return torch.sparse_coo_tensor(i, torch.ones((1, *shape[len(shape) - dense_dims:]), dtype=dtype), shape)


B, N = 2, 6


def _call(model, **kw):
    model(torch.randn(B, N, 8), torch.randn(B, N, 3), **kw)


@pytest.mark.parametrize('layout', ['csr', 'csc', 'bsr'])
def test_other_sparse_layouts_are_refused(layout):
    model = _model(attend_sparse_neighbors=True)
    dense = torch.eye(N, dtype=torch.float32)
    t = {'csr': dense.to_sparse_csr, 'csc': dense.to_sparse_csc, 'bsr': lambda: dense.to_sparse_bsr((2, 2))}[layout]()
    with pytest.raises(ValueError, match=r'to_sparse_coo\(\)'):
        _call(model, adj_mat=t)


@pytest.mark.parametrize('name,t', [
    ('adj_mat', _sp(1, N, N)),                # [1, n, n] is only a neighbor_mask shape
    ('adj_mat', _sp(B, N, N + 1)),
    ('adj_mat', _sp(N, N, 3, dense_dims=1)),
    ('neighbor_mask', _sp(3, N, N)),
    ('neighbor_mask', _sp(N)),
    ('adj_mat', _sp(N, N, dtype=torch.complex64)),
])
def test_wrong_sparse_mask_shapes_and_dtypes_are_refused(name, t):
    model = _model(attend_sparse_neighbors=True)
    kw = {'adj_mat': _sp(N, N)} if name != 'adj_mat' else {}
    with pytest.raises(ValueError, match=name):
        _call(model, **kw, **{name: t})


def test_two_dimensional_sparse_edges_are_refused():
    model = _model(num_edge_tokens=4, edge_dim=2)
    with pytest.raises(ValueError, match='ambiguous'):
        _call(model, edges=_sp(B, N, dtype=torch.long))


@pytest.mark.parametrize('ctor,t,match', [
    (dict(num_edge_tokens=4, edge_dim=2), _sp(B, N, N, dtype=torch.float32), 'integer dtype'),
    (dict(num_edge_tokens=4, edge_dim=2), _sp(B, N, N, dtype=torch.bool), 'integer dtype'),
    (dict(num_edge_tokens=4, edge_dim=2), _sp(B, N, N + 1, dtype=torch.long), r'\[b, n, n\]'),
    (dict(edge_dim=3), _sp(B, N, N, 3, dtype=torch.float32), '3 sparse'),   # 4 sparse dims
    (dict(edge_dim=3), _sp(B, N, N, dtype=torch.float32), 'edge_dim'),
])
def test_wrong_sparse_edges_are_refused(ctor, t, match):
    with pytest.raises(ValueError, match=match):
        _call(_model(**ctor), edges=t)


def test_graphed_refuses_sparse_pair_inputs():
    with pytest.raises(ValueError, match='graphed'):
        _model(num_adj_degrees=2, adj_dim=2).graphed(torch.randn(1, N, 8), torch.randn(1, N, 3), adj_mat=_sp(N, N))


def test_forward_packed_refuses_sparse_pair_inputs():
    model = _model(attend_sparse_neighbors=True)
    with pytest.raises(ValueError, match=r'adj_mat\[1\] is a sparse tensor'):
        model.forward_packed(torch.randn(9, 8), torch.randn(9, 3), [5, 4], adj_mat=[torch.zeros(5, 5, dtype=torch.bool), _sp(4, 4)])


# ------------------------------------------------------------------ COO -> rows
def _messy_coo(shape, dense_dims=(), dtype=torch.float32, nnz=60, seed=0):
    """Uncoalesced: duplicates, stored zeros and diagonal entries."""
    g = torch.Generator().manual_seed(seed)
    ind = torch.stack([torch.randint(0, s, (nnz,), generator=g) for s in shape])
    ind = torch.cat((ind, ind[:, :10]), 1)                            # duplicates
    ind[-1, -5:] = ind[-2, -5:]                                       # diagonal entries
    vals = torch.randint(0, 3, (ind.shape[1], *dense_dims), generator=g).to(dtype)   # a third of them stored zeros
    return torch.sparse_coo_tensor(ind, vals, (*shape, *dense_dims))


@pytest.mark.parametrize('shape,dense_dims,dtype', [((7, 7), (), torch.float32), ((1, 7, 7), (), torch.bool),
                                                    ((3, 7, 7), (), torch.int64), ((3, 7, 7), (4,), torch.float64)])
def test_coo_to_rows_matches_to_dense(shape, dense_dims, dtype):
    t = _messy_coo(shape, dense_dims, dtype)
    rows = ops.coo_to_rows(t, 7)
    assert rows.shared == (len(shape) == 2 or shape[0] == 1)
    assert rows.ptr.dtype == torch.int64 and rows.cols.dtype == torch.int32
    r = torch.repeat_interleave(torch.arange(rows.ptr.numel() - 1), rows.ptr.diff())
    key = r * 7 + rows.cols.long()
    assert bool((key[1:] > key[:-1]).all())                          # ascending and unique per row
    ref = t.to_dense()
    assert torch.equal(densify(rows, ref.shape[0] if ref.dim() > 2 + len(dense_dims) else 1, 7).reshape(ref.shape), ref)


# ------------------------------------------------------------------ the N-hop expansion and the bonded neighbours
GRAPHS = {
    'chain': lambda n: chain(n),
    'ring': lambda n: ring(n),
    'random': lambda n: random_graph(n, 0.15, 1),
    'selfloops': lambda n: random_graph(n, 0.1, 2) | torch.eye(n, dtype=torch.bool),
}


def _adj(graph, batched, n=11):
    if batched:
        return torch.stack([GRAPHS[graph](n), random_graph(n, 0.2, 3), chain(n) | ring(n)])
    return GRAPHS[graph](n)


@pytest.mark.parametrize('graph', list(GRAPHS))
@pytest.mark.parametrize('batched', [False, True])
@pytest.mark.parametrize('degrees', [None, 1, 2, 3, 4])
def test_sparse_bonded_matches_dense(graph, batched, degrees):
    adj = _adj(graph, batched)
    b, n = 3, adj.shape[-1]
    model = _model(attend_sparse_neighbors=True, num_adj_degrees=degrees, adj_dim=2 if degrees else 0)
    hops, mask, num_sparse = model._bonded(adj, b, n, 'cpu')
    s_hops, s_bonded, s_num = model._bonded_sparse(adj.to_sparse(), b, n)
    assert s_num == num_sparse
    assert torch.equal(densify(s_bonded, b, n), mask.expand(b, n, n))
    if degrees is None:
        assert s_hops is None and hops is None
    else:
        assert torch.equal(densify(s_hops, b, n), hops)


def test_chain_hops_follow_the_reference_doubling():
    """M_d = (M_{d-1} @ M_{d-1}) > 0 and XOR: with 3 degrees the bond (i, i+1) has hop value 2 and the bonded set of i is
    {i +- 2, i +- 4}."""
    n = 12
    model = _model(attend_sparse_neighbors=True, num_adj_degrees=3, adj_dim=2)
    hops, bonded, num_sparse = model._bonded_sparse(chain(n).to_sparse(), 1, n)
    h, m = densify(hops, 1, n)[0], densify(bonded, 1, n)[0]
    assert [int(h[5, j]) for j in (6, 7, 8, 9, 10)] == [2, 2, 0, 3, 0]
    assert m[5].nonzero().flatten().tolist() == [1, 3, 7, 9]
    assert num_sparse == 4


def test_sparse_bonded_of_messy_coo_matches_dense():
    """Duplicates summed (values 2 become hop value 2 and weigh 2 in the row sums), stored zeros and diagonal entries."""
    t = _messy_coo((2, 9, 9), dtype=torch.int64, nnz=30)
    for degrees in (1, 2, 3):
        model = _model(attend_sparse_neighbors=True, num_adj_degrees=degrees, adj_dim=2)
        hops, mask, num_sparse = model._bonded(t.to_dense(), 2, 9, 'cpu')
        s_hops, s_bonded, s_num = model._bonded_sparse(t, 2, 9)
        assert s_num == num_sparse
        assert torch.equal(densify(s_bonded, 2, 9), mask)
        assert torch.equal(densify(s_hops, 2, 9), hops)


@pytest.mark.parametrize('batched', [False, True])
def test_sub_sampled_rows_pick_distinct_bonded_columns(batched):
    n, max_sparse = 40, 3
    adj = _adj('random', batched, n)
    b = 3
    model = _model(attend_sparse_neighbors=True, max_sparse_neighbors=max_sparse, num_adj_degrees=2, adj_dim=2)
    _, full, _ = _model(attend_sparse_neighbors=True, num_adj_degrees=2, adj_dim=2)._bonded_sparse(adj.to_sparse(), b, n)
    full = densify(full, b, n)
    assert int(full.sum(-1).max()) > max_sparse                       # the sub-sampling regime
    _, picked, num_sparse = model._bonded_sparse(adj.to_sparse(), b, n)
    assert num_sparse == max_sparse and not picked.shared
    picked = densify(picked, b, n)
    assert not bool((picked & ~full).any())                           # only bonded columns
    assert torch.equal(picked.sum(-1), full.sum(-1).clamp(max=max_sparse))


def test_sub_sampling_is_uniform():
    """A row with 8 bonded columns and max_sparse_neighbors = 2: every column is picked with probability 1/4."""
    n, draws = 9, 800
    adj = torch.zeros(n, n, dtype=torch.bool)
    adj[0, 1:] = True
    model = _model(attend_sparse_neighbors=True, max_sparse_neighbors=2)
    counts = torch.zeros(n)
    torch.manual_seed(1)
    for _ in range(draws):
        _, picked, _ = model._bonded_sparse(adj.to_sparse(), 1, n)
        counts += densify(picked, 1, n)[0, 0].float()
    freq = counts[1:] / draws
    assert float((freq - 0.25).abs().max()) < 0.07, freq              # ~4.5 standard deviations
