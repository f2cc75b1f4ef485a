"""Packed batches without a GPU: the numpy oracle against the reference-generated `varlen` fixtures (one oracle call per cloud), and
SE3Transformer.forward_packed refusing malformed input before any device work."""
import numpy as np
import pytest
import torch

from oracle import se3_oracle as O
from varlen_helpers import VARLEN_CASES, load_varlen, varlen_outputs, per_cloud_errors, varlen_params


@pytest.mark.parametrize('name', VARLEN_CASES)
def test_oracle_matches_varlen_fixture(name):
    z, cfg, feats, coors, seqlens, pairs = load_varlen(name)
    P = varlen_params(name)
    starts = np.cumsum([0] + seqlens[:-1])
    outs = []
    for c, (s, n) in enumerate(zip(starts, seqlens)):
        fc = {d: t[s:s + n][None] for d, t in feats.items()} if isinstance(feats, dict) else feats[s:s + n][None]
        kw = {k: (v[c] if k == 'adj_mat' else v[c][None]) for k, v in pairs.items()}
        outs.append(O.se3_transformer_forward(P, cfg['ctor'], fc, coors[s:s + n][None], np.ones((1, n), dtype=bool), **kw, **cfg['fwd']))
    pooled = cfg['fwd'].get('return_pooled', False)
    cat = lambda ts: np.concatenate([t if pooled else t[0] for t in ts], 0)
    res = {d: cat([o[d] for o in outs]) for d in outs[0]} if isinstance(outs[0], dict) else cat(outs)
    errs = per_cloud_errors(res, varlen_outputs(z), seqlens, pooled)
    assert max(errs) < 1e-4, errs


def _model(**kw):
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(0)
    return SE3Transformer(**{**dict(dim=8, heads=2, dim_head=4, depth=1, num_degrees=2, num_neighbors=4), **kw})


LENS = [5, 3, 4]


def _inputs(lens=LENS, dim=8):
    T = sum(lens)
    return torch.randn(T, dim), torch.randn(T, 3)


@pytest.mark.parametrize('seqlens', [[5, 3, 3], [5, 3, 5], torch.tensor([5, 3]), []])
def test_forward_packed_rejects_seqlens_not_summing_to_nodes(seqlens):
    feats, coors = _inputs()
    with pytest.raises(ValueError, match='seqlens'):
        _model().forward_packed(feats, coors, seqlens)


@pytest.mark.parametrize('seqlens', [[1, 5, 6], [4098], torch.tensor([[5, 3, 4]]), torch.tensor([5., 3., 4.])])
def test_forward_packed_rejects_bad_cloud_sizes(seqlens):
    T = int(torch.as_tensor(seqlens).sum())
    feats, coors = torch.randn(T, 8), torch.randn(T, 3)
    with pytest.raises(ValueError):
        _model().forward_packed(feats, coors, seqlens)


def test_forward_packed_rejects_bad_coors_and_feats():
    feats, coors = _inputs()
    with pytest.raises(ValueError, match='coors'):
        _model().forward_packed(feats, coors[:-1], LENS)
    with pytest.raises(ValueError, match='coors'):
        _model().forward_packed(feats, torch.randn(12, 2), LENS)
    with pytest.raises(ValueError, match='rows'):
        _model().forward_packed(feats[:-1], coors, LENS)


def _adj(lens=LENS):
    return [torch.eye(n, dtype=torch.bool).roll(1, 0) for n in lens]


@pytest.mark.parametrize('name,kw,value', [
    ('adj_mat', dict(attend_sparse_neighbors=True), _adj()[:2]),                         # wrong length
    ('adj_mat', dict(attend_sparse_neighbors=True), torch.zeros(12, 12, dtype=torch.bool)),   # one padded matrix, not a list
    ('adj_mat', dict(attend_sparse_neighbors=True), _adj()[:2] + [torch.zeros(5, 5, dtype=torch.bool)]),   # wrong shape
    ('neighbor_mask', {}, [torch.ones(n, n, dtype=torch.bool) for n in (5, 3, 3)]),
    ('neighbor_mask', {}, [torch.ones(1, n, n, dtype=torch.bool) for n in LENS]),
    ('edges', dict(num_edge_tokens=3, edge_dim=2), [torch.zeros(n, n, 2, dtype=torch.long) for n in LENS]),   # tokens are [n, n]
    ('edges', dict(edge_dim=2), [torch.zeros(n, n, dtype=torch.float) for n in LENS]),                       # features are [n, n, e]
    ('edges', dict(edge_dim=2), [torch.zeros(n, n, 2) for n in LENS[:2]]),
])
def test_forward_packed_rejects_bad_pair_inputs(name, kw, value):
    feats, coors = _inputs()
    with pytest.raises(ValueError, match=name):
        _model(**kw).forward_packed(feats, coors, LENS, **{name: value})


def test_forward_packed_refuses_global_features():
    feats, coors = _inputs()
    with pytest.raises(NotImplementedError, match='global_feats'):
        _model(global_feats_dim=4).forward_packed(feats, coors, LENS)


def test_forward_packed_valid_input_reaches_the_device_check():
    """Well-formed CPU input passes validation and stops at the CUDA-only check (no CPU path), token input and pair lists included."""
    model = _model(num_tokens=5, num_positions=6, attend_sparse_neighbors=True, num_adj_degrees=2)
    tokens, coors = torch.randint(0, 5, (sum(LENS),)), torch.randn(sum(LENS), 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        model.forward_packed(tokens, coors, torch.tensor(LENS), adj_mat=_adj())
    with pytest.raises(AssertionError, match='number of positions'):
        model.forward_packed(torch.randint(0, 5, (9,)), torch.randn(9, 3), [7, 2], adj_mat=_adj([7, 2]))
