"""CausalDecoder refuses what it cannot decode before any device work (models and inputs on the CPU here)."""
import pytest
import torch

from se3_transformer_pytorch_b200 import SE3Transformer

BASE = dict(dim=8, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=4, valid_radius=10)


@pytest.mark.parametrize('extra, match', [
    (dict(causal=False), 'not causal'),
    (dict(causal=True, attend_sparse_neighbors=True, max_sparse_neighbors=2), 'attend_sparse_neighbors'),
    (dict(causal=True, num_adj_degrees=2), 'num_adj_degrees'),
    (dict(causal=True, global_feats_dim=4), 'global_feats_dim'),
    (dict(causal=True, valid_radius=float('inf')), 'FLT_MAX'),
    (dict(causal=True, valid_radius=3.5e38), 'FLT_MAX'),
])
def test_model_refusals(extra, match):
    model = SE3Transformer(**{**BASE, **extra})
    with pytest.raises((ValueError, NotImplementedError), match=match):
        model.causal_decoder()


def _dec(b=2, **extra):
    return SE3Transformer(**{**BASE, 'causal': True, **extra}).causal_decoder(batch_size=b)


@pytest.mark.parametrize('call, match', [
    (lambda d: d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), return_pooled=True), 'return_pooled'),
    (lambda d: d.extend(torch.randn(2, 1, 8), torch.randn(2, 1, 3)), 'at least 2'),
    (lambda d: d.extend(torch.randn(1, 3, 8), torch.randn(1, 3, 3)), 'coors'),
    (lambda d: d.extend(torch.randn(2, 4, 8), torch.randn(2, 3, 3)), 'features'),
    (lambda d: d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), mask=torch.ones(2, 4, dtype=torch.bool)), 'mask'),
    (lambda d: d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), neighbor_mask=torch.ones(2, 3, 4)), 'neighbor_mask'),
    (lambda d: d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), neighbor_mask=torch.ones(2, 3, 3).to_sparse()), 'sparse'),
    (lambda d: d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), edges=torch.zeros(2, 3, 3, dtype=torch.long)), 'edge_dim'),
])
def test_input_refusals(call, match):
    with pytest.raises(ValueError, match=match):
        call(_dec())


def test_edge_and_position_refusals():
    d = _dec(num_edge_tokens=3, edge_dim=2)
    with pytest.raises(ValueError, match='pass edges'):
        d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3))
    with pytest.raises(ValueError, match='n_cur'):
        d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), edges=torch.zeros(2, 3, 4, dtype=torch.long))
    with pytest.raises(ValueError, match='sparse'):
        d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3), edges=torch.zeros(2, 3, 3, dtype=torch.long).to_sparse())
    with pytest.raises(ValueError, match='num_positions'):
        _dec(num_tokens=5, num_positions=4).extend(torch.zeros(2, 5, dtype=torch.long), torch.randn(2, 5, 3))


def test_cpu_inputs_are_refused_and_nothing_is_cached():
    d = _dec()
    with pytest.raises(RuntimeError, match='CUDA'):
        d.extend(torch.randn(2, 3, 8), torch.randn(2, 3, 3))
    assert len(d) == 0
