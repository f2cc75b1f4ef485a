"""PackedCausalDecoder refuses what it cannot decode before any device work and keeps its clouds' bookkeeping (models and
inputs on the CPU here)."""
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
])
def test_model_refusals(extra, match):
    model = SE3Transformer(**{**BASE, **extra})
    with pytest.raises((ValueError, NotImplementedError), match=f'packed_decoder: .*{match}'):
        model.packed_decoder()


def _dec(**extra):
    return SE3Transformer(**{**BASE, 'causal': True, **extra}).packed_decoder()


def _state(d):
    return d.open_ids(), {c: d.length(c) for c in d.open_ids()}


def _x(m):
    return torch.randn(m, 8), torch.randn(m, 3)


@pytest.mark.parametrize('call, match', [
    (lambda d, a, b: d.extend([a], [3], *_x(3), return_pooled=True), 'return_pooled'),
    (lambda d, a, b: d.extend([a, a], [2, 2], *_x(4)), 'distinct'),
    (lambda d, a, b: d.extend([99], [2], *_x(2)), 'not an open cloud'),
    (lambda d, a, b: d.extend([], [], *_x(0)), 'at least one'),
    (lambda d, a, b: d.extend([a, b], [2], *_x(2)), 'one count'),
    (lambda d, a, b: d.extend([a, b], [2, 0], *_x(2)), 'one count'),
    (lambda d, a, b: d.extend([a, b], [2, 3], *_x(4)), r'sum\(seqlens\)'),
    (lambda d, a, b: d.extend([a, b], [2, 2], torch.randn(5, 8), torch.randn(4, 3)), 'features'),
    (lambda d, a, b: d.extend([a, b], [2, 1], *_x(3)), 'fewer than 2'),
    (lambda d, a, b: d.extend([a], [2], *_x(2), neighbor_mask=[]), 'list of 1'),
    (lambda d, a, b: d.extend([a], [2], *_x(2), neighbor_mask=torch.ones(2, 2, dtype=torch.bool)), 'list of 1'),
    (lambda d, a, b: d.extend([a], [2], *_x(2), neighbor_mask=[torch.ones(2, 3, dtype=torch.bool)]), r'\[m, n_cur\]'),
    (lambda d, a, b: d.extend([a], [2], *_x(2), neighbor_mask=[torch.ones(2, 2).to_sparse()]), 'sparse'),
    (lambda d, a, b: d.extend([a], [2], torch.randn(2, 8), torch.randn(2, 3).to_sparse()), 'coors'),
    (lambda d, a, b: d.extend([a], [2], *_x(2), edges=[torch.zeros(2, 2, dtype=torch.long)]), 'edge_dim'),
])
def test_input_refusals_leave_the_decoder_unchanged(call, match):
    d = _dec()
    a, b = d.open(2)
    before = _state(d)
    with pytest.raises(ValueError, match=match):
        call(d, a, b)
    assert _state(d) == before


def test_edge_and_position_refusals():
    d = _dec(num_edge_tokens=3, edge_dim=2)
    a, = d.open()
    with pytest.raises(ValueError, match='pass edges'):
        d.extend([a], [3], *_x(3))
    with pytest.raises(ValueError, match=r'\[m, n_cur\]'):
        d.extend([a], [3], *_x(3), edges=[torch.zeros(3, 4, dtype=torch.long)])
    with pytest.raises(ValueError, match='sparse'):
        d.extend([a], [3], *_x(3), edges=[torch.zeros(3, 3, dtype=torch.long).to_sparse()])
    d = _dec(edge_dim=2)
    a, = d.open()
    with pytest.raises(ValueError, match='edge_dim'):
        d.extend([a], [3], *_x(3), edges=[torch.zeros(3, 3)])
    d = _dec(num_tokens=5, num_positions=4)
    a, b = d.open(2)
    with pytest.raises(ValueError, match='num_positions'):
        d.extend([a, b], [2, 5], torch.zeros(7, dtype=torch.long), torch.randn(7, 3))
    assert _state(d) == ([a, b], {a: 0, b: 0})


def test_cpu_inputs_are_refused_and_nothing_is_cached():
    d = _dec()
    a, b = d.open(2)
    with pytest.raises(RuntimeError, match='CUDA'):
        d.extend([a, b], [3, 2], *_x(5))
    assert _state(d) == ([a, b], {a: 0, b: 0})
    assert d.coors is None and not d.stages


def test_lifecycle_bookkeeping():
    d = _dec()
    ids = d.open(3)
    assert ids == [0, 1, 2] and d.open_ids() == ids
    assert [d._slot[c] for c in ids] == [0, 1, 2]
    d.close(1)
    for call in (lambda: d.close(1), lambda: d.length(1), lambda: d.truncate(1, 0), lambda: d.fork(1),
                 lambda: d.extend([1], [2], *_x(2))):
        with pytest.raises(ValueError, match='not an open cloud'):
            call()
    new, = d.open()
    assert new == 3 and d._slot[new] == 1, 'ids are never reused; cache rows are'
    assert d.open_ids() == [0, 2, 3]
    assert d.length(0) == 0
    with pytest.raises(ValueError, match=r'\[0, 0\]'):
        d.truncate(0, 1)
    d._len[0] = 5                      # as after extend; truncate and fork move lengths only (nothing is cached here)
    d.truncate(0, 3)
    assert d.length(0) == 3
    with pytest.raises(ValueError, match=r'\[0, 3\]'):
        d.truncate(0, 4)
    d.truncate(0, 0)
    f = d.fork(0)
    assert f == 4 and d.length(f) == 0 and d._slot[f] == 3
    with pytest.raises(ValueError, match='count'):
        d.open(0)
