"""The node-chunk planner of the edge budget (model.plan_node_chunks, block_edge_bytes) and its switch, on CPU."""
import pytest
import torch

from se3_transformer_pytorch_b200 import model as M, switches


def _edges(c, n, k):
    """[e0, e1) of chunk c in the [b, n, k] layout."""
    return (c.b0 * n + c.n0) * k, ((c.b1 - 1) * n + c.n1) * k


@pytest.mark.parametrize('b,n,k', [(1, 1, 1), (1, 7, 3), (3, 5, 4), (4, 1024, 16), (2, 2049, 2048), (1, 100000, 16)])
@pytest.mark.parametrize('budget_edges', [0, 1, 3, 17, 64, 1000, 10 ** 9])
def test_chunks_cover_every_node_once_in_order(b, n, k, budget_edges):
    per_edge = 100
    chunks = M.plan_node_chunks(b, n, k, per_edge, budget_edges * per_edge)
    e = 0
    for c in chunks:
        assert c.b0 < c.b1 and c.n0 < c.n1
        # whole rows, or a node range inside one row: the chunk's edges are whole neighbour lists, one contiguous range
        assert (c.n0, c.n1) == (0, n) or c.b1 == c.b0 + 1
        e0, e1 = _edges(c, n, k)
        assert e0 == e and e0 % k == 0 and e1 % k == 0
        e = e1
        nodes = (c.b1 - c.b0) * (c.n1 - c.n0)
        assert nodes == 1 or nodes * k * per_edge <= budget_edges * per_edge
    assert e == b * n * k
    assert len(chunks) == 1 or not chunks[0].whole


def test_one_chunk_when_the_budget_is_large_or_unset():
    for budget in (None, 10 ** 15):
        (c,) = M.plan_node_chunks(4, 1024, 16, 80_000, budget)
        assert c == (0, 4, 0, 1024, True)


def test_one_node_chunks_when_the_budget_is_tiny():
    chunks = M.plan_node_chunks(2, 5, 3, 100, 0)
    assert [(c.b0, c.n0, c.n1) for c in chunks] == [(r, i, i + 1) for r in range(2) for i in range(5)]


def test_row_chunks_take_whole_rows_and_are_balanced():
    chunks = M.plan_node_chunks(5, 10, 4, 10, 2 * 10 * 4 * 10)         # two rows fit
    assert [(c.b0, c.b1, c.n0, c.n1) for c in chunks] == [(0, 2, 0, 10), (2, 4, 0, 10), (4, 5, 0, 10)]
    chunks = M.plan_node_chunks(1, 10, 4, 10, 4 * 4 * 10)              # four nodes fit: 3 balanced chunks of 4, 3, 3
    assert [(c.n0, c.n1) for c in chunks] == [(0, 4), (4, 8), (8, 10)]


def test_chunk_views():
    c = M.NodeChunk(1, 2, 3, 5)
    t = torch.arange(2 * 6 * 4).view(2, 6, 4)
    assert torch.equal(c.rows(t), t[1:2, 3:5])
    src = c.src(t)                                 # starts at the row's first node, as many nodes as the chunk
    assert src.shape == (1, 2, 4) and src.data_ptr() == t[1].data_ptr() and src.is_contiguous()
    assert c.rows(None) is None and torch.equal(c.rows({'0': t})['0'], t[1:2, 3:5])


def _decision(C, degrees, route, lowrank=True, pool=False):
    fiber = M.Fiber([(d, C) for d in range(degrees)])
    conv = M.ConvSE3(fiber, fiber, pool=pool, self_interaction=False)
    d = M.ConvDecision.__new__(M.ConvDecision)
    d.conv, d.route, d.lr = conv, route, ({pair: {} for pair in conv.pairs} if lowrank else {})
    d.direct = not lowrank
    return d


@pytest.mark.parametrize('route,lowrank', [('production', True), ('aligned', True), ('rfirst', True), ('rfirst', False)])
def test_estimate_grows_with_width_and_k(route, lowrank):
    small = M.block_edge_bytes([_decision(128, 3, route, lowrank)] * 2, 2, keep_aligned=route == 'production')
    wide = M.block_edge_bytes([_decision(256, 3, route, lowrank)] * 2, 2, keep_aligned=route == 'production')
    deep = M.block_edge_bytes([_decision(128, 4, route, lowrank)] * 2, 3, keep_aligned=route == 'production')
    assert 0 < small < wide and small < deep
    # more neighbours per node: fewer nodes per chunk under the same budget
    counts = [len(M.plan_node_chunks(1, 4096, k, small, 2 ** 30)) for k in (16, 256, 4096)]
    assert counts[0] < counts[1] < counts[2]


def test_pooled_production_keeps_no_edge_outputs():
    pooled = M.block_edge_bytes([_decision(128, 3, 'production', pool=True)], 2)
    unpooled = M.block_edge_bytes([_decision(128, 3, 'production', pool=False)], 2)
    assert unpooled - pooled == 4 * 128 * (1 + 3 + 5)


def test_switch_parses_and_round_trips(monkeypatch):
    monkeypatch.delenv('SE3B200_EDGE_BUDGET_MB', raising=False)
    assert switches.current().edge_budget_mb is None
    monkeypatch.setenv('SE3B200_EDGE_BUDGET_MB', '8192')
    assert switches.current().edge_budget_mb == 8192.0
    assert M.edge_budget_bytes(switches.current(), 'cpu') == 8192 * 2 ** 20
    monkeypatch.setenv('SE3B200_EDGE_BUDGET_MB', '0.5')
    assert M.edge_budget_bytes(switches.current(), 'cpu') == 2 ** 19
    monkeypatch.delenv('SE3B200_EDGE_BUDGET_MB')
    for v in (0, 64, 0.25):
        with switches.override(edge_budget_mb=v):
            assert switches.current().edge_budget_mb == v
        assert switches.current().edge_budget_mb is None
