"""PagedCausalDecoder on the CPU: its page bookkeeping (PageTables), and the refusals it shares with PackedCausalDecoder, made
before any device work with the same messages."""
import pytest
import torch

from se3_transformer_pytorch_b200 import SE3Transformer, PagedCausalDecoder, DecoderCacheFull
from se3_transformer_pytorch_b200.model import PageTables

import test_packed_decode_host as packed
from test_packed_decode_host import BASE, _x


# ---- page bookkeeping ---------------------------------------------------------------------------------------------------------
def _step(book, ids, n_prev, seqlens):
    return book.commit(book.plan(ids, n_prev, seqlens), ids)


def test_pages_are_taken_fresh_then_reused_after_close():
    book = PageTables(4)
    book.open(0), book.open(1)
    assert _step(book, [0, 1], [0, 0], [10, 3]) == []
    assert book.tables == {0: [0, 1, 2], 1: [3]} and book.reserved == 4 and book.pages_in_use() == 4
    book.close(0)
    assert book.pages_in_use() == 1 and sorted(book.free) == [0, 1, 2]
    book.open(2)
    _step(book, [2], [0], [5])
    assert sorted(book.tables[2]) == [1, 2] and book.reserved == 4, 'freed pages come first'
    _step(book, [1, 2], [3, 5], [6, 4])               # 1: page 3 then two more; 2: one more: pool doubles, no page id moves
    assert book.reserved == 8 and book.tables[1][0] == 3 and sorted(book.tables[2][:2]) == [1, 2]
    assert len(book.tables[1]) == 3 and len(book.tables[2]) == 3
    assert sorted(p for t in book.tables.values() for p in t) == sorted(set(p for t in book.tables.values() for p in t))


def test_fork_shares_pages_and_copy_on_write_after_fork():
    book = PageTables(4)
    book.open(0)
    _step(book, [0], [0], [10])                       # pages 0, 1, 2; node 10 in page 2 at row 2
    book.fork(0, 1, 10)
    assert book.tables[1] == [0, 1, 2] and [book.refs[p] for p in (0, 1, 2)] == [2, 2, 2]
    assert book.pages_in_use() == 3
    plan = book.plan([0], [10], [1])
    assert plan.cow == [(0, 2, 2)] and plan.fresh == [0]
    copies = book.commit(plan, [0])
    new = book.tables[0][2]
    assert copies == [(2, new, 2)] and new not in (0, 1, 2)
    assert book.tables[1] == [0, 1, 2] and book.refs[2] == 1 and book.refs[new] == 1
    assert _step(book, [1], [10], [2]) == [], 'page 2 is now the sibling\'s alone: written in place'


def test_fork_on_a_page_boundary_needs_no_copy():
    book = PageTables(4)
    book.open(0)
    _step(book, [0], [0], [8])
    book.fork(0, 1, 8)
    plan = book.plan([0, 1], [8, 8], [1, 1])
    assert plan.cow == [] and plan.fresh == [1, 1]


def test_siblings_writing_one_shared_page_in_one_step_copy_it_once():
    book = PageTables(4)
    book.open(0)
    _step(book, [0], [0], [6])
    book.fork(0, 1, 6)
    book.fork(0, 2, 6)                                # page 1 held three times; clouds 0 and 1 write it, 2 does not
    plan = book.plan([0, 1], [6, 6], [1, 1])
    assert plan.cow == [(0, 1, 2), (1, 1, 2)]
    book.commit(plan, [0, 1])
    assert book.tables[2] == [0, 1] and book.refs[1] == 1
    book.close(2)
    plan = book.plan([0, 1], [7, 7], [1, 1])          # each writes its own copy now
    assert plan.cow == []


def test_truncate_into_a_shared_page_then_both_siblings_extend():
    book = PageTables(4)
    book.open(0)
    _step(book, [0], [0], [12])
    book.fork(0, 1, 12)
    book.truncate(0, 6)                               # cloud 0 keeps pages 0, 1 (both shared); page 2 is cloud 1's alone
    assert book.tables[0] == [0, 1] and book.refs[2] == 1 and book.pages_in_use() == 3
    plan = book.plan([0, 1], [6, 12], [3, 1])
    assert plan.cow == [(0, 1, 2)] and plan.fresh == [1, 1]
    copies = book.commit(plan, [0, 1])
    assert copies[0][0] == 1 and book.tables[1] == [0, 1, 2, book.tables[1][3]]
    book.truncate(1, 0)
    assert book.tables[1] == [] and book.refs[0] == 1 and book.refs[1] == 0


def test_close_and_truncate_free_pages():
    book = PageTables(3)
    book.open(0)
    _step(book, [0], [0], [9])
    book.fork(0, 1, 9)
    book.truncate(0, 4)
    assert book.pages_in_use() == 3 and book.free == []
    book.close(1)
    assert book.pages_in_use() == 2 and book.free == [2]
    book.close(0)
    assert book.pages_in_use() == 0 and sorted(book.free) == [0, 1, 2]


def test_capped_pool_refuses_before_any_change():
    book = PageTables(4, max_pages=3)
    book.open(0), book.open(1)
    _step(book, [0], [0], [6])
    assert book.reserved == 3, 'a capped pool is reserved whole at the first step'
    state = (dict((c, list(t)) for c, t in book.tables.items()), list(book.refs), list(book.free), book.reserved)
    with pytest.raises(DecoderCacheFull, match='needs 2 free pages'):
        book.plan([0, 1], [6, 0], [3, 2])
    assert (book.tables, book.refs, book.free, book.reserved) == state
    _step(book, [1], [0], [2])                        # exactly fits
    assert book.pages_in_use() == 3 and issubclass(DecoderCacheFull, RuntimeError)


# ---- the decoder: options and refusals ---------------------------------------------------------------------------------------
def _dec(page_size=4, max_nodes=None, **extra):
    return SE3Transformer(**{**BASE, 'causal': True, **extra}).packed_decoder(page_size=page_size, max_nodes=max_nodes)


def test_page_size_selects_the_decoder():
    model = SE3Transformer(**{**BASE, 'causal': True})
    assert type(model.packed_decoder()).__name__ == 'PackedCausalDecoder'
    d = model.packed_decoder(page_size=16, max_nodes=100)
    assert isinstance(d, PagedCausalDecoder) and d.page_size == 16
    assert d.pages_in_use() == 0 and d.pages_reserved() == 0


@pytest.mark.parametrize('kw, match', [
    (dict(page_size=0), 'page_size'),
    (dict(page_size=-3), 'page_size'),
    (dict(page_size=2.0), 'page_size'),
    (dict(page_size=True), 'page_size'),
    (dict(page_size=4, max_nodes=0), 'max_nodes'),
    (dict(page_size=4, max_nodes=1.5), 'max_nodes'),
    (dict(max_nodes=64), 'give a page_size'),
])
def test_invalid_page_size_and_max_nodes(kw, match):
    model = SE3Transformer(**{**BASE, 'causal': True})
    with pytest.raises(ValueError, match=f'packed_decoder: .*{match}'):
        model.packed_decoder(**kw)


@pytest.mark.parametrize('extra, match', [
    (dict(causal=False), 'not causal'),
    (dict(attend_sparse_neighbors=True, max_sparse_neighbors=2), 'attend_sparse_neighbors'),
    (dict(global_feats_dim=4), 'global_feats_dim'),
])
def test_model_refusals(extra, match):
    model = SE3Transformer(**{**BASE, 'causal': True, **extra})
    with pytest.raises((ValueError, NotImplementedError), match=f'packed_decoder: .*{match}'):
        model.packed_decoder(page_size=8)


def _state(d):
    return d.open_ids(), {c: d.length(c) for c in d.open_ids()}, {c: list(t) for c, t in d._book.tables.items()}


_PACKED_REFUSALS = next(m for m in packed.test_input_refusals_leave_the_decoder_unchanged.pytestmark
                        if m.name == 'parametrize').args[1]


@pytest.mark.parametrize('call, match', _PACKED_REFUSALS)
def test_input_refusals_match_the_packed_decoder(call, match):
    """Every input refusal of PackedCausalDecoder, with its message, and the paged decoder's clouds and pages stay as they were."""
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
    d = _dec(num_tokens=5, num_positions=4)
    a, b = d.open(2)
    with pytest.raises(ValueError, match='num_positions'):
        d.extend([a, b], [2, 5], torch.zeros(7, dtype=torch.long), torch.randn(7, 3))
    assert _state(d) == ([a, b], {a: 0, b: 0}, {a: [], b: []})


def test_cpu_inputs_are_refused_before_any_page_moves():
    d = _dec()
    a, b = d.open(2)
    before = _state(d)
    with pytest.raises(RuntimeError, match='CUDA'):
        d.extend([a, b], [3, 2], *_x(5))
    assert _state(d) == before and d.pages_in_use() == 0 and d.pages_reserved() == 0
    assert d.coors is None and not d.stages


def test_cache_full_leaves_the_decoder_unchanged():
    """A capped pool refuses a step it cannot hold before the device is touched: inputs on the CPU, which the step body would
    refuse, show that the refusal comes first."""
    d = _dec(page_size=4, max_nodes=8)
    a, b = d.open(2)
    before = _state(d)
    with pytest.raises(DecoderCacheFull, match='needs 3 free pages'):
        d.extend([a, b], [7, 3], *_x(10))
    assert _state(d) == before and d.pages_reserved() == 0 and d.coors is None


def test_lifecycle_bookkeeping():
    d = _dec(page_size=3)
    ids = d.open(3)
    assert ids == [0, 1, 2] and d.open_ids() == ids
    d.close(1)
    for call in (lambda: d.close(1), lambda: d.length(1), lambda: d.truncate(1, 0), lambda: d.fork(1),
                 lambda: d.extend([1], [2], *_x(2))):
        with pytest.raises(ValueError, match='not an open cloud'):
            call()
    new, = d.open()
    assert new == 3 and d.open_ids() == [0, 2, 3]
    with pytest.raises(ValueError, match=r'\[0, 0\]'):
        d.truncate(0, 1)
    _step(d._book, [0], [0], [7])                     # as an extend of 7 nodes would (nothing is computed here)
    d._len[0] = 7
    f = d.fork(0)
    assert f == 4 and d.length(f) == 7 and d._book.tables[f] == d._book.tables[0] and d.pages_in_use() == 3
    d.truncate(0, 2)
    assert d.length(0) == 2 and d._book.tables[0] == d._book.tables[f][:1] and d.pages_in_use() == 3
    with pytest.raises(ValueError, match=r'\[0, 2\]'):
        d.truncate(0, 3)
    d.close(f)
    assert d.pages_in_use() == 1
    with pytest.raises(ValueError, match='count'):
        d.open(0)
