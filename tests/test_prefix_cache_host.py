"""The prefix cache of PagedCausalDecoder on the CPU (DESIGN.md 10.4): PageTables with the cache (registration, LRU eviction,
what is never evicted, DecoderCacheFull, rollback), the decoder's counters, the host page-key chain against a pure-Python
statement, option validation, and every input refusal of the packed decoder with the cache on."""
import numpy as np
import pytest

from se3_transformer_pytorch_b200 import SE3Transformer, DecoderCacheFull
from se3_transformer_pytorch_b200.model import PageTables, prefix_page_keys, PREFIX_SEEDS, PREFIX_GOLD

import test_paged_decode_host as paged
from test_packed_decode_host import BASE, _x

M64 = (1 << 64) - 1


def _step(book, ids, n_prev, seqlens, hits=()):
    return book.commit(book.plan(ids, n_prev, seqlens, hits), ids)


def _prompt(book, c, n, keys):
    """Cloud c takes an n-node prompt and registers its full pages under keys[q], as the decoder does after the step."""
    _step(book, [c], [0], [n])
    for q in range(n // book.P):
        book.register(keys[q], book.tables[c][q])


def _state(book):
    return ({c: list(t) for c, t in book.tables.items()}, list(book.refs), list(book.free), list(book.cached.items()),
            dict(book.page_key), book.reserved)


def _consistent(book):
    """Counts recomputed from the tables and the cache match the running ones; no referenced page is free or evictable."""
    held = [0] * book.reserved
    for t in book.tables.values():
        for p in t:
            held[p] += 1
    for p in book.cached.values():
        held[p] += 1
    assert held == book.refs
    assert sorted(book.free) == [p for p in range(book.reserved) if not held[p]]
    assert book.n_evictable == sum(book.refs[p] == 1 for p in book.cached.values())
    assert book.pages_in_use() == len({p for t in book.tables.values() for p in t})


# ---- PageTables with the cache ---------------------------------------------------------------------------------------------
def test_registration_holds_one_reference_and_keeps_the_first_entry():
    book = PageTables(4, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 10, ['a', 'b'])                  # pages 0, 1 full and registered; page 2 holds nodes 8, 9
    assert list(book.cached.items()) == [('a', 0), ('b', 1)] and book.refs[:3] == [2, 2, 1]
    assert book.pages_cached() == 2 and book.pages_in_use() == 3
    _step(book, [1], [0], [8])
    book.register('a', book.tables[1][0])             # an equal prompt in the same step: the existing entry stays
    assert book.cached['a'] == 0 and book.refs[book.tables[1][0]] == 1
    book.close(0)
    assert book.pages_in_use() == 2 and book.pages_cached() == 2 and 2 in book.free and 0 not in book.free, 'cached pages are not free'
    assert book.lookup(['a', 'b', 'c']) == [0, 1] and book.lookup(['b']) == [1] and book.lookup(['z', 'a']) == []


def test_a_hit_attaches_pages_and_counts_as_a_use():
    book = PageTables(4, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 8, ['a', 'b'])
    _prompt(book, 1, 4, ['x'])
    book.close(0), book.close(1)
    assert list(book.cached) == ['a', 'b', 'x'] and book.pages_in_use() == 0
    book.open(2)
    hits = book.lookup(['a'])
    plan = book.plan([2], [4], [3], hits=[(2, hits)])
    assert plan.fresh == [1] and plan.cow == []
    _step(book, [2], [4], [3], hits=[(2, hits)])
    assert book.tables[2][0] == 0 and book.refs[0] == 2 and list(book.cached) == ['a', 'b', 'x'], 'a use once the step succeeds'
    book.use(hits)
    assert list(book.cached) == ['b', 'x', 'a']
    _consistent(book)


def test_eviction_is_least_recently_used_and_spares_referenced_and_hit_pages():
    book = PageTables(2, max_pages=6, cache=True)
    for c in range(4):
        book.open(c)
    _prompt(book, 0, 2, ['a'])
    _prompt(book, 1, 2, ['b'])
    _prompt(book, 2, 2, ['c'])
    _prompt(book, 3, 2, ['d'])
    pa, pb, pc, pd = (book.cached[k] for k in 'abcd')
    book.close(0), book.close(1), book.close(2)      # 'a', 'b', 'c' are held only by the cache; 'd' by cloud 3 too
    assert book.pages_in_use() == 1 and len(book.free) == 2
    book.open(4)
    hit = book.lookup(['b'])                         # cloud 4 hits 'b': b is not evictable in this step
    _step(book, [4], [2], [6], hits=[(4, hit)])      # 3 fresh pages: 2 free, then evicts 'a' (the least recently used)
    book.use(hit)
    assert list(book.cached) == ['c', 'd', 'b'] and pa in book.tables[4]
    assert pb == book.tables[4][0] and book.refs[pb] == 2
    book.open(5)
    _step(book, [5], [0], [2])                       # no free page: evicts 'c'; 'd' and 'b' are referenced
    assert list(book.cached) == ['d', 'b'] and book.tables[5] == [pc]
    with pytest.raises(DecoderCacheFull):
        book.plan([5], [2], [1])
    assert pd in book.tables[3]
    _consistent(book)


def test_cache_full_counts_free_and_evictable_pages_only():
    book = PageTables(2, max_pages=4, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 4, ['a', 'b'])                  # 2 pages, cached
    book.close(0)
    book.open(2)
    _step(book, [1], [0], [2])                       # 1 free page left, 2 evictable
    assert book.pages_in_use() == 1
    before = _state(book)
    with pytest.raises(DecoderCacheFull, match='needs 4 free pages'):
        book.plan([2], [0], [8])                     # 4 > 1 free + 2 evictable
    with pytest.raises(DecoderCacheFull, match='needs 3 free pages'):
        book.plan([2], [2], [6], hits=[(2, book.lookup(['a']))])    # the hit page is not evictable: 1 + 1 < 3
    assert _state(book) == before
    plan = book.plan([2], [0], [6])                  # 3 = 1 free + 2 evictable
    book.commit(plan, [2])
    assert book.pages_cached() == 0 and book.pages_in_use() == 4


def test_rollback_restores_hits_evictions_and_entries():
    book = PageTables(2, max_pages=7, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 4, ['a', 'b'])
    _prompt(book, 1, 2, ['c'])
    book.close(0), book.close(1)
    book.open(2), book.open(3)
    _step(book, [3], [0], [3])                       # two free pages taken; cloud 3 mid-page
    book.fork(3, 4, 3)
    tables, refs, free, entries = _state(book)[:4]
    hits = [(2, book.lookup(['a']))]
    plan = book.plan([2, 3], [2, 3], [4, 2], hits)   # 2 fresh for cloud 2; copy-on-write and 1 fresh for cloud 3
    copies = book.commit(plan, [2, 3])
    gone = [(k, p) for k, p in entries if k not in book.cached]
    assert copies and [k for k, _ in gone] == ['b', 'c'], 'the step evicted the two least recently used entries it could'
    _consistent(book)
    book.rollback(plan, [2, 3], copies)
    _consistent(book)
    # the evicted entries stay out (the failed step may have written their pages), and their pages are free again
    assert book.tables == tables and list(book.cached.items()) == [e for e in entries if e not in gone]
    assert sorted(book.free) == sorted(free + [p for _, p in gone])
    assert [r for p, r in enumerate(book.refs) if p not in dict(gone).values()] == \
        [r for p, r in enumerate(refs) if p not in dict(gone).values()]


def test_a_page_copied_on_write_is_not_evicted_by_the_same_step_and_rollback_keeps_its_count():
    """A truncates into its registered page 1 and extends with no free page: the copy on write leaves page 1 held by the cache
    alone, but the step's own allocations must not evict it; a rollback gives A its page back with both references."""
    book = PageTables(2, max_pages=5, cache=True)
    for c in 'ABCD':
        book.open(c)
    _prompt(book, 'A', 4, ['a0', 'a1'])
    _prompt(book, 'C', 2, ['c'])
    _prompt(book, 'D', 2, ['d'])
    book.close('C'), book.close('D')
    _step(book, ['B'], [0], [1])                     # the last free page
    book.truncate('A', 3)
    assert book.free == [] and book.n_evictable == 2
    tables, refs = _state(book)[:2]
    plan = book.plan(['A'], [3], [2])
    assert plan.cow == [('A', 1, 1)] and plan.fresh == [1]
    copies = book.commit(plan, ['A'])
    old, new, _ = copies[0]
    assert old == 1 and 1 in book.page_key and book.refs[1] == 1, 'page 1 kept: the cache holds it'
    assert {new, book.tables['A'][2]} == {2, 3} and list(book.cached) == ['a0', 'a1'], 'C\'s and D\'s pages were evicted instead'
    _consistent(book)
    book.rollback(plan, ['A'], copies)
    _consistent(book)
    assert book.tables == tables and book.refs[:2] == refs[:2] == [2, 2] and book.n_evictable == 0
    assert list(book.cached) == ['a0', 'a1'] and sorted(book.free) == [2, 3]


def test_grown_pool_takes_free_then_evicted_pages_before_new_ones():
    book = PageTables(2, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 4, ['a', 'b'])
    book.close(0)
    assert book.reserved == 2 and book.free == []
    _step(book, [1], [0], [8])                       # 4 pages: the 2 evictable, then 2 new
    assert sorted(book.tables[1][:2]) == [0, 1] and book.reserved == 4 and book.pages_cached() == 0


def test_clear_frees_pages_only_the_cache_held():
    book = PageTables(2, cache=True)
    book.open(0), book.open(1)
    _prompt(book, 0, 4, ['a', 'b'])
    _prompt(book, 1, 2, ['c'])
    book.close(1)
    book.clear()
    assert book.pages_cached() == 0 and 2 in book.free and book.refs[:3] == [1, 1, 0] and book.pages_in_use() == 2


def test_without_the_cache_nothing_changes():
    book = PageTables(4)
    book.open(0)
    _step(book, [0], [0], [9])
    assert book.cached is None and book.pages_cached() == 0 and book.lookup(['a']) == []
    book.clear()
    assert book.pages_in_use() == 3


# ---- the host page-key chain ------------------------------------------------------------------------------------------------
def _mix(z):
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & M64
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _keys_statement(d, P):
    keys, k = [], list(PREFIX_SEEDS)
    for q in range(len(d) // P):
        for lane in range(2):
            s = sum(_mix((int(d[q * P + r][lane]) + (r + 1) * PREFIX_GOLD) & M64) for r in range(P)) & M64
            k[lane] = _mix(k[lane] ^ _mix(s))
        keys.append((q, k[0], k[1]))
    return keys


@pytest.mark.parametrize('P, n', [(1, 5), (7, 23), (16, 16), (16, 15), (3, 40)])
def test_page_keys_match_a_pure_python_statement(P, n):
    d = np.random.default_rng(P * 100 + n).integers(0, 2 ** 63, size=(n, 2), dtype=np.uint64) * np.uint64(3)
    assert prefix_page_keys(d, P) == _keys_statement(d, P)


def test_page_keys_name_the_whole_prefix():
    d = np.random.default_rng(1).integers(0, 2 ** 63, size=(40, 2), dtype=np.uint64)
    base = prefix_page_keys(d, 8)
    e = d.copy()
    e[17, 1] ^= np.uint64(1)                         # a node of page 2
    changed = prefix_page_keys(e, 8)
    assert changed[:2] == base[:2] and all(a != b for a, b in zip(changed[2:], base[2:]))
    f = d.copy()
    f[[8, 9]] = f[[9, 8]]                            # two nodes of page 1 swapped
    assert prefix_page_keys(f, 8)[1] != base[1]


# ---- the decoder -------------------------------------------------------------------------------------------------------------
def _dec(page_size=4, max_nodes=None, **extra):
    return SE3Transformer(**{**BASE, 'causal': True, **extra}).packed_decoder(page_size=page_size, max_nodes=max_nodes,
                                                                            prefix_cache=True)


@pytest.mark.parametrize('kw, match', [
    (dict(page_size=4, prefix_cache=1), 'prefix_cache must be a bool'),
    (dict(page_size=4, prefix_cache='yes'), 'prefix_cache must be a bool'),
    (dict(page_size=4, prefix_cache=None), 'prefix_cache must be a bool'),
    (dict(prefix_cache=True), 'give a page_size'),
    (dict(prefix_cache=2), 'prefix_cache must be a bool'),
])
def test_invalid_prefix_cache(kw, match):
    model = SE3Transformer(**{**BASE, 'causal': True})
    with pytest.raises(ValueError, match=f'packed_decoder: .*{match}'):
        model.packed_decoder(**kw)


def test_the_cache_is_off_by_default():
    model = SE3Transformer(**{**BASE, 'causal': True})
    assert model.packed_decoder(page_size=4).prefix_cache is False
    assert model.packed_decoder(page_size=4)._book.cached is None
    d = model.packed_decoder(page_size=4, prefix_cache=True)
    assert d.prefix_cache and d.pages_cached() == 0


def test_counters_and_clear():
    d = _dec(page_size=2)
    a, b = d.open(2)
    paged._step(d._book, [a], [0], [5])               # as the prompt step would, without the device
    d._len[a] = 5
    d._book.register('k0', d._book.tables[a][0])
    d._book.register('k1', d._book.tables[a][1])
    assert d.pages_in_use() == 3 and d.pages_cached() == 2 and d.prefix_nodes(a) == 0
    d._prefix[b] = 4
    d._len[b] = 6
    d.truncate(b, 3)
    assert d.prefix_nodes(b) == 3
    f = d.fork(b)
    assert d.prefix_nodes(f) == 3
    d.close(a)
    assert d.pages_in_use() == 0 and d.pages_cached() == 2
    d.clear_prefix_cache()
    assert d.pages_cached() == 0 and sorted(d._book.free) == [0, 1, 2]
    with pytest.raises(ValueError, match='not an open cloud'):
        d.prefix_nodes(a)


@pytest.mark.parametrize('call, match', paged._PACKED_REFUSALS)
def test_input_refusals_with_the_cache_on(call, match):
    """Every input refusal of PackedCausalDecoder, with its message; clouds, pages and cache entries stay as they were."""
    d = _dec()
    a, b = d.open(2)
    before = paged._state(d), d.pages_cached()
    with pytest.raises(ValueError, match=match):
        call(d, a, b)
    assert (paged._state(d), d.pages_cached()) == before


def test_cpu_inputs_are_refused_before_any_lookup():
    d = _dec()
    a, b = d.open(2)
    with pytest.raises(RuntimeError, match='CUDA'):
        d.extend([a, b], [4, 5], *_x(9))
    assert d.coors is None and d.pages_reserved() == 0 and d.pages_cached() == 0


def test_cache_full_with_the_cache_on_leaves_the_decoder_unchanged():
    """A decode step that does not fit is refused before the device is touched (inputs on the CPU, which the step body would
    refuse, show that the refusal comes first)."""
    d = _dec(page_size=4, max_nodes=8)
    a, b = d.open(2)
    for c in (a, b):                                  # a fixed pool of 2 pages, both taken (as two prompt steps would)
        d._book.commit(d._book.plan([c], [0], [2]), [c])
        d._len[c] = 2
    before = paged._state(d), d.pages_cached()
    with pytest.raises(DecoderCacheFull, match='needs 1 free pages'):
        d.extend([a, b], [3, 1], *_x(4))
    assert (paged._state(d), d.pages_cached()) == before
