"""The prefix cache of PagedCausalDecoder (DESIGN.md 10.4): se3_prefix_keys_fwd bit for bit against a numpy statement of its
digest, what the digest covers, and decoders with the cache whose every step's rows are torch.equal to the same schedule on a
decoder without it on the production route (within 1e-5 elsewhere): full and partial hits, pair inputs, tokens, rotary
positions, mixed steps, copy-on-write of a cached page, eviction and DecoderCacheFull, graph-replayed steps after a hit, and the
cache cleared when a switch or a plan changes."""
import numpy as np
import pytest
import torch

import test_gpu_packed_decode as packed

DEV = 'cuda'
pytestmark = pytest.mark.gpu
U64 = np.uint64
SEEDS = (U64(0x243F6A8885A308D3), U64(0x13198A2E03707344))
GOLD = U64(0x9E3779B97F4A7C15)


# ---- the digest, restated in numpy ---------------------------------------------------------------------------------------------
def _mix(z):
    z = z ^ (z >> U64(30))
    z = z * U64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> U64(27))
    z = z * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def np_digest(feat, xyz, i, edge=None, mask=None):
    """Node i's two lanes from its conv_in row feat (float32 [W]), coordinates (float32 [3]), edge row (int64 [n] or float32
    [n, E]) and mask row (bool [n]): per lane, mix64 of the wrapping sum of mix64(word ^ mix64(seed + (4 k + tag + 1) G))."""
    words, idx = [feat.view(np.uint32).astype(U64), xyz.view(np.uint32).astype(U64)], \
        [4 * np.arange(feat.size, dtype=U64) + U64(1), 4 * np.arange(3, dtype=U64) + U64(2)]
    if edge is not None:
        e = edge[:i].reshape(-1)
        words.append(e.view(U64) if e.dtype == np.int64 else e.view(np.uint32).astype(U64))
        idx.append(4 * np.arange(e.size, dtype=U64) + U64(3))
    if mask is not None:
        words.append(mask[:i].astype(U64))
        idx.append(4 * np.arange(i, dtype=U64) + U64(4))
    w, k = np.concatenate(words), np.concatenate(idx)
    with np.errstate(over='ignore'):
        return [int(_mix(_mix(w ^ _mix(seed + k * GOLD)).sum(dtype=U64))) for seed in SEEDS]


def _keys(feats, coors, seqlens, n_prev=None, edges=None, masks=None):
    from se3_transformer_pytorch_b200 import ops
    got = ops.prefix_keys(feats.to(DEV), coors.to(DEV), seqlens, n_prev, edges=None if edges is None else [e.to(DEV) for e in edges],
                          neighbor_mask=None if masks is None else [m.to(DEV) for m in masks])
    return got.cpu().numpy().view(U64)


def _statement(feats, coors, seqlens, n_prev=None, edges=None, masks=None):
    n_prev = n_prev or [0] * len(seqlens)
    out, at = [], 0
    for c, (m, p) in enumerate(zip(seqlens, n_prev)):
        for r in range(m):
            out.append(np_digest(feats[at + r].numpy(), coors[at + r].numpy(), p + r,
                                 None if edges is None else edges[c][r].numpy(), None if masks is None else masks[c][r].numpy()))
        at += m
    return np.array(out, dtype=U64)


@pytest.mark.parametrize('pairs', [None, 'tokens', 'float', 'mask', 'tokens+mask', 'float+mask'])
@pytest.mark.parametrize('width', [1, 13, 128, 300])
def test_prefix_keys_match_the_numpy_statement(pairs, width):
    g = torch.Generator().manual_seed(width)
    seqlens, n_prev = [5, 1, 40, 3], [0, 7, 0, 130]
    M = sum(seqlens)
    feats, coors = torch.randn(M, width, generator=g), torch.randn(M, 3, generator=g)
    feats[0, 0] = -0.0
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    edges = masks = None
    if pairs and 'tokens' in pairs:
        edges = [torch.randint(-2 ** 40, 2 ** 40, (m, n), generator=g) for m, n in zip(seqlens, n_cur)]
    if pairs and 'float' in pairs:
        edges = [torch.randn(m, n, 3, generator=g) for m, n in zip(seqlens, n_cur)]
    if pairs and 'mask' in pairs:
        masks = [torch.rand(m, n, generator=g) > 0.4 for m, n in zip(seqlens, n_cur)]
    got = _keys(feats, coors, seqlens, n_prev, edges, masks)
    assert np.array_equal(got, _statement(feats, coors, seqlens, n_prev, edges, masks))


def test_prefix_keys_of_one_row_and_two_input_degrees():
    g = torch.Generator().manual_seed(1)
    f0, f1 = torch.randn(1, 7, 1, generator=g), torch.randn(1, 7, 3, generator=g)
    feats = torch.cat([f0.reshape(1, -1), f1.reshape(1, -1)], dim=1)          # the decoder's layout for input_degrees = 2
    coors = torch.randn(1, 3, generator=g)
    assert np.array_equal(_keys(feats, coors, [1]), _statement(feats, coors, [1]))


@pytest.mark.parametrize('P', [1, 7, 16])
def test_page_keys_from_kernel_digests(P):
    from se3_transformer_pytorch_b200.model import prefix_page_keys
    g = torch.Generator().manual_seed(P)
    n = 3 * P + 2
    feats, coors = torch.randn(n, 40, generator=g), torch.randn(n, 3, generator=g)
    edges = [torch.randint(0, 5, (n, n), generator=g)]
    got = _keys(feats, coors, [n], edges=edges)
    assert np.array_equal(got, _statement(feats, coors, [n], edges=edges))
    keys = prefix_page_keys(got, P)
    assert [k[0] for k in keys] == list(range(n // P))
    feats[2 * P, 5] = feats[2 * P, 5] + 1.0
    changed = prefix_page_keys(_keys(feats, coors, [n], edges=edges), P)
    assert changed[:2] == keys[:2] and all(a != b for a, b in zip(changed[2:], keys[2:]))


def test_digest_covers_columns_before_the_node_only():
    g = torch.Generator().manual_seed(2)
    n, i = 12, 7
    feats, coors = torch.randn(n, 20, generator=g), torch.randn(n, 3, generator=g)
    edges = [torch.randn(n, n, 2, generator=g)]
    masks = [torch.rand(n, n, generator=g) > 0.5]
    base = _keys(feats, coors, [n], edges=edges, masks=masks)

    def flipped(t, at):                               # one bit of entry `at`
        t = t.clone()
        if t.dtype == torch.bool:
            t[at] = ~t[at]
        else:
            t.view(torch.int32)[at] ^= 1
        return t
    for j in range(n):                                # edge value and mask of column j of row i
        for which in ('edge', 'mask'):
            e = [flipped(edges[0], (i, j, 1))] if which == 'edge' else edges
            m = [flipped(masks[0], (i, j))] if which == 'mask' else masks
            got = _keys(feats, coors, [n], edges=e, masks=m)
            assert np.array_equal(np.delete(got, i, 0), np.delete(base, i, 0))
            assert (not np.array_equal(got[i], base[i])) == (j < i), (which, j)
    for k in range(20):
        got = _keys(flipped(feats, (i, k)), coors, [n], edges=edges, masks=masks)
        assert not np.array_equal(got[i], base[i]) and np.array_equal(np.delete(got, i, 0), np.delete(base, i, 0))
    for k in range(3):
        got = _keys(feats, flipped(coors, (i, k)), [n], edges=edges, masks=masks)
        assert not np.array_equal(got[i], base[i])


# ---- decoders with and without the cache ----------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def prod_model():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = packed._model(packed.PROD, seed=5)
    model.pack_weights(free_master=True, max_distance=1.1 * 12 * 3 ** 0.5)      # coordinates in a cube of side 12
    return model


class Pair:
    """The same schedule on a decoder with the prefix cache and on one without it (eagerly, with eager_ref); each request's
    inputs are given whole and consumed in order.  Every step's rows must agree: torch.equal, or within 1e-5 (exact=False)."""

    def __init__(self, model, P, max_nodes=None, exact=True, eager_ref=False):
        self.dec = model.packed_decoder(page_size=P, max_nodes=max_nodes, prefix_cache=True)
        self.ref = model.packed_decoder(page_size=P, max_nodes=max_nodes)
        self.P, self.exact, self.eager_ref = P, exact, eager_ref
        self.ids, self.data, self.done = {}, {}, {}

    def open(self, name, feats, coors, **pairs):
        self.ids[name] = (self.dec.open()[0], self.ref.open()[0])
        self.data[name] = (feats, coors, pairs)
        self.done[name] = 0

    def inputs(self, steps):
        fs, cs, kw = [], [], {}
        for name, m in steps:
            f, c, pairs = self.data[name]
            n0, n1 = self.done[name], self.done[name] + m
            fs.append(packed._rows(f, n0, n1))
            cs.append(c[n0:n1])
            for key, t in pairs.items():
                kw.setdefault(key, []).append(t[n0:n1, :n1])
        return packed._cat(fs), torch.cat(cs), kw

    def extend(self, *steps):
        from se3_transformer_pytorch_b200 import switches
        f, c, kw = self.inputs(steps)
        got = self.dec.extend([self.ids[n][0] for n, _ in steps], [m for _, m in steps], f, c, **kw)
        with switches.override(no_decode_graphs=self.eager_ref):
            want = self.ref.extend([self.ids[n][1] for n, _ in steps], [m for _, m in steps], f, c, **kw)
        if not self.exact:
            assert packed._errs(got, want) < 1e-5
        elif isinstance(want, dict):
            packed._assert_equal(got, want)
        else:
            assert torch.equal(got, want)
        for name, m in steps:
            self.done[name] += m
        return got

    def truncate(self, name, n):
        self.dec.truncate(self.ids[name][0], n)
        self.ref.truncate(self.ids[name][1], n)
        self.done[name] = n

    def close(self, name):
        self.dec.close(self.ids[name][0])
        self.ref.close(self.ids[name][1])

    def prefix(self, name):
        return self.dec.prefix_nodes(self.ids[name][0])


def _cloud(n, g, dim=128, side=12.0):
    return torch.randn(n, dim, generator=g).to(DEV), (torch.rand(n, 3, generator=g) * side).to(DEV)


def _with_tail(f, c, keep, tail, g, dim=128, side=12.0):
    tf, tc = _cloud(tail, g, dim, side)
    return torch.cat([f[:keep], tf]), torch.cat([c[:keep], tc])


def test_a_separate_request_with_the_same_prompt_hits_its_full_pages(prod_model):
    P = 16
    g = torch.Generator().manual_seed(0)
    t = Pair(prod_model, P)
    fa, ca = _cloud(5 * P + 3 + 4, g)
    t.open('A', fa, ca)
    t.extend(('A', 5 * P + 3))
    assert t.prefix('A') == 0 and t.dec.pages_cached() == 5
    t.open('B', *_with_tail(fa, ca, 5 * P + 3, 14, g))
    t.extend(('B', 5 * P + 13))
    assert t.prefix('B') == 5 * P
    assert t.dec.pages_in_use() == 7 and t.ref.pages_in_use() == 12, 'the 5 shared pages are counted once'
    for _ in range(4):
        t.extend(('A', 1), ('B', 1))


def test_partial_hits_stop_at_the_first_page_that_differs(prod_model):
    P = 16
    g = torch.Generator().manual_seed(1)
    t = Pair(prod_model, P)
    fa, ca = _cloud(5 * P + 3, g)
    t.open('A', fa, ca)
    t.extend(('A', 5 * P + 3))
    fc = fa.clone()
    fc[2 * P + 1, 3] = (fc[2 * P + 1, 3].view(torch.int32) ^ 1).view(torch.float32)        # one bit of node 2P + 1
    t.open('C', fc, ca)
    t.extend(('C', 5 * P + 3))
    assert t.prefix('C') == 2 * P
    cd = ca.clone()
    cd[4 * P, 2] = (cd[4 * P, 2].view(torch.int32) ^ 1).view(torch.float32)                 # one bit of a coordinate
    t.open('D', fa, cd)
    t.extend(('D', 5 * P + 3))
    assert t.prefix('D') == 4 * P


def _edge_model(kind):
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=5, valid_radius=10, causal=True, edge_dim=3,
               **({'num_edge_tokens': 4} if kind == 'tokens' else {}))
    return packed._model(cfg, seed=3)


@pytest.mark.parametrize('kind', ['tokens', 'float'])
def test_edges_decide_hits_only_through_columns_before_the_node(kind):
    P, n = 4, 22
    g = torch.Generator().manual_seed(2)
    model = _edge_model(kind)
    e = torch.randint(0, 4, (n, n), generator=g).to(DEV) if kind == 'tokens' else torch.randn(n, n, 3, generator=g).to(DEV)
    f, c = _cloud(n, g, dim=16, side=3.0)
    t = Pair(model, P, exact=False)
    t.open('A', f, c, edges=e)
    t.extend(('A', n))
    e2 = e.clone()
    e2[13, 9] = (e2[13, 9] + 1) % 4 if kind == 'tokens' else e2[13, 9] + 0.5     # j < i: node 13's page (3) misses
    t.open('B', f, c, edges=e2)
    t.extend(('B', n))
    assert t.prefix('B') == 3 * P
    e3 = e.clone()
    e3[13, 17] = (e3[13, 17] + 1) % 4 if kind == 'tokens' else e3[13, 17] + 0.5   # j >= i: nothing a row reads
    e3[13, 13] = (e3[13, 13] + 1) % 4 if kind == 'tokens' else e3[13, 13] + 0.5
    t.open('C', f, c, edges=e3)
    t.extend(('C', n))
    assert t.prefix('C') == 5 * P


def test_neighbor_masks_on_the_production_route(prod_model):
    P, n = 8, 45
    g = torch.Generator().manual_seed(3)
    f, c = _cloud(n + 4, g)
    nm = (torch.rand(n + 4, n + 4, generator=g) > 0.2).to(DEV)
    t = Pair(prod_model, P)
    t.open('A', f, c, neighbor_mask=nm)
    t.extend(('A', n))
    nm2 = nm.clone()
    nm2[30, 11] = ~nm2[30, 11]                       # j < i in page 3
    t.open('B', f, c, neighbor_mask=nm2)
    t.extend(('B', n))
    assert t.prefix('B') == 3 * P
    t.open('C', f, c, neighbor_mask=nm)
    t.extend(('C', n), ('A', 2))
    assert t.prefix('C') == 5 * P
    t.extend(('A', 1), ('B', 2), ('C', 1))


def test_tokens_with_positions():
    P, n = 5, 31
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=6, valid_radius=10, causal=True, num_tokens=7,
               num_positions=64)
    model = packed._model(cfg, seed=6)
    g = torch.Generator().manual_seed(4)
    tok = torch.randint(0, 7, (n,), generator=g).to(DEV)
    c = (torch.rand(n, 3, generator=g) * 3).to(DEV)
    t = Pair(model, P, exact=False)
    t.open('A', tok, c)
    t.extend(('A', n - 2))
    t.open('B', tok, c)
    t.extend(('B', n - 4))
    assert t.prefix('B') == 5 * P
    t.extend(('A', 2), ('B', 4))


def test_rotary_positions():
    from varlen_helpers import load_varlen
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_rotary_causal')
    model = packed._model(cfg['ctor'])
    P, dim = 3, cfg['ctor']['dim']
    g = torch.Generator().manual_seed(5)
    f, c = _cloud(26, g, dim=dim, side=3.0)
    t = Pair(model, P, exact=False)
    t.open('A', f, c)
    t.extend(('A', 20))
    t.open('B', *_with_tail(f, c, 20, 4, g, dim=dim, side=3.0))
    t.extend(('B', 22))
    assert t.prefix('B') == 6 * P
    t.extend(('A', 3), ('B', 2))


def test_a_step_mixing_cached_prompts_and_decode_rows(prod_model, monkeypatch):
    from se3_transformer_pytorch_b200 import ops
    P = 16
    g = torch.Generator().manual_seed(6)
    t = Pair(prod_model, P, max_nodes=2048)
    fa, ca = _cloud(6 * P + 8, g)
    t.open('A', fa, ca)
    t.open('X', *_cloud(40, g))
    t.extend(('A', 5 * P + 3), ('X', 30))
    t.open('D', fa, ca)                               # fully cached: exactly A's first 5 pages
    t.open('E', *_with_tail(fa, ca, 3 * P + 2, 24, g))  # partly cached: 3 pages
    t.extend(('A', 1), ('D', 5 * P), ('X', 2), ('E', 3 * P + 22))
    assert t.prefix('D') == 5 * P and t.prefix('E') == 3 * P
    t.open('F', fa, ca)
    f, c, _ = t.inputs([('F', 4 * P)])

    def no_search(*a, **kw):
        raise AssertionError('a fully cached prompt searched neighbours')
    with monkeypatch.context() as patch:
        patch.setattr(ops, 'knn_rows_paged', no_search)
        got = t.dec.extend([t.ids['F'][0]], [4 * P], f, c)      # alone in its step: no neighbour search, no step body
    packed._assert_equal(got, t.ref.extend([t.ids['F'][1]], [4 * P], f, c))
    t.done['F'] += 4 * P
    assert t.prefix('F') == 4 * P
    t.extend(('A', 1), ('D', 1), ('E', 1), ('F', 1), ('X', 1))


def test_copy_on_write_keeps_cached_pages(prod_model):
    P = 16
    g = torch.Generator().manual_seed(7)
    t = Pair(prod_model, P, max_nodes=1024)          # free pages enough: no entry is evicted
    fa, ca = _cloud(4 * P, g)
    t.open('A', fa, ca)
    first = t.extend(('A', 4 * P))
    t.truncate('A', 2 * P + 5)                        # into registered page 2
    t.data['A'] = _with_tail(fa, ca, 2 * P + 5, 3 * P, g) + ({},)
    t.extend(('A', 3 * P))                            # other nodes: page 2 is copied on write
    t.open('C', fa, ca)
    again = t.extend(('C', 4 * P))
    assert t.prefix('C') == 4 * P
    packed._assert_equal(again, first)


def test_eviction_and_cache_full_under_max_nodes(prod_model):
    from se3_transformer_pytorch_b200 import DecoderCacheFull
    P = 16
    g = torch.Generator().manual_seed(8)
    t = Pair(prod_model, P, max_nodes=12 * P)
    fa, ca = _cloud(5 * P + 3, g)
    t.open('A', fa, ca)
    t.extend(('A', 5 * P + 3))
    t.close('A')
    assert t.dec.pages_in_use() == 0 and t.dec.pages_cached() == 5
    t.open('X', *_cloud(10 * P, g))
    t.extend(('X', 10 * P))                           # 7 free pages, then 3 of A's, least recently used first
    assert t.dec.pages_cached() == 12 and t.dec.pages_in_use() == 10
    assert [k[0] for k in t.dec._book.cached][:2] == [3, 4], 'A\'s pages 0 .. 2 went first'

    t.open('B', fa, ca)
    dec, b = t.dec, t.ids['B'][0]
    before = (dec.pages_in_use(), dec.pages_cached(), list(dec._book.cached.items()), list(dec._book.free), dec.length(b))
    f, c, _ = t.inputs([('B', 5 * P + 3)])
    with pytest.raises(DecoderCacheFull):
        dec.extend([b], [5 * P + 3], f, c)            # A's page 0 was evicted: a miss, and 6 pages > 0 free + 2 evictable
    assert (dec.pages_in_use(), dec.pages_cached(), list(dec._book.cached.items()), list(dec._book.free), dec.length(b)) == before
    assert dec.prefix_nodes(b) == 0


def test_a_failed_step_drops_the_entries_it_evicted(prod_model):
    """S's pages are evicted for T, whose inputs equal S's but for one mask entry j < i of page 0; T's step writes them and then
    fails (a node beyond the low-rank plan's range).  S's entries must not come back: a later request with S's prompt misses."""
    from se3_transformer_pytorch_b200 import switches
    from se3_transformer_pytorch_b200.model import LowRankPlanMiss
    P = 16
    g = torch.Generator().manual_seed(12)
    with switches.override(lowrank_min_edges=1):      # prompts this small take the low-rank route too
        t = Pair(prod_model, P, max_nodes=4 * P)
        fs, cs = _cloud(2 * P, g)
        nm = (torch.rand(2 * P, 2 * P, generator=g) > 0.2).to(DEV)
        t.open('S', fs, cs, neighbor_mask=nm)
        t.extend(('S', 2 * P))
        t.close('S')
        t.open('X', *_cloud(2 * P, g))
        t.extend(('X', 2 * P))                         # the pool's last free pages: S's two pages are the only spare ones
        dec = t.dec
        assert dec.pages_cached() == 4 and dec.pages_in_use() == 2
        nm_t = nm.clone()
        nm_t[9, 4] = ~nm_t[9, 4]
        ct = cs.clone()
        ct[-1] = torch.tensor([1e4, 1e4, 1e4])
        tid = dec.open()[0]
        with pytest.raises(LowRankPlanMiss):
            dec.extend([tid], [2 * P], fs, ct, neighbor_mask=[nm_t])
        assert dec.length(tid) == 0 and dec.pages_in_use() == 2
        assert dec.pages_cached() == 2 and all(p not in dec._book.page_key for p in range(dec.pages_reserved())
                                               if p not in dec._book.tables[t.ids['X'][0]])
        dec.close(tid)
        t.open('U', fs, cs, neighbor_mask=nm)
        t.extend(('U', 2 * P))                         # rows equal to the decoder without the cache
        assert t.prefix('U') == 0


def test_graph_steps_after_a_hit_equal_eager_steps(prod_model):
    P = 16
    g = torch.Generator().manual_seed(9)
    t = Pair(prod_model, P, max_nodes=1024, eager_ref=True)
    fa, ca = _cloud(3 * P + 20, g)
    t.open('A', fa, ca)
    t.extend(('A', 3 * P + 2))
    t.open('B', *_with_tail(fa, ca, 3 * P + 2, 20, g))
    t.extend(('B', 3 * P + 5), ('A', 1))
    assert t.prefix('B') == 3 * P
    for i in range(6):
        t.extend(('A', 1), ('B', 1 + i % 2))
    assert t.dec.graph_replays >= 5 and t.ref.graph_replays == 0


def test_a_switch_or_plan_change_clears_the_cache(prod_model):
    from se3_transformer_pytorch_b200 import switches
    P = 16
    g = torch.Generator().manual_seed(10)
    t = Pair(prod_model, P)
    fa, ca = _cloud(3 * P, g)
    t.open('A', fa, ca)
    t.extend(('A', 3 * P))
    assert t.dec.pages_cached() == 3
    with switches.override(edge_budget_mb=4096):
        t.open('B', fa, ca)
        t.extend(('B', 3 * P))
        assert t.prefix('B') == 0 and t.dec.pages_cached() == 3, 'entries of the old switches were dropped, B registered'
    t.open('C', fa, ca)
    t.extend(('C', 3 * P))
    assert t.prefix('C') == 0
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=6, valid_radius=10, causal=True)
    model = packed._model(cfg, seed=7)
    t = Pair(model, 4, exact=False)
    f, c = _cloud(20, g, dim=16, side=3.0)
    t.open('A', f, c)
    t.extend(('A', 20))
    conv = model.conv_modules()[0]
    conv._lr_blocked = not conv._lr_blocked           # the route of one ConvSE3 changes
    t.open('B', f, c)
    t.extend(('B', 20))
    assert t.prefix('B') == 0
    t.open('C', f, c)
    t.extend(('C', 20))
    assert t.prefix('C') == 20


def test_non_production_route_within_tolerance():
    cfg = dict(dim=16, heads=2, dim_head=8, depth=2, num_degrees=3, num_neighbors=6, valid_radius=10, causal=True)
    model = packed._model(cfg, seed=4)
    g = torch.Generator().manual_seed(11)
    t = Pair(model, 5, exact=False)
    f, c = _cloud(40, g, dim=16, side=3.0)
    t.open('A', f, c)
    t.extend(('A', 27))
    t.open('B', *_with_tail(f, c, 27, 9, g, dim=16, side=3.0))
    t.extend(('B', 33), ('A', 2))
    assert t.prefix('B') == 25
    t.extend(('A', 1), ('B', 3))
