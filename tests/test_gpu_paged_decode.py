"""PagedCausalDecoder (SE3Transformer.packed_decoder(page_size=...)): the neighbour search through block tables equals the
contiguous search, and the paged decoder's rows equal forward and the unpaged packed decoder on schedules with joins, leaves,
forks of forks, truncates into shared pages and pool growth; forks share memory, and a capped pool refuses a step unchanged."""
import numpy as np
import pytest
import torch

import test_gpu_packed_decode as packed
from helpers import load_case, case_inputs
from varlen_helpers import load_varlen

DEV = 'cuda'
pytestmark = pytest.mark.gpu


# ---- the neighbour search through block tables -----------------------------------------------------------------------------
def _check_paged_rows(clouds, P, permute, radius=2.5, seed=0):
    """clouds: [(n_prev, m, k, neighbour mask [m, n_cur] or None)], each cloud's coordinates in one row of a contiguous store and
    in pages of P nodes of a pool (in order, or at randomly permuted page ids); ops.knn_rows_paged against ops.knn_rows_packed."""
    from se3_transformer_pytorch_b200 import ops
    n_prev, ms, ks, masks = zip(*clouds)
    n_cur = [p + m for p, m in zip(n_prev, ms)]
    ld = max(n_cur) + 5
    g = torch.Generator().manual_seed(seed)
    store = torch.randn(len(clouds), ld, 3, generator=g).to(DEV)
    counts = [-(-n // P) for n in n_cur]
    order = torch.randperm(sum(counts) + 3, generator=g).tolist() if permute else list(range(sum(counts) + 3))
    tables, at = [], 0
    pool = torch.full((sum(counts) + 3, P, 3), float('nan'), device=DEV)
    for c, n in enumerate(n_cur):
        tables.append(order[at:at + counts[c]])
        at += counts[c]
        for q, page in enumerate(tables[c]):
            rows = store[c, q * P:min(n, (q + 1) * P)]
            pool[page, :rows.shape[0]] = rows
    nbr = None if all(t is None for t in masks) else list(masks)
    want = ops.knn_rows_packed(store, range(len(clouds)), n_prev, ms, ks, radius, causal=True, neighbor_mask=nbr)
    idx, col, mask, rel_pos, rel_dist = ops.knn_rows_paged(pool, tables, n_prev, ms, ks, radius, causal=True, neighbor_mask=nbr)
    slot = torch.repeat_interleave(torch.arange(len(clouds)), torch.tensor(ms)).to(DEV)
    assert torch.equal(col, want[0] - slot[:, None] * ld)
    flat = torch.tensor([p for t in tables for p in t], device=DEV)
    start = torch.repeat_interleave(torch.tensor([0] + counts[:-1]).cumsum(0), torch.tensor(ms)).to(DEV)
    assert torch.equal(idx, flat[start[:, None] + col // P] * P + col % P)
    assert torch.equal(pool.view(-1, 3)[idx], store.view(-1, 3)[want[0]])
    for a, w in zip((mask, rel_pos, rel_dist), want[1:]):
        assert torch.equal(a, w)


@pytest.mark.parametrize('P', [1, 3, 16, 64])
@pytest.mark.parametrize('permute', [False, True])
def test_paged_rows_several_rows_per_cloud(P, permute):
    _check_paged_rows([(30, 5, 16, None), (0, 12, 11, None), (3, 2, 4, None), (1, 1, 1, None), (200, 7, 32, None)], P, permute)


@pytest.mark.parametrize('P', [1, 3, 16, 64])
def test_paged_rows_tiled_branch_beside_a_two_node_cloud(P):
    _check_paged_rows([(0, 2, 1, None), (4990, 10, 16, None), (1, 2, 2, None)], P, True, radius=10.0, seed=1)


@pytest.mark.parametrize('P', [1, 3, 16, 64])
def test_paged_rows_with_neighbour_masks_on_some_clouds(P):
    g = torch.Generator().manual_seed(3)
    masks = [(torch.rand(m, n, generator=g) > 0.3).to(DEV) for m, n in ((4, 70), (3, 9))]
    _check_paged_rows([(66, 4, 16, masks[0]), (20, 6, 16, None), (6, 3, 8, masks[1])], P, True, seed=2)


# ---- the model: the same schedule on the paged and the unpaged decoder -------------------------------------------------------
class Twin:
    """Runs every call on a paged and an unpaged packed decoder, asserts that each step's rows are torch.equal, and keeps every
    cloud's nodes and output rows so that they can be checked against forward."""

    def __init__(self, model, page_size, seed, feats_dim=128, side=12.0, **kw):
        self.paged, self.ref = model.packed_decoder(page_size=page_size, **kw), model.packed_decoder()
        self.g = torch.Generator().manual_seed(seed)
        self.feats_dim, self.side = feats_dim, side
        self.ids, self.nodes, self.outs = {}, {}, {}

    def open(self, *names):
        for name, a, b in zip(names, self.paged.open(len(names)), self.ref.open(len(names))):
            self.ids[name], self.nodes[name], self.outs[name] = (a, b), [], []

    def extend(self, *steps):
        f = torch.randn(sum(m for _, m in steps), self.feats_dim, generator=self.g).to(DEV)
        c = (torch.rand(f.shape[0], 3, generator=self.g) * self.side).to(DEV)
        got = self.paged.extend([self.ids[n][0] for n, _ in steps], [m for _, m in steps], f, c)
        want = self.ref.extend([self.ids[n][1] for n, _ in steps], [m for _, m in steps], f, c)
        packed._assert_equal(got, want)
        at = 0
        for n, m in steps:
            self.nodes[n] += [(f[at + r], c[at + r]) for r in range(m)]
            self.outs[n] += [{d: v[at + r] for d, v in got.items()} for r in range(m)]
            at += m
            assert self.paged.length(self.ids[n][0]) == self.ref.length(self.ids[n][1]) == len(self.nodes[n])

    def fork(self, src, name):
        self.ids[name] = (self.paged.fork(self.ids[src][0]), self.ref.fork(self.ids[src][1]))
        self.nodes[name], self.outs[name] = list(self.nodes[src]), list(self.outs[src])

    def truncate(self, name, n):
        self.paged.truncate(self.ids[name][0], n)
        self.ref.truncate(self.ids[name][1], n)
        del self.nodes[name][n:], self.outs[name][n:]

    def close(self, name, model=None):
        if model is not None:
            self.check(model, name)
        self.paged.close(self.ids[name][0])
        self.ref.close(self.ids[name][1])
        del self.ids[name]

    def check(self, model, name):
        """The cloud's rows so far are torch.equal to one forward over its nodes."""
        f = torch.stack([x for x, _ in self.nodes[name]])
        c = torch.stack([y for _, y in self.nodes[name]])
        full = packed._forward(model, f, c)
        packed._assert_equal({d: torch.stack([o[d] for o in self.outs[name]]) for d in full}, full)


def test_paged_schedule_is_bit_identical_to_forward_and_to_the_unpaged_decoder(prod_model):
    t = Twin(prod_model, page_size=16, seed=0)
    t.open('a', 'b')
    t.extend(('a', 40), ('b', 19))
    t.extend(('a', 1), ('b', 2))
    t.open('c')
    t.extend(('a', 1), ('c', 30))                  # a join
    freed = set(t.paged._book.tables[t.ids['b'][0]])
    t.close('b', prod_model)                       # a leave: b's pages are free ...
    t.open('d')
    t.extend(('d', 20), ('c', 1))                  # ... and taken first
    assert freed <= set(t.paged._book.tables[t.ids['d'][0]]) | set(t.paged._book.tables[t.ids['c'][0]])
    t.fork('a', 'a1')                              # a at 42 nodes: inside page 2
    t.fork('a1', 'a2')                             # a fork of a fork
    t.extend(('a1', 3), ('a2', 1))                 # both copy page 2 on write; a keeps it
    t.close('a', prod_model)                       # a fork whose parent then closes
    t.extend(('a1', 1), ('a2', 5), ('c', 2))
    t.fork('a2', 'a3')                             # a2 at 48 nodes: a page boundary
    t.truncate('a3', 37)                           # into the middle of a page a2 still holds
    t.extend(('a2', 2), ('a3', 4))                 # siblings of one shared page in the same step
    t.check(prod_model, 'a2')
    reserved = t.paged.pages_reserved()
    t.fork('d', 'd1')
    t.truncate('d1', 5)                            # inside d's first page
    short = reserved - t.paged.pages_in_use()
    t.extend(('d1', 16 * (short + 2)), ('a3', 1))  # needs more pages than are free, and one copy on write: the pool grows
    assert t.paged.pages_reserved() > reserved
    t.extend(('d', 1), ('d1', 1), ('c', 1), ('a1', 1), ('a2', 1), ('a3', 1))
    for name in list(t.ids):
        t.check(prod_model, name)
    assert t.paged.pages_in_use() == len({p for name in t.ids for p in t.paged._book.tables[t.ids[name][0]]})


@pytest.fixture(scope='module')
def prod_model():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = packed._model(packed.PROD, seed=5)
    model.pack_weights(free_master=True, max_distance=1.1 * 12 * 3 ** 0.5)
    return model


@pytest.mark.parametrize('P', [1, 3, 16])
def test_paged_production_decode_matches_forward(prod_model, P):
    """The packed decoder's production schedule, paged with pages smaller than, near and past its steps."""
    lens = [300, 37, 150, 90]
    clouds = packed._prod_clouds(lens, 0)
    schedule = [[(0, 120)], [(0, 1), (1, 2)], [(0, 1), (1, 1), (2, 60)]]
    schedule += [[(0, 1), (1, 1), (2, 1), (3, 2)]] * 12 + [[(0, 3), (2, 1), (3, 1)]] * 8
    sent = [sum(m for step in schedule for i, m in step if i == c) for c in range(4)]
    schedule.append([(c, n - s) for c, (n, s) in enumerate(zip(lens, sent))])
    _, res = packed._run(prod_model.packed_decoder(page_size=P), clouds, schedule)
    for (f, c), out in zip(clouds, res):
        packed._assert_equal(out, packed._forward(prod_model, f, c))


# ---- pair inputs and the reference fixtures (within 1e-5, as the packed decoder) ---------------------------------------------
@pytest.mark.parametrize('edge_kind', ['tokens', 'float'])
def test_edges_and_neighbor_masks_match_forward(edge_kind):
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=5, valid_radius=10, causal=True, edge_dim=3,
               **({'num_edge_tokens': 4} if edge_kind == 'tokens' else {}))
    model = packed._model(cfg, seed=3)
    g = torch.Generator().manual_seed(0)
    lens = [21, 9, 14]
    clouds = [(torch.randn(n, 16, generator=g).to(DEV), torch.randn(n, 3, generator=g).to(DEV)) for n in lens]
    edges = [(torch.randint(0, 4, (n, n), generator=g) if edge_kind == 'tokens' else torch.randn(n, n, 3, generator=g)).to(DEV)
             for n in lens]
    nbr = [(torch.rand(n, n, generator=g) > 0.3).to(DEV) for n in lens]
    _, res = packed._run(model.packed_decoder(page_size=4), clouds, packed._schedule(lens, 'staggered', seed=2),
                         pairs=dict(edges=edges, neighbor_mask=nbr))
    for (f, c), out, e, m in zip(clouds, res, edges, nbr):
        assert packed._errs(out, packed._forward(model, f, c, edges=e[None], neighbor_mask=m[None])) < 1e-5


@pytest.mark.parametrize('P', [3, 16])
def test_rotary_causal_fixture_matches_forward(P):
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_rotary_causal')
    model = packed._model(cfg['ctor'])
    starts = np.cumsum([0] + seqlens[:-1])
    clouds = [(packed._t(feats[s:s + n]), packed._t(coors[s:s + n])) for s, n in zip(starts, seqlens)]
    _, res = packed._run(model.packed_decoder(page_size=P), clouds, packed._schedule(seqlens, 'sit_out'), **cfg['fwd'])
    for (f, c), out in zip(clouds, res):
        assert packed._errs(out, packed._forward(model, f, c, **cfg['fwd'])) < 1e-5


@pytest.mark.parametrize('P', [2, 5])
def test_causal_fixture_matches_forward(P):
    z, cfg = load_case('causal')
    feats, coors, mask, extra = case_inputs(z)
    model = packed._model(cfg['ctor'])
    lens = [16, 7, 11]
    clouds = [(packed._t(feats[0, :n]), packed._t(coors[0, :n])) for n in lens]
    _, res = packed._run(model.packed_decoder(page_size=P), clouds, packed._schedule(lens, 'staggered', seed=1), **cfg['fwd'])
    for (f, c), out in zip(clouds, res):
        assert packed._errs(out, packed._forward(model, f, c, **cfg['fwd'])) < 1e-5


# ---- memory ------------------------------------------------------------------------------------------------------------------
def test_fork_allocates_nothing_and_forks_share_their_prefix(prod_model):
    P, n, W, g = 16, 2000, 6, 20
    (f, c), = packed._prod_clouds([n + W * g], 4)
    dec = prod_model.packed_decoder(page_size=P)
    a, = dec.open()
    dec.extend([a], [n], f[:n], c[:n])
    torch.cuda.synchronize()
    mem, pages = torch.cuda.memory_allocated(), dec.pages_in_use()
    forks = [dec.fork(a) for _ in range(W)]
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == mem and dec.pages_in_use() == pages == -(-n // P)
    for _ in range(g):
        dec.extend(forks, [1] * W, f[n:n + W], c[n:n + W])
    assert dec.pages_in_use() <= -(-n // P) + W * (-(-g // P) + 1)


def test_cache_full_leaves_the_decoder_as_if_the_step_was_never_sent(prod_model):
    from se3_transformer_pytorch_b200 import DecoderCacheFull
    P = 8
    (fa, ca), (fb, cb) = packed._prod_clouds([60, 60], 5)
    runs = []
    for refused in (False, True):
        dec = prod_model.packed_decoder(page_size=P, max_nodes=64)
        a, b = dec.open(2)
        dec.extend([a, b], [30, 20], torch.cat((fa[:30], fb[:20])), torch.cat((ca[:30], cb[:20])))
        assert dec.pages_reserved() == 8 and dec.pages_in_use() == 7
        if refused:
            state = (dec.open_ids(), [dec.length(i) for i in (a, b)], {i: list(t) for i, t in dec._book.tables.items()},
                     dec.pages_in_use())
            with pytest.raises(DecoderCacheFull):
                dec.extend([a, b], [12, 12], torch.cat((fa[30:42], fb[20:32])), torch.cat((ca[30:42], cb[20:32])))
            assert state == (dec.open_ids(), [dec.length(i) for i in (a, b)],
                             {i: list(t) for i, t in dec._book.tables.items()}, dec.pages_in_use())
        outs = [dec.extend([a, b], [2, 5], torch.cat((fa[30:32], fb[20:25])), torch.cat((ca[30:32], cb[20:25])))]
        dec.close(b)
        outs.append(dec.extend([a], [20], fa[32:52], ca[32:52]))
        runs.append(outs)
    for got, want in zip(*runs):
        packed._assert_equal(got, want)
