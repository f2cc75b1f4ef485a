"""Paged decoding steps replayed from CUDA graphs (DESIGN.md 10.3): the plan kernel against its host statement, the padded
neighbour search against the eager one, and decoders whose every step's rows are torch.equal to the same schedule run eagerly
(SE3B200_NO_DECODE_GRAPHS) on the production route, within 1e-5 on another; no host synchronisation between the descriptor
fill and the post-replay check; plan misses; and the fixed pool."""
import numpy as np
import pytest
import torch

import test_gpu_packed_decode as packed
from test_decode_graphs_host import host_plan, _random_step

DEV = 'cuda'
pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def prod_model():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = packed._model(packed.PROD, seed=5)
    model.pack_weights(free_master=True, max_distance=1.1 * 12 * 3 ** 0.5)      # coordinates in a cube of side 12
    return model


# ---- kernels ------------------------------------------------------------------------------------------------------------------
def _step_desc(g, P, rows_max):
    from se3_transformer_pytorch_b200 import ops
    book, ids, seqlens, n_prev = _random_step(g, P, clouds=int(g.integers(1, 9)), rows_max=rows_max)
    n_cur = [p + m for p, m in zip(n_prev, seqlens)]
    tables = [book.tables[c][:-(-n // P)] for c, n in zip(ids, n_cur)]
    return book, ids, seqlens, n_prev, n_cur, tables


@pytest.mark.parametrize('P', [1, 7, 16])
def test_plan_kernel_matches_its_host_statement_at_every_padding(P):
    from se3_transformer_pytorch_b200 import ops
    g = np.random.default_rng(P)
    long_cloud = False
    for M in range(1, 65):
        book, ids, seqlens, n_prev, n_cur, tables = _step_desc(g, P, M)
        while sum(seqlens) < M:                   # exactly M rows: every padding count of every bucket
            seqlens[0] += 1
            n_cur[0] += 1
            book.commit(book.plan([ids[0]], [n_prev[0]], [seqlens[0]]), [ids[0]])
            tables[0] = book.tables[ids[0]][:-(-n_cur[0] // P)]
        long_cloud |= max(n_cur) > 4097
        rows = 1 << (M - 1).bit_length()
        desc = torch.zeros(ops.decode_desc_words(rows, sum(len(t) for t in tables)), dtype=torch.int32)
        ops.fill_decode_desc(desc, rows, n_prev, seqlens, [1] * len(ids), tables)
        got = ops.decode_plan(desc.to(DEV).view(torch.int64), rows, rows, P, 12345)
        assert torch.equal(got.cpu(), host_plan(desc, rows, rows, P, 12345)), M
    assert long_cloud


@pytest.mark.parametrize('P', [1, 7, 16])
@pytest.mark.parametrize('masks', [False, True])
def test_padded_search_matches_the_eager_search(P, masks):
    from se3_transformer_pytorch_b200 import ops
    g = np.random.default_rng(10 + P)
    for trial in range(6):
        book, ids, seqlens, n_prev, n_cur, tables = _step_desc(g, P, 40)
        M, K = sum(seqlens), min(min(n_cur) - 1, 16)
        rows = 1 << (M - 1).bit_length()
        pool = torch.randn(book.reserved, P, 3, generator=torch.Generator().manual_seed(trial)).to(DEV) * 4
        nbr = [(torch.rand(m, n) > 0.3).to(DEV) for m, n in zip(seqlens, n_cur)] if masks else None
        want = ops.knn_rows_paged(pool, tables, n_prev, seqlens, [K] * len(ids), 5.0, causal=True, neighbor_mask=nbr)
        desc = torch.zeros(ops.decode_desc_words(rows, sum(len(t) for t in tables)), dtype=torch.int32)
        ops.fill_decode_desc(desc, rows, n_prev, seqlens, [K] * len(ids), tables)
        flat = torch.cat([t.reshape(-1) for t in nbr]) if masks else None
        got = ops.knn_rows_paged_bucket(pool, desc.to(DEV).view(torch.int64), rows, rows, book.reserved * P, K, 5.0, causal=True,
                                        neighbor_mask=flat)
        for a, w in zip(got, want):
            assert torch.equal(a[:M], w)
            assert torch.equal(a[M:], w[M - 1:M].expand((rows - M,) + tuple(w.shape[1:])))     # padding repeats row M - 1


# ---- the decoder: every step against the same schedule run eagerly ------------------------------------------------------------
class Twin:
    """The same calls on a decoder that replays graphs and on one whose steps run under SE3B200_NO_DECODE_GRAPHS (the graphed
    one first, so that what it does to shared model state happens before the eager step); every step's rows must agree."""

    def __init__(self, model, P, max_nodes, seed, feats_dim=128, side=12.0, exact=True, pairs=None):
        self.dec, self.ref = (model.packed_decoder(page_size=P, max_nodes=max_nodes) for _ in range(2))
        self.g = torch.Generator().manual_seed(seed)
        self.feats_dim, self.side, self.exact, self.pairs = feats_dim, side, exact, pairs
        self.ids = {}
        self.max_nodes, self.P = max_nodes, P

    def open(self, *names):
        for name, a, b in zip(names, self.dec.open(len(names)), self.ref.open(len(names))):
            self.ids[name] = (a, b)

    def inputs(self, steps):
        M = sum(m for _, m in steps)
        f = torch.randn(M, self.feats_dim, generator=self.g).to(DEV)
        c = (torch.rand(M, 3, generator=self.g) * self.side).to(DEV)
        kw = {}
        if self.pairs:
            n_cur = [self.dec.length(self.ids[n][0]) + m for n, m in steps]
            kw = {name: [make(m, n, self.g) for (_, m), n in zip(steps, n_cur)] for name, make in self.pairs.items()}
        return f, c, kw

    def extend(self, *steps, inputs=None):
        from se3_transformer_pytorch_b200 import switches
        f, c, kw = inputs or self.inputs(steps)
        got = self.dec.extend([self.ids[n][0] for n, _ in steps], [m for _, m in steps], f, c, **kw)
        with switches.override(no_decode_graphs=True):
            want = self.ref.extend([self.ids[n][1] for n, _ in steps], [m for _, m in steps], f, c, **kw)
        if not self.exact:
            assert packed._errs(got, want) < 1e-5
        elif isinstance(want, dict):
            packed._assert_equal(got, want)
        else:
            assert torch.equal(got, want)
        assert self.dec.pages_reserved() == self.ref.pages_reserved() == -(-self.max_nodes // self.P)
        assert self.dec.pages_in_use() == self.ref.pages_in_use()
        return got

    def fork(self, src, name):
        self.ids[name] = (self.dec.fork(self.ids[src][0]), self.ref.fork(self.ids[src][1]))

    def truncate(self, name, n):
        self.dec.truncate(self.ids[name][0], n)
        self.ref.truncate(self.ids[name][1], n)

    def close(self, name):
        self.dec.close(self.ids[name][0])
        self.ref.close(self.ids[name][1])
        del self.ids[name]


def _schedule(t):
    """Joins, closes, forks, a truncate into a shared page, multi-row steps, prompt steps among decode steps, and M at every
    power of two up to 64 and at 65."""
    names = [f'c{i}' for i in range(40)]
    t.open(*names[:20])
    t.extend(*[(n, 17 + i) for i, n in enumerate(names[:20])])         # prompts (k_c = 16 from 17 nodes on)
    t.extend(('c0', 1))                                                  # M = 1
    t.extend(('c1', 1), ('c2', 1))                                       # M = 2
    t.extend(('c3', 2), ('c4', 1), ('c5', 1))                            # M = 4, multi-row
    t.open(*names[20:24])
    t.extend(('c6', 1), ('c20', 17))                                     # a join: a prompt step with a decode row
    t.extend(*[(n, 1) for n in names[:8]])                               # M = 8
    t.close('c7')
    t.fork('c8', 'f8')                                                   # c8 at 25 nodes: inside its second page
    t.fork('f8', 'ff8')                                                  # a fork of a fork
    t.extend(('f8', 2), ('ff8', 1), ('c8', 1))                           # copies on write
    t.extend(*[(n, 1) for n in names[:7] + names[8:17]])                 # M = 16
    t.fork('c9', 'f9')
    t.truncate('f9', 19)                                                 # into the middle of a page c9 still holds
    t.extend(('c9', 1), ('f9', 3))
    t.extend(*[(n, 1) for n in names[:7] + names[8:20]], *[(n, 2) for n in ('f8', 'ff8', 'f9')], ('c20', 7))   # M = 32
    t.extend(('c21', 17), ('c22', 17), ('c0', 1))                        # prompts again
    rest = names[:7] + names[8:20] + names[21:23]
    t.extend(*[(n, 1) for n in rest], *[(n, 3) for n in ('f8', 'ff8', 'f9')], ('c23', 17), ('c20', 17))   # M = 64 (c23's prompt)
    rest.append('c23')
    t.extend(*[(n, 1) for n in rest], *[(n, 3) for n in ('f8', 'ff8', 'f9')], ('c20', 33))                # M = 64
    t.extend(*[(n, 1) for n in rest], *[(n, 3) for n in ('f8', 'ff8', 'f9')], ('c20', 34))                # M = 65
    for _ in range(3):                                                   # replays of captured buckets
        t.extend(*[(n, 1) for n in names[:5]])
        t.extend(('c1', 1))


def test_graph_schedule_is_bit_identical_to_eager_steps(prod_model):
    t = Twin(prod_model, P=16, max_nodes=4096, seed=0)
    _schedule(t)
    assert t.dec.graph_replays >= 10 and t.ref.graph_replays == 0
    assert {rows for rows, _ in t.dec.graph_capture_s} == {1, 2, 4, 8, 16, 32, 64}


def test_pages_of_one_node_and_odd_pages(prod_model):
    for P in (1, 7):
        t = Twin(prod_model, P=P, max_nodes=3000, seed=P)
        t.open('a', 'b', 'c')
        t.extend(('a', 30), ('b', 19), ('c', 20))
        for i in range(4):
            t.extend(('a', 1), ('b', 1 + i), ('c', 2))
        t.fork('b', 'd')
        t.truncate('d', 22)
        t.extend(('b', 1), ('d', 2))
        assert t.dec.graph_replays == 5


# ---- other inputs ----------------------------------------------------------------------------------------------------------------
def _edge_model(kind):
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=5, valid_radius=10, causal=True, edge_dim=3,
               **({'num_edge_tokens': 4} if kind == 'tokens' else {}))
    return packed._model(cfg, seed=3)


def _short_schedule(t):
    t.open('a', 'b', 'c')
    t.extend(('a', 30), ('b', 20), ('c', 17))
    for i in range(5):
        t.extend(('a', 1), ('b', 1), ('c', 1 + i % 2))
    t.fork('a', 'd')
    t.extend(('a', 2), ('d', 1))
    t.extend(('a', 1), ('b', 1), ('c', 1), ('d', 1))
    assert t.dec.graph_replays == 7


@pytest.mark.parametrize('kind', ['tokens', 'float'])
def test_edges_and_neighbor_masks(kind):
    model = _edge_model(kind)
    edge = (lambda m, n, g: torch.randint(0, 4, (m, n), generator=g).to(DEV)) if kind == 'tokens' else \
        (lambda m, n, g: torch.randn(m, n, 3, generator=g).to(DEV))
    mask = lambda m, n, g: (torch.rand(m, n, generator=g) > 0.3).to(DEV)
    for pairs in (dict(edges=edge), dict(edges=edge, neighbor_mask=mask)):
        _short_schedule(Twin(model, P=4, max_nodes=200, seed=1, feats_dim=16, side=3.0, exact=False, pairs=pairs))


def test_neighbor_masks_on_the_production_route(prod_model):
    mask = lambda m, n, g: (torch.rand(m, n, generator=g) > 0.2).to(DEV)
    _short_schedule(Twin(prod_model, P=8, max_nodes=300, seed=2, pairs=dict(neighbor_mask=mask)))


def test_rotary_positions():
    from varlen_helpers import load_varlen
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_rotary_causal')
    model = packed._model(cfg['ctor'])
    _short_schedule(Twin(model, P=3, max_nodes=500, seed=3, feats_dim=cfg['ctor']['dim'], side=3.0, exact=False))


def test_non_production_route_within_tolerance():
    cfg = dict(dim=16, heads=2, dim_head=8, depth=2, num_degrees=3, num_neighbors=6, valid_radius=10, causal=True)
    _short_schedule(Twin(packed._model(cfg, seed=4), P=5, max_nodes=300, seed=4, feats_dim=16, side=3.0, exact=False))


# ---- no synchronisation ---------------------------------------------------------------------------------------------------------
def test_replay_makes_no_host_synchronisation(prod_model, monkeypatch):
    from se3_transformer_pytorch_b200 import model as model_mod, ops
    t = Twin(prod_model, P=16, max_nodes=1024, seed=5)
    t.open('a', 'b')
    t.extend(('a', 20), ('b', 30))
    t.extend(('a', 1), ('b', 1))                  # captures bucket (2, 16)
    fill, check = ops.fill_decode_desc, model_mod.check_lowrank_stats
    windows = []

    def fill_then_forbid(*a, **kw):
        out = fill(*a, **kw)
        torch.cuda.set_sync_debug_mode('error')
        windows.append(1)
        return out

    def allow_then_check(checks):
        torch.cuda.set_sync_debug_mode(0)
        return check(checks)
    monkeypatch.setattr(ops, 'fill_decode_desc', fill_then_forbid)
    monkeypatch.setattr(model_mod, 'check_lowrank_stats', allow_then_check)
    try:
        before = t.dec.graph_replays
        for _ in range(3):
            t.dec.extend([t.ids['a'][0], t.ids['b'][0]], [1, 1], *t.inputs([('a', 1), ('b', 1)])[:2])
        assert t.dec.graph_replays == before + 3 and len(windows) == 3
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---- plan misses -----------------------------------------------------------------------------------------------------------------
def test_plan_miss_with_masters_drops_the_graphs_and_equals_eager():
    from se3_transformer_pytorch_b200 import ops, switches
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = packed._model(packed.PROD, seed=5)
    model.pack_weights(max_distance=1.1 * 12 * 3 ** 0.5)
    with switches.override(lowrank_min_edges=1):  # decode steps have few edges: take the low-rank route anyway
        t = Twin(model, P=8, max_nodes=500, seed=6)
        t.open('a', 'b')
        t.extend(('a', 20), ('b', 20))
        t.extend(('a', 1), ('b', 1))
        t.extend(('a', 1), ('b', 1))
        assert t.dec.graph_replays == 2 and t.dec._graphs
        f, c, _ = t.inputs([('a', 1), ('b', 1)])
        c[1] = torch.tensor([80.0, 80.0, 80.0])   # far beyond the plan's range
        t.extend(('a', 1), ('b', 1), inputs=(f, c, {}))
        assert not t.dec._graphs
        t.extend(('a', 1), ('b', 1))
        assert t.dec._graphs


def test_plan_miss_with_released_masters_raises_and_changes_nothing(prod_model):
    from se3_transformer_pytorch_b200.model import LowRankPlanMiss
    t = Twin(prod_model, P=8, max_nodes=500, seed=7)
    t.open('a', 'b')
    t.extend(('a', 20), ('b', 20))
    t.extend(('a', 1), ('b', 1))
    t.fork('a', 'c')                              # a at 21 nodes: the next step copies a shared page on write
    dec = t.dec
    ids = [t.ids[n][0] for n in ('a', 'b', 'c')]
    state = lambda: ([dec.length(i) for i in ids], {i: list(p) for i, p in dec._book.tables.items()}, dec.pages_in_use(),
                     list(dec._book.free))
    before, replays = state(), dec.graph_replays
    f, c, _ = t.inputs([('a', 2), ('b', 1), ('c', 1)])
    c[0] = torch.tensor([1e4, 1e4, 1e4])
    with pytest.raises(LowRankPlanMiss):
        dec.extend(ids, [2, 1, 1], f, c)
    assert dec.graph_replays == replays + 1 and state() == before and not dec._graphs
    t.extend(('a', 2), ('b', 1), ('c', 1))        # the decoder goes on as if the step was never sent


# ---- the fixed pool --------------------------------------------------------------------------------------------------------------
def test_fixed_pool_and_cache_full(prod_model):
    from se3_transformer_pytorch_b200 import DecoderCacheFull
    P = 8
    t = Twin(prod_model, P=P, max_nodes=64, seed=8)
    t.open('a', 'b')
    t.extend(('a', 30), ('b', 20))
    t.extend(('a', 1), ('b', 2))
    dec = t.dec
    state = lambda: (dec.open_ids(), {i: list(p) for i, p in dec._book.tables.items()}, dec.pages_in_use(), dec.pages_reserved())
    before = state()
    f, c, _ = t.inputs([('a', 12), ('b', 12)])
    with pytest.raises(DecoderCacheFull):
        dec.extend([t.ids['a'][0], t.ids['b'][0]], [12, 12], f, c)
    assert state() == before
    t.extend(('a', 1), ('b', 2))                  # fits in the pages the clouds hold
    t.close('b')
    t.extend(('a', 20))
    assert dec.graph_replays == 3 and dec.pages_reserved() == 8


# ---- low-rank plans that eager steps can still rebuild (masters kept) ------------------------------------------------------------
def _masters_model():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = packed._model(packed.PROD, seed=5)
    model.pack_weights(max_distance=1.1 * 12 * 3 ** 0.5)
    return model


def _plan_range(model):
    return model.conv_modules()[0]._packed['lr']['D']


def test_a_capture_that_rebuilds_the_plan_drops_the_graphs_of_the_old_plan():
    from se3_transformer_pytorch_b200 import switches
    model = _masters_model()
    with switches.override(lowrank_min_edges=1):  # decode steps have few edges: take the low-rank route anyway
        t = Twin(model, P=8, max_nodes=600, seed=9)
        t.open('a', 'b')
        t.extend(('a', 20), ('b', 20))
        t.extend(('a', 1))
        t.extend(('a', 1))                        # bucket 1 captured and replayed
        assert [k[:2] for k in t.dec._graphs] == [(1, 16)] and t.dec.graph_replays == 2
        D = _plan_range(model)
        f, c, _ = t.inputs([('a', 1), ('b', 1)])
        c[1] = torch.tensor([40.0, 40.0, 40.0])   # bucket 2: its warm-up meets distances beyond D and rebuilds the plan
        t.extend(('a', 1), ('b', 1), inputs=(f, c, {}))
        assert _plan_range(model) > D
        assert [k[:2] for k in t.dec._graphs] == [(2, 16)]
        t.extend(('a', 1))                        # bucket 1 again, captured anew against the new plan
        t.extend(('a', 1))
        assert sorted(k[:2] for k in t.dec._graphs) == [(1, 16), (2, 16)] and t.dec.graph_replays == 5


def test_a_step_just_beyond_the_plan_range_runs_eagerly():
    from se3_transformer_pytorch_b200 import switches
    model = _masters_model()
    # radial coordinates from the trunk, not the plan's table: the table flags every distance past D itself, the trunk's residual
    # check only one that leaves the plan's subspace, which a distance just past D need not do
    with switches.override(lowrank_min_edges=1, no_utable=True):
        t = Twin(model, P=8, max_nodes=600, seed=10)
        t.open('a')
        coords = []
        for m in (20, 1, 1):                      # bucket 1 captured and replayed
            f, c, _ = t.inputs([('a', m)])
            coords.append(c)
            t.extend(('a', m), inputs=(f, c, {}))
        assert t.dec._graphs and t.dec.graph_replays == 2
        D = _plan_range(model)
        prev = torch.cat(coords).double().cpu()
        u = torch.ones(3, dtype=torch.float64) / 3 ** 0.5
        kth = lambda s: float((prev - (prev.mean(0) + s * u)).norm(dim=1).sort().values[15])
        lo, hi = 0.0, 10 * D
        for _ in range(100):                      # the new node's 16th nearest neighbour, its farthest, at 1.002 D
            mid = (lo + hi) / 2
            lo, hi = (mid, hi) if kth(mid) < 1.002 * D else (lo, mid)
        f, _, _ = t.inputs([('a', 1)])
        c = (prev.mean(0) + hi * u).float()[None].to(DEV)
        t.extend(('a', 1), inputs=(f, c, {}))     # the eager step rebuilds its plan: the replay must not keep the old one
        assert _plan_range(model) > D and not t.dec._graphs and t.dec.graph_replays == 3
        t.extend(('a', 1))
        assert t.dec._graphs and t.dec.graph_replays == 4


# ---- the descriptor's room ---------------------------------------------------------------------------------------------------------
def test_descriptor_room_grows_with_the_pages_a_step_reads(prod_model):
    t = Twin(prod_model, P=1, max_nodes=3000, seed=11)
    t.open('a')
    t.extend(('a', 1020))
    for _ in range(8):                            # 1021 .. 1028 pages of one node: the room of 1024 ids is outgrown
        t.extend(('a', 1))
    assert [g.room for g in t.dec._graphs.values()] == [2048] and t.dec.graph_replays == 8
