"""PackedCausalDecoder (SE3Transformer.packed_decoder): clouds of different lengths decoded together on ragged schedules give,
for every cloud, the rows of one forward over that cloud alone -- against the reference fixtures, against forward within 1e-5,
and bit for bit on the production path -- across close, truncate, fork and cache growth; and the ragged new-row search equals
the single-cloud search."""
import numpy as np
import pytest
import torch

from detfill import fill_state_dict
from helpers import load_case, rel_err, case_inputs, case_outputs
from varlen_helpers import load_varlen, varlen_outputs

DEV = 'cuda'
pytestmark = pytest.mark.gpu


def _model(cfg, seed=11):
    from se3_transformer_pytorch_b200 import SE3Transformer
    model = SE3Transformer(**cfg)
    fill_state_dict(model, seed=seed)
    return model.to(DEV).eval()


def _rows(x, n0, n1):
    return {d: v[n0:n1] for d, v in x.items()} if isinstance(x, dict) else x[n0:n1]


def _cat(parts):
    if isinstance(parts[0], dict):
        return {d: torch.cat([p[d] for p in parts]) for d in parts[0]}
    return torch.cat(parts)


def _run(dec, clouds, schedule, ids=None, pairs=None, **kw):
    """Decode clouds [(feats [n, ...] or {d: [n, ...]}, coors [n, 3])] on `schedule`, a list of steps [(cloud, m), ...]; pairs:
    {name: one [n, n, ...] tensor per cloud}.  Returns (ids, each cloud's outputs concatenated)."""
    ids = dec.open(len(clouds)) if ids is None else ids
    done, outs = [0] * len(clouds), [[] for _ in clouds]
    for step in schedule:
        f, c, extra = [], [], {name: [] for name in (pairs or {})}
        for i, m in step:
            n0, n1 = done[i], done[i] + m
            f.append(_rows(clouds[i][0], n0, n1))
            c.append(clouds[i][1][n0:n1])
            for name, per in (pairs or {}).items():
                extra[name].append(per[i][n0:n1, :n1])
        out = dec.extend([ids[i] for i, _ in step], [m for _, m in step], _cat(f), torch.cat(c), **extra, **kw)
        at = 0
        for i, m in step:
            outs[i].append(_rows(out, at, at + m))
            at += m
            done[i] += m
            assert dec.length(ids[i]) == done[i]
    return ids, [_cat(o) for o in outs]


def _schedule(lens, kind, seed=0):
    """Steps of 1 .. 3 nodes per cloud (the first of each cloud >= 2).  'staggered': cloud c joins at step 2c; 'sit_out': every
    cloud but the first sits out every third step in turn."""
    rng = np.random.default_rng(seed)
    left, steps, t = list(lens), [], 0
    while any(left):
        step = []
        for c, n in enumerate(lens):
            if not left[c] or (kind == 'staggered' and t < 2 * c) or (kind == 'sit_out' and c and (t + c) % 3 == 0):
                continue
            m = min(left[c], int(rng.integers(1, 4)) + (left[c] == n))
            step.append((c, m))
            left[c] -= m
        if step:
            steps.append(step)
        t += 1
    return steps


def _errs(res, ref):
    res = res if isinstance(res, dict) else {'': res}
    ref = ref if isinstance(ref, dict) else {'': ref}
    return max(rel_err(np.asarray(res[d].cpu() if torch.is_tensor(res[d]) else res[d]),
                       np.asarray(ref[d].cpu() if torch.is_tensor(ref[d]) else ref[d])) for d in ref)


def _forward(model, feats, coors, **kw):
    out = model(feats[None] if torch.is_tensor(feats) else {d: v[None] for d, v in feats.items()}, coors[None], **kw)
    return {d: v[0] for d, v in out.items()} if isinstance(out, dict) else out[0]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---- the ragged new-row search ---------------------------------------------------------------------------------------------
def _check_rows(store, clouds, radius=2.5):
    """clouds: [(slot, n_prev, m, k, neighbour mask [m, n_cur] or None)]; each cloud's rows of ops.knn_rows_packed against
    ops.knn_rows on that cloud alone."""
    from se3_transformer_pytorch_b200 import ops
    slots, n_prev, ms, ks, masks = zip(*clouds)
    got = ops.knn_rows_packed(store, slots, n_prev, ms, ks, radius, causal=True,
                              neighbor_mask=None if all(t is None for t in masks) else list(masks))
    K, ld = max(ks), store.shape[1]
    assert got[0].shape == (sum(ms), K)
    at = 0
    for s, p, m, k, nbr in clouds:
        want = ops.knn_rows(store[s:s + 1], p + m, p, m, k, radius, causal=True, neighbor_mask=None if nbr is None else nbr[None])
        idx, mask, rel_pos, rel_dist = (t[at:at + m] for t in got)
        assert torch.equal(idx[:, :k] - s * ld, want[0][0])
        for a, w in zip((mask, rel_pos, rel_dist), want[1:]):
            assert torch.equal(a[:, :k], w[0])
        assert not mask[:, k:].any()
        for a in (idx, rel_pos, rel_dist):
            assert torch.equal(a[:, k:], a[:, k - 1:k].expand_as(a[:, k:]))
        at += m


def _store(S, ld, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S, ld, 3, generator=g).to(DEV)


def test_ragged_rows_several_rows_per_cloud_and_short_clouds():
    store = _store(4, 64)
    _check_rows(store, [(3, 30, 5, 16, None), (0, 0, 12, 11, None), (2, 3, 2, 4, None), (1, 1, 1, 1, None)])


def test_ragged_rows_tiled_branch_beside_a_tiny_cloud():
    store = _store(2, 5008, seed=2)
    _check_rows(store, [(1, 0, 3, 2, None), (0, 4990, 10, 16, None)], radius=10.0)


def test_ragged_rows_with_and_without_neighbour_masks():
    g = torch.Generator().manual_seed(3)
    store = _store(3, 96, seed=4)
    masks = [(torch.rand(m, n, generator=g) > 0.3).to(DEV) for m, n in ((4, 70), (3, 9))]
    _check_rows(store, [(2, 66, 4, 16, masks[0]), (0, 20, 6, 16, None), (1, 6, 3, 8, masks[1])])


# ---- the reference fixtures ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['staggered', 'sit_out'])
def test_rotary_causal_fixture_decodes_to_reference(kind):
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_rotary_causal')
    assert not pairs
    ref = varlen_outputs(z)
    model = _model(cfg['ctor'])
    starts = np.cumsum([0] + seqlens[:-1])
    clouds = [(_t(feats[s:s + n]), _t(coors[s:s + n])) for s, n in zip(starts, seqlens)]
    _, res = _run(model.packed_decoder(), clouds, _schedule(seqlens, kind), **cfg['fwd'])
    for (f, c), out, s, n in zip(clouds, res, starts, seqlens):
        want = {d: v[s:s + n] for d, v in ref.items()} if isinstance(ref, dict) else ref[s:s + n]
        assert _errs(out, want) < 1e-4, n
        assert _errs(out, _forward(model, f, c, **cfg['fwd'])) < 1e-5, n


@pytest.mark.parametrize('kind', ['staggered', 'sit_out'])
def test_causal_fixture_decodes_to_reference(kind):
    """The fixture's cloud of 16 beside its prefixes of 7 and 11 nodes, whose reference rows are the first rows of the cloud's."""
    z, cfg = load_case('causal')
    feats, coors, mask, extra = case_inputs(z)
    assert not extra and mask.all() and coors.shape[0] == 1
    ref = case_outputs(z)
    model = _model(cfg['ctor'])
    lens = [16, 7, 11]
    clouds = [(_t(feats[0, :n]), _t(coors[0, :n])) for n in lens]
    _, res = _run(model.packed_decoder(), clouds, _schedule(lens, kind, seed=1), **cfg['fwd'])
    for (f, c), out, n in zip(clouds, res, lens):
        want = {d: v[0, :n] for d, v in ref.items()} if isinstance(ref, dict) else ref[0, :n]
        assert _errs(out, want) < 1e-4, n
        assert _errs(out, _forward(model, f, c, **cfg['fwd'])) < 1e-5, n


# ---- the production route: bit for bit -------------------------------------------------------------------------------------
PROD = dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=3, output_degrees=2, num_neighbors=16, valid_radius=10, causal=True)


def _prod_clouds(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, 128, generator=g).to(DEV), (torch.rand(n, 3, generator=g) * 12).to(DEV)) for n in lens]


@pytest.fixture(scope='module')
def prod_model():
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    model = _model(PROD, seed=5)
    model.pack_weights(free_master=True, max_distance=1.1 * 12 * 3 ** 0.5)      # _prod_clouds: coordinates in a cube of side 12
    return model


def _assert_equal(res, full):
    for d in full:
        assert torch.equal(res[d], full[d]), (d, float((res[d] - full[d]).abs().max()))


def test_production_decode_is_bit_identical_to_forward(prod_model):
    from se3_transformer_pytorch_b200 import ops
    lens = [300, 37, 150, 90]
    clouds = _prod_clouds(lens, 0)
    schedule = [[(0, 120)], [(0, 1), (1, 2)], [(0, 1), (1, 1), (2, 60)]]
    schedule += [[(0, 1), (1, 1), (2, 1), (3, 2)]] * 12 + [[(0, 3), (2, 1), (3, 1)]] * 8
    sent = [sum(m for step in schedule for i, m in step if i == c) for c in range(4)]
    schedule.append([(c, n - s) for c, (n, s) in enumerate(zip(lens, sent))])
    before = ops.SPLIT_LAUNCHES
    _, res = _run(prod_model.packed_decoder(), clouds, schedule)
    assert ops.SPLIT_LAUNCHES > before, 'no production GEMM of the steps ran split-K'
    for (f, c), out in zip(clouds, res):
        _assert_equal(out, _forward(prod_model, f, c))


# ---- lifecycle ----------------------------------------------------------------------------------------------------------------
def test_closed_slot_is_reused_exactly(prod_model):
    (fa, ca), (fb, cb), (fc, cc) = _prod_clouds([40, 30, 25], 1)
    dec = prod_model.packed_decoder()
    a, b = dec.open(2)
    dec.extend([a, b], [20, 10], torch.cat((fa[:20], fb[:10])), torch.cat((ca[:20], cb[:10])))
    dec.close(a)
    c, = dec.open()
    assert dec._slot[c] == 0
    _, (res,) = _run(dec, [(fc, cc)], [[(0, 4)], [(0, 1)], [(0, 20)]], ids=[c])
    _, (fresh,) = _run(prod_model.packed_decoder(), [(fc, cc)], [[(0, 2)], [(0, 23)]])
    _assert_equal(res, fresh)
    _assert_equal(res, _forward(prod_model, fc, cc))


def test_truncate_and_fork_continue_exactly(prod_model):
    (f, c), (f2, c2), (f3, c3) = _prod_clouds([50, 50, 50], 2)
    dec = prod_model.packed_decoder()
    a, = dec.open()
    dec.extend([a], [30], f[:30], c[:30])
    dec.truncate(a, 18)                            # rewind, then continue with different nodes: f[:18] + f2[18:]
    g, gc = torch.cat((f[:18], f2[18:])), torch.cat((c[:18], c2[18:]))
    out = dec.extend([a], [12], g[18:30], gc[18:30])
    b = dec.fork(a)                                # two continuations of the same 30-node prefix
    h, hc = torch.cat((g[:30], f3[30:])), torch.cat((gc[:30], c3[30:]))
    o = dec.extend([a, b], [20, 20], torch.cat((g[30:], h[30:])), torch.cat((gc[30:], hc[30:])))
    res_a = _cat([out, _rows(o, 0, 20)])
    res_b = _rows(o, 20, 40)
    full_g, full_h = _forward(prod_model, g, gc), _forward(prod_model, h, hc)
    _assert_equal(res_a, _rows(full_g, 18, 50))
    _assert_equal(res_b, _rows(full_h, 30, 50))


def test_slot_and_capacity_growth_keep_every_cloud_exact(prod_model):
    lens = [70, 9, 40, 33, 12]
    clouds = _prod_clouds(lens, 3)
    dec = prod_model.packed_decoder()
    ids, done, outs = {}, [0] * len(lens), [[] for _ in lens]

    def step(pairs):
        f = _cat([_rows(clouds[i][0], done[i], done[i] + m) for i, m in pairs])
        c = torch.cat([clouds[i][1][done[i]:done[i] + m] for i, m in pairs])
        out, at = dec.extend([ids[i] for i, _ in pairs], [m for _, m in pairs], f, c), 0
        for i, m in pairs:
            outs[i].append(_rows(out, at, at + m))
            at, done[i] = at + m, done[i] + m
    ids[0], = dec.open()
    step([(0, 2)])
    ids[1], ids[2] = dec.open(2)                   # three clouds in a one-row cache: the slot axis grows
    step([(0, 10), (1, 3), (2, 14)])
    step([(0, 1), (2, 1)])
    step([(0, 20), (1, 6)])                        # cloud 0 reaches 33 nodes: cap grows past 16
    dec.close(ids[1])
    ids[3], ids[4] = dec.open(2)                   # one takes the freed row 1, one row 3: the slot axis grows again
    assert [dec._slot[ids[i]] for i in (3, 4)] == [1, 3]
    step([(0, 37), (2, 25), (3, 33), (4, 12)])     # cap grows past 64
    assert dec.S >= 4 and dec.cap >= 70 and done == lens
    for i, cloud in enumerate(clouds):
        _assert_equal(_cat(outs[i]), _forward(prod_model, *cloud))


# ---- pair inputs ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('edge_kind', ['tokens', 'float'])
def test_edges_and_neighbor_masks_match_forward(edge_kind):
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=5, valid_radius=10, causal=True, edge_dim=3,
               **({'num_edge_tokens': 4} if edge_kind == 'tokens' else {}))
    model = _model(cfg, seed=3)
    g = torch.Generator().manual_seed(0)
    lens = [21, 9, 14]
    clouds = [(torch.randn(n, 16, generator=g).to(DEV), torch.randn(n, 3, generator=g).to(DEV)) for n in lens]
    edges = [(torch.randint(0, 4, (n, n), generator=g) if edge_kind == 'tokens' else torch.randn(n, n, 3, generator=g)).to(DEV)
             for n in lens]
    nbr = [(torch.rand(n, n, generator=g) > 0.3).to(DEV) for n in lens]
    _, res = _run(model.packed_decoder(), clouds, _schedule(lens, 'staggered', seed=2), pairs=dict(edges=edges, neighbor_mask=nbr))
    for (f, c), out, e, m in zip(clouds, res, edges, nbr):
        assert _errs(out, _forward(model, f, c, edges=e[None], neighbor_mask=m[None])) < 1e-5
