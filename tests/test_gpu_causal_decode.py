"""CausalDecoder (SE3Transformer.causal_decoder): decoding a causal model node by node gives the rows of one forward over all
nodes -- against the reference fixtures, against forward within 1e-5, and bit for bit on the production path, where the step's
production GEMMs run split-K -- and the new-row neighbour search equals the whole-cloud search on the valid slots."""
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
    return {d: v[:, n0:n1] for d, v in x.items()} if isinstance(x, dict) else x[:, n0:n1]


def _decode(model, feats, coors, steps, b=1, mask=None, pairs=None, **kw):
    """Outputs of extend() over `steps` (node counts per call), concatenated along the node axis."""
    dec = model.causal_decoder(batch_size=b)
    outs, n0 = [], 0
    for m in steps:
        n1 = n0 + m
        extra = {k: v[:, n0:n1, :n1] for k, v in (pairs or {}).items()}
        outs.append(dec.extend(_rows(feats, n0, n1), coors[:, n0:n1], None if mask is None else mask[:, n0:n1], **extra, **kw))
        n0 = n1
        assert len(dec) == n1
    if isinstance(outs[0], dict):
        return {d: torch.cat([o[d] for o in outs], dim=1) for d in outs[0]}
    return torch.cat(outs, dim=1)


def _errs(res, ref):
    res = res if isinstance(res, dict) else {'': res}
    ref = ref if isinstance(ref, dict) else {'': ref}
    return max(rel_err(np.asarray(res[d].cpu() if torch.is_tensor(res[d]) else res[d]), np.asarray(ref[d].cpu() if torch.is_tensor(ref[d]) else ref[d])) for d in ref)


def _steps(n, pattern):
    """Node counts per extend() call: a 2-node prefill then single nodes, or 3, 1, 5 and the rest (cut to n nodes)."""
    out, left = [], n
    for m in ([2] + [1] * n) if pattern == 'single' else [3, 1, 5, n]:
        if left > 0:
            out.append(min(m, left))
            left -= out[-1]
    return out


@pytest.mark.parametrize('pattern', ['single', 'uneven'])
def test_causal_fixture_decodes_to_reference(pattern):
    z, cfg = load_case('causal')
    feats, coors, mask, extra = case_inputs(z)
    assert not extra and mask.all()
    model = _model(cfg['ctor'])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    feats = {k: t(v) for k, v in feats.items()} if isinstance(feats, dict) else t(feats)
    n = coors.shape[1]
    res = _decode(model, feats, t(coors), _steps(n, pattern), **cfg['fwd'])
    assert _errs(res, case_outputs(z)) < 1e-4
    full = model(feats, t(coors), **cfg['fwd'])
    assert _errs(res, full) < 1e-5


@pytest.mark.parametrize('pattern', ['single', 'uneven'])
def test_rotary_causal_fixture_decodes_to_reference(pattern):
    """varlen_rotary_causal: every cloud decoded on its own against the reference's per-cloud output."""
    z, cfg, feats, coors, seqlens, pairs = load_varlen('varlen_rotary_causal')
    assert not pairs
    ref = varlen_outputs(z)
    model = _model(cfg['ctor'])
    s = 0
    for n in seqlens:
        f = torch.from_numpy(np.ascontiguousarray(feats[s:s + n]))[None].to(DEV)
        c = torch.from_numpy(np.ascontiguousarray(coors[s:s + n]))[None].to(DEV)
        res = _decode(model, f, c, _steps(n, pattern), **cfg['fwd'])
        want = {d: v[s:s + n][None] for d, v in ref.items()} if isinstance(ref, dict) else ref[s:s + n][None]
        assert _errs(res, want) < 1e-4, n
        assert _errs(res, model(f, c, **cfg['fwd'])) < 1e-5, n
        s += n


PROD = dict(dim=128, heads=2, dim_head=64, depth=1, num_degrees=3, output_degrees=2, num_neighbors=16, valid_radius=10, causal=True)


def _production_model(coors):
    model = _model(PROD, seed=5)
    d = float(torch.cdist(coors.float(), coors.float()).max())
    model.pack_weights(free_master=True, max_distance=1.1 * d)
    return model


@pytest.mark.parametrize('b', [1, 2])
def test_production_decode_is_bit_identical_to_forward(b):
    from detfill import det_inputs
    from se3_transformer_pytorch_b200 import ops
    if not ops.tc_supported(DEV, 128, 1):
        pytest.skip('needs sm_90')
    n = 300
    feats = torch.from_numpy(det_inputs('decode/feats', (b, n, 128), 1)).to(DEV)
    coors = torch.from_numpy(det_inputs('decode/coors', (b, n, 3), 2) * 3).to(DEV)
    mask = None
    if b == 2:
        mask = torch.ones((b, n), dtype=torch.bool, device=DEV)
        mask[1, 7::11] = False
    model = _production_model(coors)
    full = model(feats, coors, mask)
    before = ops.SPLIT_LAUNCHES
    steps = [2] + [1] * 30 + [47, 5] + [1] * 16
    steps.append(n - sum(steps))
    res = _decode(model, feats, coors, steps, b=b, mask=mask)
    assert ops.SPLIT_LAUNCHES > before, 'no production GEMM of the steps ran split-K'
    for d in full:
        assert torch.equal(res[d], full[d]), (d, float((res[d] - full[d]).abs().max()))


def test_edge_tokens_and_neighbor_mask_match_forward():
    cfg = dict(dim=16, heads=2, dim_head=8, depth=1, num_degrees=2, num_neighbors=5, valid_radius=10, causal=True,
               num_edge_tokens=4, edge_dim=3)
    model = _model(cfg, seed=3)
    g = torch.Generator().manual_seed(0)
    b, n = 2, 21
    feats = torch.randn(b, n, 16, generator=g).to(DEV)
    coors = torch.randn(b, n, 3, generator=g).to(DEV)
    edges = torch.randint(0, 4, (b, n, n), generator=g).to(DEV)
    nbr = (torch.rand(b, n, n, generator=g) > 0.3).to(DEV)
    full = model(feats, coors, edges=edges, neighbor_mask=nbr)
    res = _decode(model, feats, coors, [4, 1, 1, 6, 1, 8], b=b, pairs=dict(edges=edges, neighbor_mask=nbr))
    assert _errs(res, full) < 1e-5


@pytest.mark.parametrize('k', [3, 16])
def test_new_row_search_equals_whole_cloud_rows(k):
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator().manual_seed(1)
    b, n, ld = 3, 90, 128
    store = torch.zeros(b, ld, 3)
    store[:, :n] = torch.randn(b, n, 3, generator=g)
    store = store.to(DEV)
    nm = torch.ones(b, ld, dtype=torch.bool, device=DEV)
    nm[0, 5] = False
    nbr = torch.rand(b, n, n, generator=g).to(DEV) > 0.2
    whole = ops.knn(store[:, :n].contiguous(), k, 2.5, node_mask=nm[:, :n].contiguous(), neighbor_mask=nbr, causal=True)
    for n0, m in ((40, 1), (60, 7), (n - 3, 3)):
        rows = ops.knn_rows(store, n, n0, m, k, 2.5, node_mask=nm, neighbor_mask=nbr[:, n0:n0 + m].contiguous(), causal=True)
        valid = whole[1][:, n0:n0 + m]
        assert torch.equal(rows[1], valid)
        for a, w in zip(rows, whole):
            assert torch.equal(a[valid], w[:, n0:n0 + m][valid])
