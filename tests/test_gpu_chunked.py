"""The edge budget on the GPU (SE3B200_EDGE_BUDGET_MB, model.plan_node_chunks): a forward whose blocks run their edge work over
node chunks gives outputs bit-identical to the forward that runs each block as one chunk, on every fixture, route and entry
point; and forwards whose whole-graph edge tensors would not fit the card run under a bounded peak."""
import numpy as np
import pytest
import torch

from helpers import MODEL_CASES, Z_CASES, DEG_CASES, GOLDEN, load_case, case_inputs, rel_err
from detfill import fill_state_dict
from test_gpu_model import build_model, run_model, check_outputs
from varlen_helpers import VARLEN_CASES, load_varlen, varlen_outputs, per_cloud_errors

pytestmark = pytest.mark.gpu
DEV = 'cuda'
UNLIMITED = 2 ** 40                 # MiB: every block is one chunk


def _as_dict(o):
    return o if isinstance(o, dict) else {'': o}


def _equal(a, b):
    a, b = _as_dict(a), _as_dict(b)
    assert a.keys() == b.keys()
    for d in a:
        assert torch.equal(a[d], b[d]), f'degree {d}: max abs diff {(a[d] - b[d]).abs().max().item():.3e}'


class _Plans:
    """Records the node chunks of every block (model.plan_node_chunks).  Mode 'rows' sets the budget to one batch row, 'thirds'
    to a third of a row (chunks inside rows); otherwise the budget stands."""

    def __init__(self, monkeypatch, mode=None):
        from se3_transformer_pytorch_b200 import model as M
        self.plans, orig = [], M.plan_node_chunks

        def plan(b, n, k, edge_bytes, budget):
            if mode == 'rows':
                budget = n * k * edge_bytes
            elif mode == 'thirds':
                budget = -(-n // 3) * k * edge_bytes
            chunks = orig(b, n, k, edge_bytes, budget)
            self.plans.append(chunks)
            return chunks
        monkeypatch.setattr(M, 'plan_node_chunks', plan)

    def chunks(self):
        return sum(len(p) for p in self.plans)


def _chunked(monkeypatch, fn, mode='nodes', **switches_):
    """fn() under the default budget, then under a budget that forces chunks (one node each, a third of a row, or whole batch
    rows) -> (default result, chunked result, chunks run, blocks run), both under the switches given."""
    from se3_transformer_pytorch_b200 import switches
    with torch.no_grad(), switches.override(**switches_):
        ref = fn()
        rec = _Plans(monkeypatch, mode)
        with switches.override(edge_budget_mb=0):
            got = fn()
    return ref, got, rec.chunks(), len(rec.plans)


@pytest.mark.parametrize('mode', ['thirds', 'rows'])
@pytest.mark.parametrize('name', MODEL_CASES + Z_CASES + DEG_CASES)
def test_fixture_is_bit_identical_in_node_chunks(name, mode, monkeypatch):
    z, cfg = load_case(name)
    b = case_inputs(z)[1].shape[0]
    if mode == 'rows' and b == 1:
        pytest.skip('one batch row: row chunks are the whole graph')
    model = build_model(cfg)
    ref, got, chunks, blocks = _chunked(monkeypatch, lambda: run_model(model, z, cfg), mode)
    assert chunks > blocks, (chunks, blocks)
    _equal(got, ref)
    check_outputs(got, z)
    check_outputs(ref, z)


@pytest.mark.parametrize('name', ['cfg1', 'ragged', 'z128', 'rotary_both'])
def test_one_node_chunks_are_bit_identical(name, monkeypatch):
    z, cfg = load_case(name)
    model = build_model(cfg)
    ref, got, chunks, blocks = _chunked(monkeypatch, lambda: run_model(model, z, cfg), 'nodes')
    n = int(np.prod(case_inputs(z)[1].shape[:2]))
    assert chunks == blocks * n, (chunks, blocks, n)
    _equal(got, ref)


ROUTES = [dict(lowrank_min_edges=0), dict(lowrank_min_edges=0, no_zgemm=True), dict(lowrank_min_edges=0, no_aligned=True),
          dict(lowrank_min_edges=0, no_aligned=True, no_input_side=True), dict(force_simt=True), dict(no_attn_rotate=True),
          dict(lowrank_min_edges=0, no_attn_rotate=True)]


@pytest.mark.parametrize('sw', ROUTES, ids=lambda s: ','.join(s))
@pytest.mark.parametrize('name', ['z128', 'tc_deg2', 'rotary_dist_linkeys'])
def test_every_route_is_bit_identical_in_node_chunks(name, sw, monkeypatch):
    from se3_transformer_pytorch_b200 import ops
    z, cfg = load_case(name)
    model = build_model(cfg)
    ops.PROFILE = []
    try:
        ref, got, chunks, blocks = _chunked(monkeypatch, lambda: run_model(model, z, cfg), 'thirds', **sw)
    finally:
        kinds, ops.PROFILE = {p[0] for p in ops.PROFILE}, None
    assert chunks > blocks
    _equal(got, ref)
    check_outputs(got, z)
    if sw.get('lowrank_min_edges') == 0 and name == 'z128' and len(sw) == 1:
        assert 'zgemm' in kinds, kinds


@pytest.mark.parametrize('name', VARLEN_CASES)
def test_forward_packed_is_bit_identical_in_node_chunks(name, monkeypatch):
    z, cfg, feats, coors, seqlens, pairs = load_varlen(name)
    from se3_transformer_pytorch_b200 import SE3Transformer
    model = SE3Transformer(**cfg['ctor'])
    fill_state_dict(model, seed=11)
    model = model.to(DEV).eval()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    f = {k: t(v) for k, v in feats.items()} if isinstance(feats, dict) else t(feats)
    run = lambda: model.forward_packed(f, t(coors), seqlens, **{k: [t(x) for x in v] for k, v in pairs.items()}, **cfg['fwd'])
    ref, got, chunks, blocks = _chunked(monkeypatch, run, 'thirds')
    assert chunks > blocks
    _equal(got, ref)
    pooled = bool(cfg['fwd'].get('return_pooled'))
    got_np = {k: v.cpu().numpy() for k, v in got.items()} if isinstance(got, dict) else got.cpu().numpy()
    assert max(per_cloud_errors(got_np, varlen_outputs(z), seqlens, pooled)) < 1e-4


@pytest.mark.parametrize('name', ['edges_sparse', 'adjdeg', 'nbrmask', 'contedges'])
def test_sparse_pair_inputs_are_bit_identical_in_node_chunks(name, monkeypatch):
    z, cfg = load_case(name)
    model = build_model(cfg)
    feats, coors, mask, extra = case_inputs(z)
    cu = lambda a: torch.from_numpy(a).to(DEV)
    feats = {k: cu(v) for k, v in feats.items()} if isinstance(feats, dict) else cu(feats)
    dense = {k: torch.from_numpy(v) for k, v in extra.items()}
    sparse = {k: v.to_sparse(v.dim() - (k == 'edges' and v.dim() == 4)).to(DEV) for k, v in dense.items()}
    ref, got, chunks, blocks = _chunked(monkeypatch, lambda: model(feats, cu(coors), cu(mask), **sparse, **cfg['fwd']), 'thirds')
    assert chunks > blocks
    _equal(got, ref)
    check_outputs(got, z)


def test_graphed_replay_is_bit_identical_in_node_chunks(monkeypatch):
    from se3_transformer_pytorch_b200 import switches
    z, cfg = load_case('z128')
    model = build_model(cfg)
    feats, coors, mask, _ = case_inputs(z)
    t = lambda a: torch.from_numpy(a).to(DEV)
    with torch.no_grad(), switches.override(lowrank_min_edges=0):
        ref = run_model(model, z, cfg)
        rec = _Plans(monkeypatch)
        with switches.override(edge_budget_mb=0):
            g = model.graphed(t(feats), t(coors), t(mask), **cfg['fwd'])
        assert rec.chunks() > len(rec.plans)
        got = g(t(feats), t(coors), t(mask))                 # the chunk loop was captured: the budget is no longer read
    _equal(got, ref)


def test_plan_miss_behaves_as_unchunked(monkeypatch):
    """A forward that leaves its low-rank plans warns and runs again on the direct kernels, chunked or not, with the same result;
    with released masters it raises LowRankPlanMiss, chunked or not."""
    from se3_transformer_pytorch_b200 import model as M, switches
    z, cfg = load_case('z128')
    monkeypatch.setattr(M.ConvSE3, 'LR_RUNTIME_TOL', -1.0)          # every plan check fails
    outs = []
    for budget in (None, 0):
        model = build_model(cfg)
        with torch.no_grad(), switches.override(lowrank_min_edges=0, edge_budget_mb=budget):
            with pytest.warns(UserWarning, match='left their low-rank radial plan'):
                outs.append(run_model(model, z, cfg))
        assert all(conv._lr_blocked for conv in model.conv_modules())
    _equal(outs[1], outs[0])
    for budget in (None, 0):
        model = build_model(cfg)
        model.pack_weights(free_master=True, max_distance=12.0)
        with torch.no_grad(), switches.override(lowrank_min_edges=0, edge_budget_mb=budget), pytest.raises(M.LowRankPlanMiss):
            run_model(model, z, cfg)


# ------------------------------------------------------------------ forwards whose edge tensors exceed the card
def _rot():
    return torch.from_numpy(np.load(f'{GOLDEN}/rot_15_0_45.npz')['R']).float().to(DEV)


def _all_neighbour_model(n, seed=0):
    from se3_transformer_pytorch_b200 import SE3Transformer
    torch.manual_seed(seed)
    with torch.device(DEV):
        model = SE3Transformer(dim=128, heads=2, dim_head=64, depth=1, num_degrees=4, output_degrees=2,
                               num_neighbors=float('inf')).eval()
    feats = torch.randn(1, n, 128, device=DEV)
    coors = torch.randn(1, n, 3, device=DEV) * 3
    return model, feats, coors, torch.ones(1, n, dtype=torch.bool, device=DEV)


def _peak_run(model, *args, **sw):
    from se3_transformer_pytorch_b200 import switches
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad(), switches.override(**sw):
        out = model(*args)
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated()


def test_all_neighbours_on_2049_points_under_8_gb(monkeypatch):
    """num_neighbors = inf on 2049 points: k = 2048, 4.2 M edges, about 230 GB of whole-graph edge tensors.  Under an 8 GB budget
    the peak stays under 24 GB, 8 GB and 4 GB budgets agree bit for bit, the output is rotation-equivariant and the fused
    rotate-back matches the separate one."""
    model, feats, coors, mask = _all_neighbour_model(2049)
    rec = _Plans(monkeypatch)
    out, peak = _peak_run(model, feats, coors, mask, edge_budget_mb=8192)
    print(f'2049 points, 2048 neighbours, dim 128, 4 degrees, 8 GB budget: peak {peak / 1e9:.2f} GB, '
          f'{rec.chunks()} chunks over {len(rec.plans)} blocks')
    assert rec.chunks() > len(rec.plans)
    assert peak < 24e9
    small, _ = _peak_run(model, feats, coors, mask, edge_budget_mb=4096)
    _equal(small, out)
    sep, _ = _peak_run(model, feats, coors, mask, edge_budget_mb=8192, no_attn_rotate=True)
    for d in ('0', '1'):
        assert rel_err(out[d].cpu().numpy(), sep[d].cpu().numpy()) < 1e-5, d
    R = _rot()
    out_rot, _ = _peak_run(model, feats, coors @ R, mask, edge_budget_mb=8192)
    assert (out_rot['1'] - out['1'] @ R).abs().max().item() / out['1'].abs().max().item() < 2e-5
    assert (out_rot['0'] - out['0']).abs().max().item() / out['0'].abs().max().item() < 2e-5


def test_thousand_neighbours_under_8_gb(monkeypatch):
    """The 999-neighbour model of test_gpu_envelope under an 8 GB budget: bit-identical to one chunk per block, at a fraction of
    its peak (54-59 GB measured as one chunk)."""
    model, feats, coors, mask = _all_neighbour_model(1000)
    rec = _Plans(monkeypatch)
    out, peak = _peak_run(model, feats, coors, mask, edge_budget_mb=8192)
    print(f'1000 points, 999 neighbours, dim 128, 4 degrees, 8 GB budget: peak {peak / 1e9:.2f} GB, '
          f'{rec.chunks()} chunks over {len(rec.plans)} blocks')
    assert rec.chunks() > len(rec.plans)
    assert peak < 20e9
    whole, whole_peak = _peak_run(model, feats, coors, mask, edge_budget_mb=UNLIMITED)
    print(f'  one chunk per block: peak {whole_peak / 1e9:.2f} GB')
    _equal(out, whole)
