"""ConvSE3.forward over node chunks on CPU: a pooled convolution with self-interaction, evaluated over whole batch rows under
the edge budget, must give outputs bit-identical to the whole graph on every route, with every op replaced by the float64
emulation of tests/dispatch_emulation.py.  Host logic only: tests/test_gpu_chunked.py runs the kernels."""
import numpy as np
import pytest
import torch

from dispatch_emulation import Emulation
from se3_transformer_pytorch_b200 import model as M, ops, switches

ROUTES = {
    'production': dict(C=128),
    'aligned': dict(C=32),
    'global': dict(C=32, no_aligned=True),
    'no_lowrank': dict(C=32, no_lowrank=True),
    'force_simt': dict(C=32, force_simt=True),
}


def _graph(b, n, k, L, C):
    coors = torch.randn(b, n, 3)
    idx = torch.stack([torch.randperm(n - 1)[:k] for _ in range(b * n)]).reshape(b, n, k)
    idx = idx + (idx >= torch.arange(n).view(1, n, 1)).long()                        # neighbours != self
    rel_pos = torch.stack([coors[r][:, None, :] - coors[r][idx[r]] for r in range(b)])   # x_i - x_j
    nmask = torch.rand(b, n, k) < 0.9
    inp = {str(d): torch.randn(b, n, C, 2 * d + 1) for d in range(L + 1)}
    return idx, nmask, rel_pos, inp


@pytest.mark.parametrize('route', sorted(ROUTES))
def test_row_chunks_are_bit_identical_on_cpu_emulation(monkeypatch, route):
    from oracle import se3_oracle as O
    spec = dict(ROUTES[route])
    C = spec.pop('C')
    b, n, k, L = 2, 24, 6, 2
    torch.manual_seed(0)
    fiber = M.Fiber([(d, C) for d in range(L + 1)])
    conv = M.ConvSE3(fiber, fiber, edge_dim=0, pool=True, self_interaction=True)
    idx, nmask, rel_pos, inp = _graph(b, n, k, L, C)
    rel_dist = rel_pos.norm(dim=-1)

    emu = Emulation()
    for name, fn in emu.patches().items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(torch.cuda, 'is_current_stream_capturing', lambda: False)
    # the flat basis of a chunk is its rel_pos; the R-first kernels read the oracle basis of those edges
    monkeypatch.setattr(ops, 'basis_flat', lambda rp, max_degree: (rp, None))

    def basis_pairs(flat, plan, E):
        Bo = O.get_basis(flat.reshape(E, 3).double().numpy(), L)
        return {(di, do): torch.from_numpy(np.asarray(Bo[f'{di},{do}'])).float().reshape(-1)
                for di in range(L + 1) for do in range(L + 1)}
    monkeypatch.setattr(ops, 'basis_pairs', basis_pairs)

    rows = []
    orig = M.plan_node_chunks

    def one_row(b_, n_, k_, edge_bytes, budget):
        chunks = orig(b_, n_, k_, edge_bytes, n_ * k_ * edge_bytes)
        rows.append(chunks)
        return chunks

    def forward(budget):
        geom = M.Geometry(rel_pos, L, deferred=[], edge_budget=budget)
        n0 = len(emu.trace)
        out = conv(inp, (idx, nmask, None), rel_dist=rel_dist, basis=(None, None, geom))
        assert not M.check_lowrank_stats(geom.deferred)
        return out, len(emu.trace) - n0

    sw = dict(dict.fromkeys(switches.FIELDS), host_frames=True, lowrank_min_edges=1, **spec)
    with switches.override(**sw), torch.no_grad():
        forward(None)                                   # builds the low-rank plan and the weight images
        whole, whole_launches = forward(None)
        monkeypatch.setattr(M, 'plan_node_chunks', one_row)
        chunked, chunked_launches = forward(0)
    assert [len(p) for p in rows] == [b]
    assert chunked_launches > whole_launches, (whole_launches, chunked_launches)
    assert whole.keys() == chunked.keys() == {str(d) for d in range(L + 1)}
    for d in whole:
        assert whole[d].shape == (b, n, C, 2 * int(d) + 1)
        assert torch.equal(whole[d], chunked[d]), f'degree {d}: max abs diff {(whole[d] - chunked[d]).abs().max().item():.3e}'
