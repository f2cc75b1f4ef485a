"""float64 torch restatements of the ops that model.conv_forward launches, for checking its host dispatch on CPU.

Every emulation computes what its kernel's contract says (include/se3b200.h) and appends one record to `trace`: the op name,
its integer / bool / string arguments, the shapes of its tensor arguments and, for plan images, which image was passed.  The
images made by the packers (pack_lowrank, pack_w3, zgemm_image) are the float64 weight matrices themselves, labelled by the
order they were packed in and their shape.  No CUDA is needed: tc_supported skips its device check, radial_trunk reads the
packed trunk parameters.
"""
import contextlib

import torch
import torch.nn.functional as F

from se3_transformer_pytorch_b200 import ops


def fingerprint(t):
    """[sum |t|, |t|_2, sum t w] with fixed pseudo-random weights w in [-1, 1): pins a tensor up to the last-bit differences
    that the float64 linear algebra of plan building (QR, SVD) may show between machines; compare with match()."""
    t = t.detach().double().reshape(-1)
    w = torch.rand(t.numel(), generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 2 - 1
    return [list(t.shape), float(f'{float(t.abs().sum()):.12g}'), float(f'{float(t.norm()):.12g}'), float(f'{float(t @ w):.12g}')]


def match(got, want, rtol=1e-6):
    """Fingerprints agree to rtol of the L1 norm (which bounds every entry of both)."""
    return got[0] == want[0] and all(abs(g - w) <= rtol * want[1] for g, w in zip(got[1:], want[1:]))


def trunk64(feat, params):
    """g [pairs, E, 128] of the radial trunk from the packed parameters (ConvSE3.packed()['trunk'], layout of trunk_params)."""
    M = ops.RADIAL_MID
    d = feat.shape[1]
    out = []
    for p in params.double():
        sizes = [d * M, M, M, M, M * M, M, M, M]
        W0, b0, w1, c1, W1, b1, w2, c2 = torch.split(p, sizes)
        h = F.gelu(F.layer_norm(feat.double() @ W0.view(d, M) + b0, (M,), w1, c1))
        out.append(F.gelu(F.layer_norm(h @ W1.view(M, M) + b1, (M,), w2, c2)))
    return torch.stack(out)


def tile_edges(E, tile_begin, tile_count):
    if tile_count is None:
        tile_count = (E + ops.TILE_E - 1) // ops.TILE_E - tile_begin
    return tile_begin * ops.TILE_E, min(E, (tile_begin + tile_count) * ops.TILE_E)


def gather_rows(x, idx, e0, e1):
    bb, nn, Ci, Q = x.shape
    return x.reshape(bb * nn, Ci, Q)[(idx + torch.arange(bb).view(-1, 1, 1) * nn).reshape(-1)][e0:e1].double()


class Emulation:
    def __init__(self):
        self.trace = []
        self.labels = {}            # id(image) -> label
        self.images = []            # the labelled images, kept alive so that their ids are not reused

    def _label(self, img, kind, desc):
        label = f'{kind}#{len(self.labels)}[{desc}]'
        self.labels[id(img)] = label
        self.images.append(img)
        return label

    def _arg(self, v):
        if id(v) in self.labels:
            return self.labels[id(v)]
        if torch.is_tensor(v):
            return list(v.shape)
        if isinstance(v, (list, tuple)):
            return [self._arg(u) for u in v]
        if v is None or isinstance(v, (bool, int, str)):
            return v
        if isinstance(v, float):
            return round(v, 9)
        return type(v).__name__

    def rec(self, name, **kw):
        self.trace.append([name, {k: self._arg(v) for k, v in kw.items()}])

    # ---- plan images ------------------------------------------------------------------------------------
    def pack_lowrank(self, Fp, Co, Ci, F_, Kp):
        assert Fp.shape == (Co * Ci * F_, Kp) and Fp.dtype == torch.float32 and Fp.is_contiguous()
        img = Fp.double().clone()
        self.rec('pack_lowrank', image=self._label(img, 'lowrank', f'Co{Co}Ci{Ci}F{F_}K{Kp}'))
        return img

    def pack_w3(self, W3, b3, Co, Ci, F_):
        img = torch.cat([W3.double(), b3.double().unsqueeze(1)], dim=1)          # [Co*Ci*F, 129]
        self.rec('pack_w3', image=self._label(img, 'w3', f'Co{Co}Ci{Ci}F{F_}'))
        return img

    def zgemm_image(self, parts, Co, mode):
        per_seg = (lambda Ci: 3 * (Ci // 4)) if mode == 3 else (lambda Ci: Ci * min(mode, 2) // 4)
        img = [(Fp.double(), Ci) for Fp, Ci in parts]
        S = sum((Fp.shape[1] // 16) * per_seg(Ci) for Fp, Ci in parts)
        self.rec('zgemm_image', image=self._label(img, 'zgemm', f'Co{Co}mode{mode}S{S}'))
        return img, S

    def tc_supported(self, device, Co, P):
        return Co % ops.TILE_O == 0 and P <= 7

    # ---- radial functions -------------------------------------------------------------------------------
    def radial_trunk(self, feat, params, num_pairs):
        self.rec('radial_trunk', feat=feat, params=params, num_pairs=num_pairs)
        return trunk64(feat, params).float()

    def radial_trunk_u(self, feat, params, V, gmean, ones_col, stats, want_g=False):
        self.rec('radial_trunk_u', feat=feat, params=params, V=V, ones_col=ones_col.tolist(), want_g=want_g)
        g = trunk64(feat, params)
        gc = g - gmean.double()[:, None, :]
        U = torch.bmm(gc, V.double())
        resid = (gc - torch.bmm(U, V.double().transpose(1, 2))).abs().amax(dim=(1, 2))
        stats[:, 0] = torch.maximum(stats[:, 0], resid.float())
        stats[:, 1] = torch.maximum(stats[:, 1], g.abs().amax(dim=(1, 2)).float())
        U[torch.arange(params.shape[0]), :, ones_col.long()] = 1.0
        return U.float(), (g.float() if want_g else None)

    def radial_table(self, dist, table, Dmax, ones_col, stats):
        """4-point Lagrange interpolation of the plan's U(d) table; distances outside [0, Dmax] raise every pair's flag."""
        self.rec('radial_table', dist=dist, table=table, Dmax=float(Dmax), ones_col=ones_col.tolist())
        d = dist.reshape(-1).double()
        if not bool((d <= Dmax).all()):
            stats[:] = 1.0
        Gn, KT = table.shape[1], table.shape[2]
        t = d * (Gn - 1) / Dmax
        i0 = t.floor().long().clamp(1, Gn - 3)
        f = (t - i0).unsqueeze(-1)
        w = (-f * (f - 1) * (f - 2) / 6, (f + 1) * (f - 1) * (f - 2) / 2, -(f + 1) * f * (f - 2) / 2, (f + 1) * f * (f - 1) / 6)
        U = torch.zeros(table.shape[0], d.numel(), 64, dtype=torch.float64)
        U[:, :, :KT] = sum(w[j] * table.double()[:, i0 - 1 + j] for j in range(4))
        U[torch.arange(table.shape[0]), :, ones_col.long()] = 1.0
        return U.float()

    # ---- T blocks and gathers (tile layout emulated as [edges, Ci, F, P]) --------------------------------
    def tbuild(self, x, idx, basis_pair, d_in, d_out, tile_begin=0, tile_count=None, out=None):
        self.rec('tbuild', x=x, d_in=d_in, d_out=d_out, tile_begin=tile_begin, tile_count=tile_count, reuse=out is not None)
        E = idx.numel()
        P, Q, F_ = 2 * d_out + 1, 2 * d_in + 1, 2 * min(d_in, d_out) + 1
        e0, e1 = tile_edges(E, tile_begin, tile_count)
        return torch.einsum('epqf,eiq->eifp', basis_pair.reshape(E, P, Q, F_)[e0:e1].double(), gather_rows(x, idx, e0, e1))

    def tbuild_blocks(self, x, idx, blocks, P, F_, tile_begin=0, tile_count=None, out=None):
        self.rec('tbuild_blocks', x=x, P=P, F=F_, tile_begin=tile_begin, tile_count=tile_count, reuse=out is not None)
        E = idx.numel()
        Q = x.shape[3]
        e0, e1 = tile_edges(E, tile_begin, tile_count)
        return torch.einsum('epqf,eiq->eifp', blocks.reshape(E, P, Q, F_)[e0:e1].double(), gather_rows(x, idx, e0, e1))

    def gather_tiles(self, x, idx, tile_begin=0, tile_count=None, out=None):
        self.rec('gather_tiles', x=x, tile_begin=tile_begin, tile_count=tile_count)
        e0, e1 = tile_edges(idx.numel(), tile_begin, tile_count)
        return gather_rows(x, idx, e0, e1).unsqueeze(2)                             # [e, i, f = 1, q]

    def rotgather(self, x, idx, D, tile_begin=0, tile_count=None, out=None):
        self.rec('rotgather', x=x, D=D, tile_begin=tile_begin, tile_count=tile_count)
        e0, e1 = tile_edges(idx.numel(), tile_begin, tile_count)
        xj = gather_rows(x, idx, e0, e1)
        return xj if D is None else torch.einsum('eqn,eiq->ein', D[e0:e1].double(), xj)      # x'[n] = sum_q D[q,n] x[q]

    def edge_scale(self, feats, idx, max_degree):
        self.rec('edge_scale', max_degree=max_degree)
        return torch.full((idx.numel(),), 4.0)

    # ---- radial weights x T -----------------------------------------------------------------------------
    @staticmethod
    def _store(out, res, accumulate):
        out.copy_((out.double() + res.reshape(out.shape) if accumulate else res.reshape(out.shape)).float())

    def pairwise_lr(self, U, img, T, E, Co, Ci, F_, P, Kp, out, accumulate, alg_P=None, alg_units=None):
        self.rec('pairwise_lr', U=U, image=img, T=T, E=E, Co=Co, Ci=Ci, F=F_, P=P, Kp=Kp, out=out, accumulate=accumulate,
                 alg_P=alg_P, alg_units=alg_units)
        assert T.shape == (E, Ci, F_, P) and out.shape[0] == E
        R = (U[:, :Kp].double() @ img.t()).reshape(E, Co, Ci, F_)                   # bias rides on the ones column of U
        self._store(out, torch.einsum('eoif,eifp->eop', R, T), accumulate)

    def pairwise_tc(self, g, img, T, E, Co, Ci, F_, P, out, accumulate):
        self.rec('pairwise_tc', g=g, image=img, T=T, E=E, Co=Co, Ci=Ci, F=F_, P=P, out=out, accumulate=accumulate)
        R = (g.double() @ img[:, :-1].t() + img[:, -1]).reshape(E, Co, Ci, F_)
        self._store(out, torch.einsum('eoif,eifp->eop', R, T), accumulate)

    def pairwise_simt(self, g, W3, b3, T, E, Co, Ci, F_, P, out, accumulate):
        self.rec('pairwise_simt', g=g, W3=W3, T=T, E=E, Co=Co, Ci=Ci, F=F_, P=P, out=out, accumulate=accumulate)
        R = (g.double() @ W3.double().t() + b3.double()).reshape(E, Co, Ci, F_)
        self._store(out, torch.einsum('eoif,eifp->eop', R, T), accumulate)

    def zgemm(self, segs, w_img, sx, E, Co, mode, out, out_edge_stride, comp_off, flush_stages=0, alg_flops=0, tag=''):
        self.rec('zgemm', segs=[[U, X, Ci, nc, cp, cm] for U, X, Ci, nc, cp, cm in segs], image=w_img, E=E, Co=Co, mode=mode,
                 out=out, out_edge_stride=out_edge_stride, comp_off=list(comp_off), alg_flops=alg_flops, tag=tag)
        mode = min(mode, 2)                                    # mode 3 = mode 2 evaluated with three products per complex one
        assert out_edge_stride == out.shape[1] * out.shape[2] and sx.shape == (E,)
        planes = out.view(E, -1, Co)                           # component-major rows: plane index = comp_off / Co
        res = [torch.zeros(E, Co, dtype=torch.float64) for _ in range(mode)]
        si = 0
        for Fp, Ci in w_img:
            Kp = Fp.shape[1]
            Fv = Fp.reshape(Co, Ci, mode, Kp)
            for kc in range(Kp // 16):
                U, X, Ci_s, ncomp, cplus, cminus = segs[si]
                si += 1
                assert Ci_s == Ci and X.shape == (E, Ci, ncomp) and U.shape[0] == E
                w = torch.einsum('ek,oifk->eoif', U[:, :16].double(), Fv[..., 16 * kc:16 * kc + 16])
                if mode == 1:
                    res[0] += torch.einsum('eoi,ei->eo', w[..., 0], X[:, :, cplus])
                else:
                    a, b = w[..., 0], w[..., 1]
                    res[0] += torch.einsum('eoi,ei->eo', a, X[:, :, cplus]) - torch.einsum('eoi,ei->eo', b, X[:, :, cminus])
                    res[1] += torch.einsum('eoi,ei->eo', b, X[:, :, cplus]) + torch.einsum('eoi,ei->eo', a, X[:, :, cminus])
        assert si == len(segs)
        for c in range(mode):
            planes[:, comp_off[c] // Co, :] = res[c].float()

    # ---- epilogues --------------------------------------------------------------------------------------
    def fold_basis(self, S, basis_pair, E, Co, P, Q, F_, out, accumulate, component_major=False, name='fold_basis'):
        self.rec(name, S=S, basis_pair=basis_pair, E=E, Co=Co, P=P, Q=Q, F=F_, out=out, accumulate=accumulate,
                 component_major=component_major)
        res = torch.einsum('epqf,feqo->eop' if component_major else 'epqf,feoq->eop', basis_pair.reshape(E, P, Q, F_).double(), S.double())
        self._store(out, res, accumulate)

    def rotate_back(self, parts, D, E, Co, lo, out):
        self.rec('rotate_back', parts=list(parts), D=D, E=E, Co=Co, lo=lo, out=out)
        P = 2 * lo + 1
        v = torch.zeros((E, Co, P), dtype=torch.float64)
        if parts[0] is not None:
            v[:, :, lo] = parts[0].reshape(E, Co).double()
        for m in range(1, lo + 1):
            if parts[m] is not None:
                v[:, :, lo + m], v[:, :, lo - m] = parts[m][:, :, 0].double(), parts[m][:, :, 1].double()
        out.copy_(torch.einsum('epn,eon->eop', D.reshape(E, P, P).double(), v).float())

    def rotate_pool(self, Op, D, mask, self_add, nodes, K, Co, lo, out):
        self.rec('rotate_pool', Op=Op, D=D, mask=mask, self_add=self_add, nodes=nodes, K=K, Co=Co, lo=lo, out=out)
        P = 2 * lo + 1
        v = Op.double().reshape(nodes * K, P, Co)
        if D is not None:
            v = torch.einsum('epn,eno->eop', D.reshape(-1, P, P).double(), v)
        else:
            v = v.transpose(1, 2)                                                   # [e, Co, P]
        self._store(out, self._masked_mean(v.reshape(nodes, K, Co, P), None if mask is None else mask.reshape(nodes, K))
                    + (0 if self_add is None else self_add.double()), False)

    @staticmethod
    def _masked_mean(v, mask):
        if mask is None:
            return v.mean(1)
        m = mask.double().view(*mask.shape, *([1] * (v.dim() - 2)))
        return (v * m).sum(1) / m.sum(1).clamp(min=1.0)

    def pool(self, x, mask):
        self.rec('pool', x=x, mask=mask)
        b, n, k = x.shape[:3]
        v = x.double().reshape(b * n, k, *x.shape[3:])
        return self._masked_mean(v, None if mask is None else mask.reshape(b * n, k)).reshape(b, n, *x.shape[3:]).float()

    NAMES = ('pack_lowrank', 'pack_w3', 'zgemm_image', 'tc_supported', 'radial_trunk', 'radial_trunk_u', 'radial_table', 'tbuild',
             'tbuild_blocks', 'gather_tiles', 'rotgather', 'edge_scale', 'pairwise_lr', 'pairwise_tc', 'pairwise_simt', 'zgemm',
             'fold_basis', 'rotate_back', 'rotate_pool', 'pool')

    def patches(self):
        """{ops attribute: emulation}; install with monkeypatch.setattr(ops, name, fn) or installed()."""
        return {name: getattr(self, name) for name in self.NAMES}


@contextlib.contextmanager
def installed(patches, target=ops):
    """Set target.<name> = fn for the duration of the block (for scripts that have no pytest monkeypatch)."""
    saved = {name: getattr(target, name) for name in patches}
    try:
        for name, fn in patches.items():
            setattr(target, name, fn)
        yield
    finally:
        for name, fn in saved.items():
            setattr(target, name, fn)
