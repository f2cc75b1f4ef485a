"""Host-side mirror of the reference's module tree for the SE(3) attention hot path.

Same constructor, forward signature, assertions and state_dict key/shape layout as
lucidrains/se3-transformer-pytorch v0.9.0 (se3_transformer_pytorch.py:936-1375; SURVEY.md Appendix A.6), so
`ours.load_state_dict(reference.state_dict())` works.  The hot path -- neighbour graph, spherical-harmonic / CG basis,
radial trunk, pairwise tensor product (wgmma), pooling, attention -- runs in the hand-written sm_90a kernels of
libse3b200.so through `ops`; the cheap glue around it (embeddings, LinearSE3 GEMMs, NormSE3, residuals) stays torch.

Forward only: everything runs under torch.no_grad().  CUDA only: there is no CPU fallback.
"""
import numbers
import collections
import operator
from math import sqrt
from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import ops, switches
from . import aligned as _aligned


def exists(v):
    return v is not None


def default(v, d):
    return v if exists(v) else d


def _is_sparse(t):
    return torch.is_tensor(t) and t.layout != torch.strided


def to_order(degree):
    return 2 * degree + 1


class Fiber:
    """Ordered list of (degree, channels) (reference S:20-59)."""

    def __init__(self, structure):
        if isinstance(structure, dict):
            structure = list(structure.items())
        self.structure = [(int(d), int(c)) for d, c in structure]

    @staticmethod
    def create(num_degrees, dim):
        dims = dim if isinstance(dim, tuple) else (dim,) * num_degrees
        return Fiber([(d, c) for d, c in zip(range(num_degrees), dims)])

    @property
    def degrees(self):
        return [d for d, _ in self.structure]

    @property
    def dims(self):
        return list(dict.fromkeys(c for _, c in self.structure))

    def __getitem__(self, degree):
        return dict(self.structure)[degree]

    def __iter__(self):
        return iter(self.structure)

    def shared(self, other):
        """(degree, dim_self, dim_other) for degrees present in both (reference S:52-59)."""
        od = dict(other.structure)
        return [(d, c, od[d]) for d, c in self.structure if d in od]


def forward_only_guard(what, modules, tensors=()):
    """The kernels have no backward (SURVEY.md 8f row 4).  Called with autograd recording and anything that wants a gradient,
    they would silently return tensors cut off from the graph (radial weights and inputs without gradients, the torch glue
    with): fail loudly instead.  SE3Transformer.forward itself runs under torch.no_grad()."""
    if not torch.is_grad_enabled():
        return
    wants = any(t is not None and torch.is_tensor(t) and t.requires_grad for t in tensors) or \
        any(p.requires_grad for m in modules for p in m.parameters())
    if wants:
        raise RuntimeError(f'{what} is forward only (no backward kernels): call it under torch.no_grad() / torch.inference_mode(), '
                           'or use the reference implementation for training')


def residual_add(x, res):
    return {d: (t + res[d] if d in res else t) for d, t in x.items()}


class LinearSE3(nn.Module):
    """Per-degree channel mix (reference S:78-95).  Widths the tensor-core kernel takes (C_in % 64 == 0, C_out % 128 == 0) run
    on se3_linear_tc_fwd: the A operand is read in place from the reference layout, split to fp16 hi / lo on the fly (fp32
    parity), an optional residual is added in the epilogue; other widths are a plain cuBLAS GEMM."""

    def __init__(self, fiber_in, fiber_out):
        super().__init__()
        self.weights = nn.ParameterDict()
        for degree, dim_in, dim_out in fiber_in.shared(fiber_out):
            self.weights[str(degree)] = nn.Parameter(torch.randn(dim_in, dim_out) / sqrt(dim_in))
        self._images = {}

    def image(self, degree):
        w = self.weights[degree]
        ver = (w._version, w.data_ptr())
        hit = self._images.get(degree)
        if hit is None or hit[0] != ver:
            ok = float(w.detach().abs().max()) < 6.0e4              # fp16 range of the hi / lo split
            hit = (ver, ops.linear_image(w) if ok else None)
            self._images[degree] = hit
        return hit[1]

    def forward(self, x, residual=None):
        sw = switches.current()
        tc = not (sw.force_simt or sw.no_linear_tc)
        out = {}
        for degree, w in self.weights.items():
            t = x[degree]                                            # [b, n, d, m]
            res = residual.get(degree) if residual is not None else None
            if tc and t.is_cuda and t.dtype == torch.float32 and not torch.is_grad_enabled() and ops.linear_supported(w.shape[0], w.shape[1], t.device):
                img = self.image(degree)
                if img is not None:
                    out[degree] = ops.linear_tc(t, img, w.shape[1], res=res, flush_stages=sw.linear_flush())
                    continue
            y = torch.matmul(t.transpose(-1, -2), w).transpose(-1, -2).contiguous()
            out[degree] = y if res is None else y + res
        return out                                                   # (degrees only in `residual` are dropped, as ResidualSE3 S:67-76)


class NormSE3(nn.Module):
    """Norm nonlinearity (reference S:97-152)."""

    def __init__(self, fiber, nonlin=None, gated_scale=False, eps=1e-12):
        super().__init__()
        self.fiber = fiber
        self.nonlin = nonlin if nonlin is not None else nn.GELU()
        self.eps = eps
        self.transform = nn.ModuleDict()
        for degree, chan in fiber:
            pd = nn.ParameterDict()
            if gated_scale:
                pd['w_gate'] = nn.Parameter(torch.empty(chan, chan).uniform_(-1e-3, 1e-3))
            else:
                pd['scale'] = nn.Parameter(torch.ones(1, 1, chan))
            self.transform[str(degree)] = pd

    def forward(self, features):
        out = {}
        for degree, t in features.items():
            pd = self.transform[degree]
            fused = 'scale' in pd and t.is_cuda and t.dtype == torch.float32 and isinstance(self.nonlin, (nn.GELU, nn.Identity)) \
                and not (isinstance(self.nonlin, nn.GELU) and self.nonlin.approximate != 'none')
            if fused:                                    # one fused kernel (libse3b200: se3_norm_fwd)
                out[degree] = ops.norm_se3(t, pd['scale'], self.eps, isinstance(self.nonlin, nn.GELU))
                continue
            norm = t.norm(dim=-1, keepdim=True).clamp(min=self.eps)
            phase = t / norm
            pd = self.transform[degree]
            tr = norm.squeeze(-1)
            scale = pd['scale'] if 'scale' in pd else torch.matmul(tr, pd['w_gate'])
            tr = self.nonlin(tr * scale)
            out[degree] = (tr.unsqueeze(-1) * phase).view(*t.shape)
        return out


class RadialFunc(nn.Module):
    """Parameter holder for the radial MLP (reference S:270-299).  `net` keeps the reference's Sequential indices
    (0 Linear, 1 LayerNorm, 3 Linear, 4 LayerNorm, 6 Linear) so state_dict keys match; evaluation happens in the
    fused kernels, never here."""

    def __init__(self, num_freq, in_dim, out_dim, edge_dim=0, mid_dim=ops.RADIAL_MID):
        super().__init__()
        assert mid_dim == ops.RADIAL_MID
        self.num_freq, self.in_dim, self.out_dim, self.edge_dim = num_freq, in_dim, out_dim, edge_dim
        self.net = nn.ModuleDict({
            '0': nn.Linear(edge_dim + 1, mid_dim),
            '1': nn.LayerNorm(mid_dim),
            '3': nn.Linear(mid_dim, mid_dim),
            '4': nn.LayerNorm(mid_dim),
            '6': nn.Linear(mid_dim, num_freq * in_dim * out_dim),
        })

    def trunk64(self, feat):
        """The trunk (net.0 .. net.5) in float64 with torch ops: used off the hot path, to sample the curve g(d) when the
        low-rank plan of a pair is built."""
        n = self.net
        h = F.linear(feat.double(), n['0'].weight.double(), n['0'].bias.double())
        h = F.gelu(F.layer_norm(h, (h.shape[-1],), n['1'].weight.double(), n['1'].bias.double()))
        h = F.linear(h, n['3'].weight.double(), n['3'].bias.double())
        return F.gelu(F.layer_norm(h, (h.shape[-1],), n['4'].weight.double(), n['4'].bias.double()))

    def trunk_params(self):
        n = self.net
        return torch.cat([n['0'].weight.t().reshape(-1), n['0'].bias, n['1'].weight, n['1'].bias,
                          n['3'].weight.t().reshape(-1), n['3'].bias, n['4'].weight, n['4'].bias])


class PairwiseConv(nn.Module):
    """Holder for one (degree_in, degree_out) radial profile (reference S:301-343)."""

    def __init__(self, degree_in, nc_in, degree_out, nc_out, edge_dim=0):
        super().__init__()
        self.degree_in, self.degree_out, self.nc_in, self.nc_out = degree_in, degree_out, nc_in, nc_out
        self.num_freq = to_order(min(degree_in, degree_out))
        self.d_out = to_order(degree_out)
        self.rp = RadialFunc(self.num_freq, nc_in, nc_out, edge_dim)


# upper bound on the T workspace (bytes); larger convolutions are evaluated in edge chunks
T_WORKSPACE_BYTES = int(8 * 2 ** 30)


class ConvSE3(nn.Module):
    """Tensor-field-network layer (reference S:154-268) on the fused kernels."""

    def __init__(self, fiber_in, fiber_out, self_interaction=True, pool=True, edge_dim=0, fourier_encode_dist=False,
                 num_fourier_features=4, splits=4):
        super().__init__()
        self.fiber_in, self.fiber_out = fiber_in, fiber_out
        self.edge_dim = edge_dim
        self.self_interaction = self_interaction
        self.num_fourier_features = num_fourier_features
        self.fourier_encode_dist = fourier_encode_dist
        # accepted for API parity and ignored: SE3Transformer evaluates the edge work of every block over node chunks sized by
        # the edge_budget_mb switch (SE3B200_EDGE_BUDGET_MB, plan_node_chunks) instead of a fixed number of splits
        self.splits = splits
        edge_dim += 0 if not fourier_encode_dist else num_fourier_features * 2
        self.in_dim = edge_dim + 1
        self.kernel_unary = nn.ModuleDict()
        self.pairs = []
        for di, mi in fiber_in:
            for do, mo in fiber_out:
                self.kernel_unary[f'({di},{do})'] = PairwiseConv(di, mi, do, mo, edge_dim=edge_dim)
                self.pairs.append((di, do))
        self.pool = pool
        if self_interaction:
            assert self.pool, 'must pool edges if followed with self interaction'
            self.self_interact = LinearSE3(fiber_in, fiber_out)
        self._packed = None
        self.free_master = False
        self._lr_blocked = False      # set when a forward left the low-rank plan: the direct kernels from then on
        self.utable_error = None      # interpolation error of the last radial table built (radial_table)

    # ---- packed weights ---------------------------------------------------------------------------------
    def _param_version(self):
        return tuple((p._version, p.data_ptr()) for p in self.kernel_unary.parameters())

    # the switches the low-rank plan reads (it is built from tc_eligible, which reads force_simt)
    PLAN_SWITCHES = ('force_simt', 'no_aligned', 'no_zgemm', 'z_mode2', 'no_input_side', 'no_utable', 'lowrank_tol')

    def _weights(self):
        """What depends on the weights alone, built lazily and rebuilt when they change: the trunk parameter pack [pairs, stride]
        and the tensor-core images of net.6 for the direct (K = 128) kernel, filled on demand by w3_image()."""
        ver = None if self.free_master else self._param_version()
        if self._packed is None or not (self.free_master or self._packed['version'] == ver):
            with torch.no_grad():
                trunk = torch.stack([self.kernel_unary[f'({di},{do})'].rp.trunk_params() for di, do in self.pairs]).contiguous()
            self._packed = dict(version=ver, trunk=trunk, images={}, tc_ok={}, tc_key=None, lr=None, lr_key=None)
        return self._packed

    def packed(self, sw=None):
        """_weights() with the decisions tc_ok {pair: tc_eligible} and lr (lowrank_plan), each dropped when a switch it reads has
        changed in sw (default: switches.current()).  With released masters those of pack_weights stay, whatever the switches."""
        pk = self._weights()
        if not self.free_master:
            sw = switches.current() if sw is None else sw
            if pk['tc_key'] != sw.force_simt:
                pk.update(tc_key=sw.force_simt, tc_ok={})
            plan_key = tuple(getattr(sw, f) for f in self.PLAN_SWITCHES)
            if pk['lr_key'] != plan_key:
                pk.update(lr_key=plan_key, lr=None)
        return pk

    def tc_eligible(self, di, do):
        """The tensor-core kernels take this pair: not force_simt, sm_90, C_out % 32 == 0, degree_out <= 3 and operands inside
        the fp16 range of the hi/lo split (|g| <= sqrt(127) max|ln.w| + max|ln.b| after LayerNorm + GELU)."""
        sw = switches.current()
        pk = self.packed(sw)
        if (di, do) not in pk['tc_ok']:
            pc = self.kernel_unary[f'({di},{do})']
            ok = not sw.force_simt and ops.tc_supported(pk['trunk'].device, pc.nc_out, pc.d_out)
            if ok and (di, do) not in pk['images']:
                lin, ln = pc.rp.net['6'], pc.rp.net['4']
                g_bound = 11.3 * float(ln.weight.abs().max()) + float(ln.bias.abs().max())
                ok = g_bound < 6.0e4 and (lin.weight.numel() == 0 or float(lin.weight.abs().max()) < 6.0e4)
            pk['tc_ok'][(di, do)] = ok
        return pk['tc_ok'][(di, do)]

    def w3_image(self, di, do):
        pk = self._weights()
        if (di, do) not in pk['images']:
            pc = self.kernel_unary[f'({di},{do})']
            lin = pc.rp.net['6']
            if lin.weight.numel() == 0:
                raise RuntimeError(f'ConvSE3 pair ({di},{do}): the fp32 net.6 weights were released by pack_weights(free_master=True) and '
                                   'only the low-rank image was kept, but this forward needs the direct (K = 128) image (low-rank path '
                                   'switched off or not applicable); rebuild the model or pack with free_master=False')
            with torch.no_grad():
                pk['images'][(di, do)] = ops.pack_w3(lin.weight, lin.bias, pc.nc_out, pc.nc_in, pc.num_freq)
        return pk['images'][(di, do)]

    # ---- low-rank radial path ----------------------------------------------------------------------------
    LR_GRID = 16384          # float64 samples of g(d) per pair when a plan is built
    LR_RUNTIME_TOL = 1e-5    # sanity bound on max|G - (G V) V^T| / max|G| of the fp32 trunk outputs of a forward

    def encode_dist(self, rd):
        """[..., 1] distances -> radial-MLP input (reference utils.py:96-104 when fourier_encode_dist)."""
        if not self.fourier_encode_dist:
            return rd
        scales = 2 ** torch.arange(self.num_fourier_features, device=rd.device, dtype=rd.dtype)
        xs = rd / scales
        return torch.cat([xs.sin(), xs.cos(), rd], dim=-1)

    def lowrank_plan(self, d_max, sw=None):
        """Per pair: orthonormal V [128, r] spanning the curve g(d), d in [0, D], and the tensor-core images of F'' = [W3 V | b3 | 0]
        in the pair's formulation `kind`: if every pair has a plan, 'z' (in the per-(degree_out, |m|) GEMM images plan['z'],
        DESIGN.md 4.5) or 'aligned' (one image per |m|, 4.4); otherwise 'input_side' (one image per frequency, 4.3) or 'combined'
        (4.2).  Depends on the weights, D and the PLAN_SWITCHES of sw (default: switches.current()): built once, and again if one
        of them changes or a forward brings a larger distance.  Only for distance-only radial functions (no extra edge features)."""
        sw = switches.current() if sw is None else sw
        pk = self.packed(sw)
        plan = pk['lr']
        if plan is not None and plan['D'] >= d_max:
            return plan
        dev = pk['trunk'].device
        D = 1.25 * d_max
        with torch.no_grad():
            grid = torch.linspace(0.0, D, self.LR_GRID, device=dev, dtype=torch.float64).unsqueeze(-1)
            bases, ugrid = self._factor_curves(self.encode_dist(grid), sw.lowrank_tol)
            complete = len(bases) == len(self.pairs)
            aligned = not sw.no_aligned and complete
            z = aligned and not sw.no_zgemm and self.zgemm_eligible({pair: lowrank_k(rv[0]) for pair, rv in bases.items()})
            pairs, zweights = {}, {}
            for pair, (r, V, gmean) in bases.items():
                kind = 'z' if z else 'aligned' if aligned else 'input_side' if not sw.no_input_side and input_side(*pair) else 'combined'
                lin = self.kernel_unary[f'({pair[0]},{pair[1]})'].rp.net['6']
                Fp = torch.zeros((lin.weight.shape[0], lowrank_k(r)), dtype=torch.float32, device=dev)
                Fp[:, :r] = (lin.weight.double() @ V).float()
                Fp[:, r] = (lin.bias.double() + lin.weight.double() @ gmean).float()      # affine model: W3 gmean joins the bias
                if kind == 'z':
                    zweights[pair] = self.aligned_weights(pair, Fp)
                Vp = torch.zeros((ops.RADIAL_MID, 64), dtype=torch.float32, device=dev)
                Vp[:, :r] = V.float()
                pairs[pair] = dict(kind=kind, r=r, Kp=Fp.shape[1], V=Vp, gmean=gmean.float(),
                                   images=[] if kind == 'z' else self._pack_images(pair, kind, Fp))
            zplan = self._zgemm_images(zweights, 2 if sw.z_mode2 else 3) if z else None
            utab = self.radial_table(ugrid, bases, grid, dev) if complete and not sw.no_utable else None
            plan = dict(D=D, pairs=pairs, z=zplan, utab=utab, **self._plan_stacks(pairs, dev))
        pk['lr'] = plan
        return plan

    def _factor_curves(self, feat, tol):
        """Every tc-eligible pair that still has its net.6 weights and whose curve g(d) (float64 trunk on the distance grid
        `feat`) has a low-rank model within tol: {pair: (r, V, gmean)} and {pair: (U(d) = (g - gmean) V on the grid, max|g|)}."""
        bases, ugrid = {}, {}
        for di, do in self.pairs:
            pc = self.kernel_unary[f'({di},{do})']
            if self.tc_eligible(di, do) and pc.rp.net['6'].weight.numel() > 0:
                G64 = pc.rp.trunk64(feat)
                basis = ops.lowrank_basis(G64, tol)
                if basis is not None:
                    bases[(di, do)] = basis
                    ugrid[(di, do)] = ((G64 - basis[2]) @ basis[1], float(G64.abs().max()))
        return bases, ugrid

    def aligned_weights(self, pair, Fp):
        """The edge-aligned weights [w0, (a_m, b_m) for m = 1..min(di, do)] (DESIGN.md 4.4): constant combinations of the F
        frequencies (rows (o,i,f) of F'), as [Co*Ci, Kp] (m = 0) and [Co*Ci*2, Kp] (rows (o,i,(a,b))) fp32 matrices."""
        di, do = pair
        pc = self.kernel_unary[f'({di},{do})']
        Kp = Fp.shape[1]
        Fv = Fp.view(pc.nc_out, pc.nc_in, pc.num_freq, Kp).double()
        c0, ca, cb = (t.to(Fp.device) for t in _aligned.aligned_coeffs(di, do))
        ws = [torch.einsum('oifk,f->oik', Fv, c0).reshape(-1, Kp).float().contiguous()]
        for m in range(1, min(di, do) + 1):
            ab = torch.stack([torch.einsum('oifk,f->oik', Fv, ca[m - 1]), torch.einsum('oifk,f->oik', Fv, cb[m - 1])], dim=2)
            ws.append(ab.reshape(-1, Kp).float().contiguous())
        return ws

    def _pack_images(self, pair, kind, Fp):
        """pairwise_lr images of one pair in formulation `kind` (see lowrank_plan)."""
        pc = self.kernel_unary[f'({pair[0]},{pair[1]})']
        Co, Ci, nf, Kp = pc.nc_out, pc.nc_in, pc.num_freq, Fp.shape[1]
        if kind == 'aligned':
            return [ops.pack_lowrank(w, Co, Ci, 1 if m == 0 else 2, Kp) for m, w in enumerate(self.aligned_weights(pair, Fp))]
        if kind == 'input_side':
            Fv = Fp.view(Co, Ci, nf, Kp)
            return [ops.pack_lowrank(Fv[:, :, f, :].reshape(-1, Kp).contiguous(), Co, Ci, 1, Kp) for f in range(nf)]
        return [ops.pack_lowrank(Fp, Co, Ci, nf, Kp)]

    def _zgemm_images(self, zweights, mode_m):
        """{(do, m): dict(img, S, degs, mode)}: the aligned weights of the pairs (di >= m, do) as one GEMM image (DESIGN.md 4.5);
        the |m| > 0 images in kernel mode mode_m (3: three real products per complex one, 3/4 of the tensor-core work of 2)."""
        zplan = {}
        for do, mo in self.fiber_out:
            for m in range(do + 1):
                degs = [(di, mi) for di, mi in self.fiber_in if di >= m]
                if not degs:
                    continue
                mode = 1 if m == 0 else mode_m
                img, S = ops.zgemm_image([(zweights[(di, do)][m], mi) for di, mi in degs], mo, mode)
                zplan[(do, m)] = dict(img=img, S=S, degs=degs, mode=mode)
        return zplan

    def _plan_stacks(self, pairs, dev):
        """Operands of the radial kernels over all pairs (zero where a pair has no plan): Vstack [pairs, 128, 64], gmean
        [pairs, 128], ones_col [pairs] (the column of U that holds 1) and have [pairs] (the pair is in the plan)."""
        pps = [pairs.get(pair) for pair in self.pairs]
        Vs = torch.stack([pp['V'] if pp else torch.zeros((ops.RADIAL_MID, 64), device=dev) for pp in pps])
        gm = torch.stack([pp['gmean'] if pp else torch.zeros(ops.RADIAL_MID, device=dev) for pp in pps])
        return dict(Vstack=Vs, gmean=gm, ones_col=torch.tensor([pp['r'] if pp else 0 for pp in pps], dtype=torch.int32, device=dev),
                    have=torch.tensor([pp is not None for pp in pps], dtype=torch.bool, device=dev))

    UTABLE_TOL = 5e-7        # max interpolation error of the tabulated radial coordinates relative to max|g| (float64, grid midpoints)

    def radial_table(self, ugrid, bases, grid, dev):
        """The radial coordinates U(d) = (g(d) - gmean) V of every pair tabulated on the plan's uniform distance grid (float64 ->
        fp32 [pairs, G, KT]); the forward interpolates them (se3_radial_table_fwd, 4-point Lagrange) instead of evaluating the MLP
        per edge.  Accepted only if the interpolant reproduces the float64 trunk at the grid MIDPOINTS to UTABLE_TOL (smooth
        radial functions pass by orders of magnitude; a rougher one falls back to se3_radial_trunk_u_fwd)."""
        Gn = grid.shape[0]
        KT = max(lowrank_k(bases[p][0]) for p in self.pairs)
        tab = torch.zeros((len(self.pairs), Gn, KT), dtype=torch.float32, device=dev)
        mid = (grid[:-1] + grid[1:]) * 0.5
        featm = self.encode_dist(mid)
        worst = 0.0
        for pi, pair in enumerate(self.pairs):
            r, V, gmean = bases[pair]
            Ug, gmax = ugrid[pair]
            tab[pi, :, :r] = Ug.float()
            pc = self.kernel_unary[f'({pair[0]},{pair[1]})']
            exact = (pc.rp.trunk64(featm) - gmean) @ V                                      # [G-1, r] float64
            T = tab[pi, :, :r].double()
            i0 = torch.arange(Gn - 1, device=dev).clamp(1, Gn - 3)                          # as the kernel chooses its 4 nodes
            f = (torch.arange(Gn - 1, device=dev, dtype=torch.float64) + 0.5 - i0).unsqueeze(-1)
            w = (-f * (f - 1) * (f - 2) / 6, (f + 1) * (f - 1) * (f - 2) / 2, -(f + 1) * f * (f - 2) / 2, (f + 1) * f * (f - 1) / 6)
            interp = sum(w[j] * T[i0 - 1 + j] for j in range(4))
            worst = max(worst, float((interp - exact).abs().max()) / max(gmax, 1e-30))
        self.utable_error = worst
        return tab if worst <= self.UTABLE_TOL else None

    def zgemm_eligible(self, kps):
        """Shapes the one-GEMM kernel takes: every C_out a multiple of 128, every C_in a multiple of 4 (one stage = 64 K values),
        at most 16 K segments per launch (a pair with K = 16 j contributes j), and |g|_2 small enough for the fp16 operands
        (|Z| <= 2^10 |U|, |U_k| <= |g|_2 <= 11.32 (max|ln.w| + max|ln.b|))."""
        if any(mo % 128 for _, mo in self.fiber_out) or any(mi % 4 for _, mi in self.fiber_in):
            return False
        for do, _ in self.fiber_out:
            if sum(kps[(di, do)] // 16 for di, _ in self.fiber_in) > 16:
                return False
        for di, do in self.pairs:
            ln = self.kernel_unary[f'({di},{do})'].rp.net['4']
            if 11.32 * (float(ln.weight.abs().max()) + float(ln.bias.abs().max())) > 60.0:
                return False
        return True

    def pack_weights(self, free_master=False, max_distance=None):
        """Build the tensor-core weight images now.  With max_distance (an upper bound on the neighbour distances the model
        will see) and distance-only radial functions, the low-rank plan is built and pairs it covers need no direct
        (K = 128) image.  free_master=True then releases the fp32 net.6 weights of every imaged pair (inference only:
        state_dict() no longer holds them)."""
        sw = switches.current()
        covered = {}
        if max_distance is not None and self.edge_dim == 0 and not sw.no_lowrank:
            covered = self.lowrank_plan(float(max_distance) / 1.25, sw)['pairs']
        for di, do in self.pairs:
            if self.tc_eligible(di, do) and (di, do) not in covered:
                self.w3_image(di, do)
        if free_master:
            pk = self._weights()
            self.free_master = True
            for key in list(pk['images']) + list(covered):
                lin = self.kernel_unary[f'({key[0]},{key[1]})'].rp.net['6']
                lin.weight.data = torch.empty(0, device=pk['trunk'].device)
        return self.packed()

    # ---- forward ----------------------------------------------------------------------------------------
    def edge_features(self, edge_info, rel_dist):
        _, _, edges = edge_info
        rd = self.encode_dist(rel_dist.unsqueeze(-1))
        feat = torch.cat((rd, edges), dim=-1) if exists(edges) else rd
        return feat.reshape(-1, feat.shape[-1]).contiguous()

    def forward(self, inp, edge_info, rel_dist=None, basis=None):
        flat, plan, geom = split_basis(basis)
        decisions = [conv_decide(self, edge_info[0].numel(), rel_dist, geom)]
        whole_self = {}          # node chunks add their rows of the whole graph's self-interaction, made for the first of them

        def evaluate(c, cbasis, sx):
            if not c.whole and self.self_interaction and not whole_self:
                whole_self.update(self.self_interact(inp))
            return conv_forward([self], c.src(inp), c.edge_info(edge_info), c.rows(rel_dist), cbasis, decisions=decisions,
                                self_out=c.rows(whole_self) if whole_self else None, sx=sx)[0]
        return over_node_chunks((flat, plan, geom), decisions, inp, edge_info[0], evaluate)


def input_side(di, do):
    """Degree pairs evaluated with the input-side contraction on the low-rank path: out = B . (R x) instead of R (B x).
    The fused kernel then spends 2 l_in + 1 instead of 2 l_out + 1 FMAs per radial weight; worth it for l_in <= 1 < l_out
    and for l_in = 0 (measured: (0,3) 7.7 -> 2.6 ms, (1,3) 19.3 -> ~11.4 ms at cfg2 widths).  Off with the no_input_side switch."""
    return di < do and di <= 1


def lowrank_k(r):
    """K of a rank-r low-rank pair: r columns of U and its ones column, padded to a multiple of 16."""
    return 16 * ((r + 1 + 15) // 16)


class Geometry:
    """Per-forward edge geometry shared by every layer; the aligned frames and the flat basis are built on first use, the frames
    by the code that the host_frames switch selects when the Geometry is made.  chunk() gives the Geometry of the edges of one
    node chunk (NodeChunk), which builds its own frames and basis and shares the whole graph's d_max and deferred checks.

    deferred: where the run-time checks of the low-rank plans go, as (ConvSE3, stats [pairs, 2], have): None = check inside
    every ConvSE3 (one host synchronisation each); a list = the caller collects them and checks once per forward
    (SE3Transformer.forward).  edge_budget: bytes the edge-level tensors of one block may take (edge_budget_bytes), or None:
    every block runs as one chunk."""

    def __init__(self, rel_pos, max_degree, deferred=None, edge_budget=None, whole=None):
        self.rel_pos, self.max_degree, self._frames, self._basis = rel_pos, max_degree, None, None
        self.deferred, self.edge_budget = deferred, edge_budget
        self.whole = self if whole is None else whole
        self.host_frames = switches.current().host_frames if whole is None else whole.host_frames
        self._dmax = None

    def d_max(self, rel_dist):
        if self is not self.whole:
            return self.whole.d_max(rel_dist)
        if self._dmax is None:
            self._dmax = float(rel_dist.max())          # the one host synchronisation of the plan lookup, once per forward
        return self._dmax

    def chunk(self, c):
        """The Geometry of the edges of node chunk c (self when c is the whole graph)."""
        if c.whole:
            return self
        return Geometry(c.rows(self.rel_pos), self.max_degree, self.deferred, self.edge_budget, whole=self)

    def basis(self):
        """(flat basis buffer, BasisPlan) of these edges (ops.basis_flat), for the R-first route."""
        if self._basis is None:
            self._basis = ops.basis_flat(self.rel_pos, self.max_degree)
        return self._basis

    def to_global(self, akv):
        """AlignedKV -> [b, n, k, C, 2lo+1] in the global frame (the rotate-back the attention kernel otherwise fuses)."""
        if not isinstance(akv, AlignedKV):
            return akv
        b, n, k, P, C = akv.t.shape
        E = b * n * k
        out = torch.empty((E, C, P), dtype=torch.float32, device=akv.t.device)
        ops.fold_basis(akv.t.reshape(1, E, P, C), self.frames().D[akv.lo].reshape(-1), E, C, P, P, 1, out, accumulate=False,
                       component_major=True, name='rotate_back')
        return out.view(b, n, k, C, P)

    def frames(self):
        """Per-edge Wigner matrices D_l(R_e) (se3_frames_fwd, float64 arithmetic on the device; host_frames: the float64 torch
        restatement in aligned.py)."""
        if self._frames is None:
            if self.host_frames:
                self._frames = _aligned.EdgeFrames(self.rel_pos, self.max_degree)
            else:
                self._frames = _aligned.EdgeFrames(self.rel_pos, self.max_degree, D=ops.frames(self.rel_pos, self.max_degree))
        return self._frames


def check_lowrank_stats(checks):
    """checks: [(ConvSE3, stats [pairs, 2] = (max |g - U V^T|, max |g|) of one forward)].  ONE host synchronisation for all of
    them; returns the ConvSE3 modules whose cached radial basis does not cover this forward's distances."""
    global LAST_PLAN_RESIDUAL
    if not checks:
        return []
    worst = torch.stack([torch.where(have, st[:, 0] / st[:, 1].clamp(min=1e-30), torch.zeros_like(st[:, 0])).max() for _, st, have in checks]).cpu()
    LAST_PLAN_RESIDUAL = float(worst.max())      # diagnostics / tests: how close the last checked forward came to the guard
    return [conv for (conv, _, _), w in zip(checks, worst.tolist()) if not (w <= conv.LR_RUNTIME_TOL)]


LAST_PLAN_RESIDUAL = None


class AlignedKV:
    """A ConvSE3 output of degree lo >= 1 still in the edge-aligned frame (DESIGN.md 4.5): t [b, n, k, 2lo+1, C], component
    major, out[e, c, :] = D_lo(e) t[e, :, c].  AttentionSE3 hands it to the attention kernel, which rotates on the fly;
    Geometry.to_global() materialises the reference-layout tensor [b, n, k, C, 2lo+1]."""

    def __init__(self, t, lo):
        self.t, self.lo = t, lo


class LowRankPlanMiss(RuntimeError):
    """The radial trunk outputs of a forward left the cached low-rank subspace (distances beyond the plan's range)."""


def edge_chunks(E, tile_bytes):
    """(t0, tile_count, e0, ec) of consecutive chunks of edge tiles such that a chunk's workspace (tile_bytes per tile of
    ops.TILE_E edges) fits T_WORKSPACE_BYTES; edges e0 .. e0 + ec."""
    n_tiles = (E + ops.TILE_E - 1) // ops.TILE_E
    per_chunk = max(1, min(n_tiles, T_WORKSPACE_BYTES // tile_bytes))
    for t0 in range(0, n_tiles, per_chunk):
        tc = min(per_chunk, n_tiles - t0)
        e0 = t0 * ops.TILE_E
        yield t0, tc, e0, min(E - e0, tc * ops.TILE_E)


# ---- node chunks under the edge budget (DESIGN.md 4.7) -------------------------------------------------------------------
EDGE_BUDGET_FRACTION = 0.25      # default edge budget: this share of the device's total memory, per block


def edge_budget_bytes(sw, device):
    """The edge budget of a forward on `device` under the switches sw: edge_budget_mb MiB if set, else EDGE_BUDGET_FRACTION of
    the device's total (not free) memory, so that the chunking does not depend on what else is allocated."""
    if sw.edge_budget_mb is not None:
        return max(0, int(sw.edge_budget_mb * 2 ** 20))
    return int(torch.cuda.get_device_properties(device).total_memory * EDGE_BUDGET_FRACTION)


class NodeChunk(NamedTuple):
    """Nodes n0 .. n1 of batch rows b0 .. b1: whole rows (n0, n1 = 0, n) or a range inside one row (b1 = b0 + 1).  Its edges
    are one contiguous range of the [b, n, k] layout, whole neighbour lists only."""
    b0: int
    b1: int
    n0: int
    n1: int
    whole: bool = False            # the chunk is the whole graph

    def rows(self, t):
        """The chunk's rows of a [b, n, ...] tensor (node or edge level), or of every tensor of a dict; None stays None."""
        if t is None:
            return None
        if isinstance(t, dict):
            return {key: self.rows(v) for key, v in t.items()}
        return t[self.b0:self.b1, self.n0:self.n1]

    def src(self, t):
        """The node features [b, n, ...] that the chunk's neighbours are gathered from, as the kernels see them: a [b', n', ...]
        view that starts at the chunk's first batch row.  The kernels address a neighbour as (batch row of the edge) * n' + idx
        and a range inside one row has b' = 1, so every neighbour idx < n of that row lies inside the row's storage."""
        if isinstance(t, dict):
            return {key: self.src(v) for key, v in t.items()}
        return t[self.b0:self.b1, :self.n1 - self.n0]

    def edge_info(self, edge_info):
        return tuple(self.rows(t) for t in edge_info)


def plan_node_chunks(b, n, k, edge_bytes, budget):
    """Node chunks (NodeChunk) of a graph of b x n nodes with k neighbours each whose edges, at edge_bytes per edge, fit
    `budget` bytes: one chunk if the whole graph fits (or budget is None), else runs of whole batch rows, else ranges of nodes
    inside each row.  Chunks cover every node once, in order, and are balanced; the smallest is one node, whatever its size."""
    if budget is None or b * n * k * edge_bytes <= budget:
        return [NodeChunk(0, b, 0, n, whole=True)]
    cap = max(1, budget // max(1, k * edge_bytes))               # nodes per chunk
    if cap >= n:
        count = -(-b // (cap // n))
        rows = -(-b // count)
        return [NodeChunk(b0, min(b0 + rows, b), 0, n) for b0 in range(0, b, rows)]
    count = -(-n // cap)
    size = -(-n // count)
    return [NodeChunk(r, r + 1, n0, min(n0 + size, n)) for r in range(b) for n0 in range(0, n, size)]


def block_edge_bytes(decisions, max_degree, keep_aligned=False, attn_bytes=0):
    """Bytes per edge of the edge-level tensors that one node chunk of a block (the convolutions of `decisions`, which share
    inputs and graph) holds at its peak, from the fibers and routes: edge features, frames, flat basis, radial coordinates,
    outputs and the transient gathers / T blocks / out' of one edge chunk, plus attn_bytes of the attention glue.  An estimate."""
    c0 = decisions[0].conv
    fin, fout = c0.fiber_in, c0.fiber_out
    routes = {d.route for d in decisions}
    total = 4 * c0.in_dim + attn_bytes
    if routes & {'production', 'aligned'} or keep_aligned:
        total += 4 * sum(to_order(l) ** 2 for l in range(1, max_degree + 1))                          # frames D_l
    if 'production' in routes:
        total += 4 + 4 * sum(mi * to_order(di) for di, mi in fin) + 4 * max(mo * to_order(do) for do, mo in fout)   # sx, X, out'
    if routes & {'aligned', 'rfirst'}:
        total += max(ops.t_numel(1, mi, to_order(min(di, do)), to_order(do)) * 4 for di, mi in fin for do, _ in fout) // ops.TILE_E
    if 'rfirst' in routes:
        L = range(max_degree + 1)
        total += 4 * sum(to_order(do) * to_order(di) * to_order(min(di, do)) for di in L for do in L)   # flat basis
        total += 4 * max(to_order(min(di, do)) * mo * to_order(di) + mi * to_order(di) for di, mi in fin for do, mo in fout)
    for d in decisions:
        pairs = len(d.conv.pairs)
        total += 4 * 64 * pairs * bool(d.lr) + 4 * ops.RADIAL_MID * pairs * d.direct             # U, g
        if not (d.route == 'production' and d.conv.pool):
            total += 4 * sum(mo * to_order(do) for do, mo in fout)                                 # outputs
    return total


def chunk_edge_scale(decisions, inp, idx):
    """The production route's per-edge scale (ops.edge_scale) of the whole graph as [b, n, k], for the node chunks to slice: its
    node maxima cover every row, which a chunk's view of the features does not.  None if no convolution takes that route."""
    if not any(d.route == 'production' for d in decisions):
        return None
    return ops.edge_scale(inp, idx, max(di for di, _ in decisions[0].conv.fiber_in)).view(idx.shape)


def over_node_chunks(basis, decisions, inp, idx, evaluate, keep_aligned=False, attn_bytes=0):
    """The edge work of one block -- the convolutions of `decisions` on the graph idx [b, n, k] with node features inp -- over
    the node chunks that the edge budget of the block's Geometry allows (DESIGN.md 4.7); basis: (flat, BasisPlan, Geometry or
    None).  evaluate(c, chunk basis, sx) gives the outputs {key: [b', n', ...]} of NodeChunk c; sx: c's rows of the whole
    graph's edge scales (chunk_edge_scale).  The whole graph (one chunk, also without a Geometry or a budget) gets the block's
    basis and sx None, and its outputs are returned as they are; otherwise each chunk gets its own Geometry and its outputs
    land in their rows of [b, n, ...] tensors."""
    _, _, geom = basis
    b, n, k = idx.shape
    per_edge = 0 if geom is None else block_edge_bytes(decisions, geom.max_degree, keep_aligned, attn_bytes)
    chunks = plan_node_chunks(b, n, k, per_edge, None if geom is None else geom.edge_budget)
    if len(chunks) == 1:
        return evaluate(chunks[0], basis, None)
    sx = chunk_edge_scale(decisions, inp, idx)
    out = None
    for c in chunks:
        res = evaluate(c, (None, None, geom.chunk(c)), c.rows(sx))
        if out is None:
            out = {key: t.new_empty((b, n) + t.shape[2:]) for key, t in res.items()}
        for key, t in res.items():
            c.rows(out[key]).copy_(t)
    return out


class ConvDecision:
    """What one ConvSE3 decides once per forward, from the whole graph (conv_decide): the switches sw, tc_ok {pair: bool}, the
    low-rank plan or None, its covered pairs lr and the route they give, whether direct kernels need g, and the stats
    [pairs, 2] that the radial launches of every chunk accumulate into; deferred: the check is queued on Geometry.deferred."""

    def __init__(self, conv, sw, tc_ok, plan, stats, deferred):
        self.conv, self.sw, self.tc_ok, self.plan, self.stats, self.deferred = conv, sw, tc_ok, plan, stats, deferred
        self.lr = dict(plan['pairs']) if plan is not None else {}
        kinds = {pp['kind'] for pp in self.lr.values()}
        self.route = 'production' if 'z' in kinds else 'aligned' if 'aligned' in kinds else 'rfirst'
        self.direct = self.route == 'rfirst' and len(self.lr) < len(conv.pairs)


class ConvDispatch:
    """How one ConvSE3 runs on one set of edges (conv_dispatch) under its decision d (ConvDecision), which gives conv, sw, plan,
    route and lr.  route: 'production' (DESIGN.md 4.5, GEMM images plan['z']), 'aligned' (4.4) or 'rfirst' (4.1-4.3, with each
    pair's kernel in how: 'input_side', 'combined', 'tc' or 'simt').  U [pairs, E, 64]: radial coordinates of the low-rank pairs
    lr = {pair: plan entry}; g [pairs, E, 128]: trunk outputs for the direct kernels.  Outputs go to outs {do: [E, Co, 2do+1]},
    or on the production route to pooled or aligned_out."""

    def __init__(self, d, U, g, how, outs):
        self.d, self.U, self.g, self.how, self.outs = d, U, g, how, outs
        self.pooled = self.self_out = None
        self.aligned_out = {}

    conv = property(operator.attrgetter('d.conv'))
    sw = property(operator.attrgetter('d.sw'))
    plan = property(operator.attrgetter('d.plan'))
    route = property(operator.attrgetter('d.route'))
    lr = property(operator.attrgetter('d.lr'))


def _forward_plan(conv, sw, tc_ok, E, rel_dist, geom):
    """The low-rank plan this forward of `conv` reads, or None (direct kernels)."""
    pk = conv.packed(sw)
    if sw.no_lowrank or conv.edge_dim != 0:
        return None
    if conv.free_master and pk['lr'] is not None:
        return pk['lr']                     # built by pack_weights(max_distance=...) before the masters went away:
                                            # the only image there is, whatever the edge count
    if ops.lowrank_enabled(E, sw) and any(tc_ok.values()) and not conv.free_master and not conv._lr_blocked:
        if torch.cuda.is_current_stream_capturing():
            return pk['lr']                 # built by the warm-up forwards; the residual check still covers it
        # cached; needs the distance range (one host sync per forward, in Geometry)
        return conv.lowrank_plan(geom.d_max(rel_dist) if geom is not None else float(rel_dist.max()), sw)
    return None


def conv_decide(conv, E, rel_dist, geom):
    """What `conv` decides once per forward, from the whole graph (E edges, distances rel_dist): the switches, tc_ok and the
    low-rank plan, which therefore stay the same in every node chunk.  A plan's run-time check is queued on geom.deferred
    here, once, over stats that the radial launches of all chunks accumulate into; without a deferred list conv_dispatch
    checks it after its launches."""
    sw = switches.current()
    tc_ok = {pair: conv.tc_eligible(*pair) for pair in conv.pairs}
    plan = _forward_plan(conv, sw, tc_ok, E, rel_dist, geom)
    if plan is None or not plan['pairs']:
        return ConvDecision(conv, sw, tc_ok, None, None, False)
    stats = torch.zeros((len(conv.pairs), 2), dtype=torch.float32, device=rel_dist.device)
    deferred = geom is not None and geom.deferred is not None
    if deferred:
        geom.deferred.append((conv, stats, plan['have']))          # checked once per forward by the caller
    return ConvDecision(conv, sw, tc_ok, plan, stats, deferred)


def conv_dispatch(d, edge_info, rel_dist, geom):
    """Launch the radial kernels of the convolution of decision d on these edges (U of the low-rank pairs from the plan's table
    or the trunk, g for the direct kernels) and set up its outputs.  A plan miss checked here replaces d by the decision
    without a plan."""
    conv, idx = d.conv, edge_info[0]
    E, dev = idx.numel(), idx.device
    pk = conv.packed(d.sw)
    feat = conv.edge_features(edge_info, rel_dist)
    assert feat.shape[-1] == conv.in_dim, f'edge feature width {feat.shape[-1]} != {conv.in_dim}'
    U = g = None
    plan = d.plan
    if plan is not None:
        covered = len(plan['pairs']) == len(conv.pairs)
        if covered and plan['utab'] is not None and not d.sw.no_utable:
            U = ops.radial_table(rel_dist, plan['utab'], plan['D'], plan['ones_col'], d.stats)
        else:
            U, g = ops.radial_trunk_u(feat, pk['trunk'], plan['Vstack'], plan['gmean'], plan['ones_col'], d.stats, want_g=not covered)
        if not d.deferred and check_lowrank_stats([(conv, d.stats, plan['have'])]):
            # the fp32 trunk outputs of this forward leave the cached subspace (distances beyond the plan's range)
            if conv.free_master:
                raise LowRankPlanMiss('low-rank radial plan does not cover this input; pack_weights(max_distance=...) was given too '
                                      'small a distance')
            d = ConvDecision(conv, d.sw, d.tc_ok, None, None, False)       # evaluate this ConvSE3 with the direct K = 128 kernels
    if d.route != 'rfirst' and geom is None:     # edge-aligned plans cover every pair of the ConvSE3 and need the Geometry
        raise RuntimeError('ConvSE3 was called with a (flat, plan) basis: the edge-aligned low-rank plan needs the third element, '
                           'model.Geometry(rel_pos, max_degree), as SE3Transformer.forward passes it (or set SE3B200_NO_ALIGNED=1)')
    if d.direct and g is None:
        g = ops.radial_trunk(feat, pk['trunk'], len(conv.pairs))       # the direct kernels consume g itself
    how = {pair: d.lr[pair]['kind'] if pair in d.lr else 'tc' if d.tc_ok[pair] else 'simt' for pair in conv.pairs}
    # (the production route allocates the outputs it writes in _production_forward: pooled ones go to the nodes directly)
    outs = {} if d.route == 'production' else \
        {do: torch.empty((E, mo, to_order(do)), dtype=torch.float32, device=dev) for do, mo in conv.fiber_out}
    return ConvDispatch(d, U, g, how, outs)


def split_basis(basis):
    """The basis argument of ConvSE3, AttentionSE3 and conv_forward -- (flat, BasisPlan), (flat, BasisPlan, Geometry) or
    (None, None, Geometry) -- as (flat, BasisPlan, Geometry or None)."""
    if isinstance(basis, dict):
        raise TypeError("ConvSE3 takes the basis as the tuple (flat buffer, BasisPlan, Geometry) that SE3Transformer.forward builds: "
                        "`ops.basis_flat(rel_pos, max_degree) + (model.Geometry(rel_pos, max_degree),)`; the dict returned by the "
                        "drop-in get_basis() is the reference's per-pair view of the same buffer and is not accepted here")
    flat, plan = basis[:2]
    return flat, plan, basis[2] if len(basis) > 2 else None


def conv_forward(convs, inp, edge_info, rel_dist, basis, keep_aligned=False, decisions=None, self_out=None, sx=None):
    """Evaluate one or more ConvSE3 that share input features, graph and fibers (to_k / to_v of an attention block)
    in a single sweep: the T blocks (gather x basis) are built once per (degree pair, edge chunk) and consumed by every
    convolution's fused pairwise kernel.  Each convolution's decision (conv_decide, made here just before its dispatch if
    decisions is None) gives its route; the production convolutions run first, then the edge-aligned ones, then the R-first
    ones (the last two share one T workspace).

    basis: see split_basis; (None, None, Geometry) builds the flat basis from the Geometry only if an R-first route needs it.
    For one node chunk of a larger graph (over_node_chunks), the caller passes the chunk's edges, the features as
    NodeChunk.src gives them, the chunk's Geometry and the whole graph's decisions, plus the chunk's rows of the whole graph's
    self-interaction (self_out, one pooled convolution) and edge scales (sx [b', n', k], production route)."""
    c0 = convs[0]
    forward_only_guard('ConvSE3', convs, list(inp.values()) + [rel_dist])
    idx = edge_info[0]
    E = idx.numel()
    flat, plan, geom = split_basis(basis)
    states = []
    for i, conv in enumerate(convs):
        assert conv.pairs == c0.pairs and conv.in_dim == c0.in_dim
        d = decisions[i] if decisions else conv_decide(conv, E, rel_dist, geom)
        states.append(conv_dispatch(d, edge_info, rel_dist, geom))
    if self_out is not None:
        assert len(states) == 1
        states[0].self_out = self_out
    routes = {r: [st for st in states if st.route == r] for r in ('production', 'aligned', 'rfirst')}
    if routes['production']:
        _production_forward(routes['production'], inp, edge_info, geom, keep_aligned, sx)
    # the R-first routes chunk over edge tiles so that the largest T block fits the workspace
    t_bytes = max(ops.t_numel(1, mi, to_order(min(di, do)), to_order(do)) * 4 for di, mi in c0.fiber_in for do, _ in c0.fiber_out)
    workspace = None
    if routes['aligned']:
        workspace = _aligned_forward(routes['aligned'], inp, idx, geom, t_bytes, workspace)
    if routes['rfirst']:
        if flat is None:
            flat, plan = geom.basis()
        _rfirst_forward(routes['rfirst'], inp, idx, ops.basis_pairs(flat, plan, E), t_bytes, workspace)
    return [_conv_results(st, inp, edge_info) for st in states]


def _production_forward(states, inp, edge_info, geom, keep_aligned, sx=None):
    """DESIGN.md 4.5: the neighbour features rotated into the edge frame once per input degree and edge chunk, ONE GEMM per
    (conv, degree_out, |m|) over all input degrees, then the rotation back: fused with the masked mean and the self-interaction
    for pooled convolutions (conv_in / conv_out), or left to the attention kernel with keep_aligned."""
    idx, nmask, _ = edge_info
    b, n, k = idx.shape
    fiber_in = states[0].conv.fiber_in
    frames = geom.frames()
    # (a node chunk's view of the features holds the node maxima of its own rows only: it takes the whole graph's scales)
    assert sx is not None or geom.whole is geom, 'the production route of a node chunk needs the whole graph\'s edge scales'
    sx = ops.edge_scale(inp, idx, max(di for di, _ in fiber_in)) if sx is None else sx.reshape(-1)
    tile_bytes = sum(mi * to_order(di) for di, mi in fiber_in) * ops.TILE_E * 4
    chunks = list(edge_chunks(idx.numel(), tile_bytes))
    # the fused pool needs edge chunks of whole neighbour lists; decided on the whole graph, so that every node chunk of it
    # pools the same way (whole-graph chunks of whole lists imply the same for the fewer edges of a node chunk)
    fuse_pool = all(e0 % k == 0 for _, _, e0, _ in edge_chunks(geom.whole.rel_pos.numel() // 3, tile_bytes))
    for st in states:
        conv = st.conv
        if conv.pool and fuse_pool:
            st.pooled = {do: torch.empty((b * n, mo, to_order(do)), dtype=torch.float32, device=idx.device) for do, mo in conv.fiber_out}
            if st.self_out is None:
                st.self_out = conv.self_interact(inp) if conv.self_interaction else {}
        elif keep_aligned:                   # the consumer (attention) rotates back on the fly: keep out' itself
            st.aligned_out = {do: torch.empty((idx.numel(), to_order(do), mo), dtype=torch.float32, device=idx.device)
                              for do, mo in conv.fiber_out if do > 0}
        if st.pooled is None:
            st.outs = {do: torch.empty((idx.numel(), mo, to_order(do)), dtype=torch.float32, device=idx.device)
                       for do, mo in conv.fiber_out if do not in st.aligned_out}
    nmask_flat = None if nmask is None else nmask.reshape(-1)
    for t0, tc, e0, ec in chunks:
        X = {di: ops.rotgather(inp[str(di)], idx, frames.D[di] if di > 0 else None, t0, tc) for di, _ in fiber_in}
        for st in states:
            for do, mo in st.conv.fiber_out:
                P = to_order(do)
                Op = _zgemm_degree(st, do, mo, X, sx, e0, ec)
                if st.pooled is not None:        # rotate back + masked mean over k + self-interaction, one kernel
                    sa = st.self_out.get(str(do))
                    ops.rotate_pool(Op, frames.D[do][e0:e0 + ec] if do > 0 else None, None if nmask_flat is None else nmask_flat[e0:e0 + ec],
                                    None if sa is None else sa.reshape(b * n, mo, P)[e0 // k:(e0 + ec) // k], ec // k, k, mo, do,
                                    st.pooled[do][e0 // k:(e0 + ec) // k])
                elif do > 0 and do not in st.aligned_out:        # back to the global frame: out = D_lo out'
                    ops.fold_basis(Op.view(1, ec, P, mo), frames.D[do][e0:e0 + ec].reshape(-1), ec, mo, P, P, 1,
                                   st.outs[do][e0:e0 + ec], accumulate=False, component_major=True, name='rotate_back')
        del X


def _zgemm_degree(st, do, mo, X, sx, e0, ec):
    """out' [ec, 2do+1, Co] (edge frame, component major) of output degree do on edges e0 .. e0 + ec: one zgemm per |m|, whose
    K segments are the 16-column blocks of U of every input degree."""
    conv, P = st.conv, to_order(do)
    z = st.plan['z']
    full = all((do, m) in z for m in range(do + 1))
    if do == 0 and st.pooled is None:
        Op = st.outs[0][e0:e0 + ec]                   # [ec, mo, 1] is [ec, 1, mo]
    elif do in st.aligned_out:
        Op = st.aligned_out[do][e0:e0 + ec]
        if not full:
            Op.zero_()
    else:
        Op = (torch.empty if full else torch.zeros)((ec, P, mo), dtype=torch.float32, device=sx.device)
    for m in range(do + 1):
        zp = z.get((do, m))
        if zp is None:
            continue
        segs, alg = [], 0
        for di, mi in zp['degs']:
            pi = conv.pairs.index((di, do))
            for kc in range(st.lr[(di, do)]['Kp'] // 16):
                segs.append((st.U[pi, e0:e0 + ec, 16 * kc:], X[di], mi, to_order(di), di + m, di - m))
            alg += ec * mo * mi * 2 * (ops.RADIAL_MID + P) * (1 if m == 0 else 2)
        ops.zgemm(segs, zp['img'], sx[e0:e0 + ec], ec, mo, zp['mode'], Op, P * mo, [(do + m) * mo, (do - m) * mo],
                  flush_stages=st.sw.zgemm_flush(zp['mode']), alg_flops=alg, tag=f'mode{zp["mode"]}lo{do}m{m}Co{mo}S{zp["S"]}')
    return Op


def _aligned_forward(states, inp, idx, geom, t_bytes, workspace):
    """DESIGN.md 4.4: per edge chunk and (input degree, |m|), the neighbour features rotated into the edge frame (T blocks of
    the aligned basis), two output components per pairwise_lr launch, then the rotation back to the global frame."""
    c0 = states[0].conv
    frames = geom.frames()
    for t0, tc, e0, ec in edge_chunks(idx.numel(), t_bytes):
        # out' of degree do lives in one dense buffer per |m|: [edges, C_out] for m = 0, [edges, C_out, 2] = (+m, -m) otherwise
        # (the kernel's native layout); first contribution overwrites, later input degrees accumulate
        outp = [{} for _ in states]
        for di, mi in c0.fiber_in:
            for m in range(di + 1):
                targets = [(do, mo) for do, mo in c0.fiber_out if do >= m]
                if not targets:
                    continue
                Pk = Fk = 1 if m == 0 else 2
                workspace = ops.tbuild_blocks(inp[str(di)], idx, frames.block(di, m), Pk, Fk, t0, tc, out=workspace)
                for do, mo in targets:
                    P = to_order(do)
                    for st, op in zip(states, outp):
                        lrp = st.lr[(di, do)]
                        first = (do, m) not in op
                        if first:
                            op[(do, m)] = st.outs[do][e0:e0 + ec] if do == 0 else torch.empty((ec, mo, Pk), dtype=torch.float32, device=idx.device)
                        ops.pairwise_lr(st.U[c0.pairs.index((di, do)), e0:e0 + ec], lrp['images'][m], workspace, ec, mo, mi, Fk, Pk,
                                        lrp['Kp'], op[(do, m)], accumulate=not first, alg_units=Fk * 2 * (ops.RADIAL_MID + P))
        for st, op in zip(states, outp):
            for do, mo in c0.fiber_out:
                if do > 0:                      # back to the global frame: out = D_lo out'
                    ops.rotate_back([op.get((do, m)) for m in range(do + 1)], frames.D[do][e0:e0 + ec].reshape(-1), ec, mo, do,
                                    st.outs[do][e0:e0 + ec])
                elif (0, 0) not in op:
                    st.outs[0][e0:e0 + ec].zero_()
        del outp
    return workspace


def _rfirst_forward(states, inp, idx, bpairs, t_bytes, workspace):
    """DESIGN.md 4.1-4.3 in the global frame: per edge chunk and degree pair one T block (gather x basis) shared by every
    convolution, then per convolution the pair's kernel -- combined low-rank, direct tensor-core or SIMT -- accumulating over
    the input degrees; or the input-side contraction, on the gathered neighbour features, folded with the basis afterwards."""
    c0 = states[0].conv
    for t0, tc, e0, ec in edge_chunks(idx.numel(), t_bytes):
        gathered = {}                            # degree_in -> neighbour features of this chunk in tile layout
        for do, mo in c0.fiber_out:
            P = to_order(do)
            accumulate = False                   # the first input degree overwrites, the others accumulate
            for di, mi in c0.fiber_in:
                Fq, Q = to_order(min(di, do)), to_order(di)
                pi = c0.pairs.index((di, do))
                hows = [st.how[(di, do)] for st in states]
                if 'input_side' in hows and di not in gathered:
                    gathered[di] = ops.gather_tiles(inp[str(di)], idx, t0, tc)
                if any(h != 'input_side' for h in hows):
                    workspace = ops.tbuild(inp[str(di)], idx, bpairs[(di, do)], di, do, t0, tc, out=workspace)
                for st, how in zip(states, hows):
                    conv = st.conv
                    out = st.outs[do][e0:e0 + ec]
                    if how == 'input_side':
                        # S[f,e,o,q] = sum_i R[e,o,i,f] x[j(e),i,q], then out[e,o,p] (+)= sum_{f,q} B[e,p,q,f] S[f,e,o,q]
                        S = torch.empty((Fq, ec, mo, Q), dtype=torch.float32, device=idx.device)
                        for f in range(Fq):
                            ops.pairwise_lr(st.U[pi, e0:e0 + ec], st.lr[(di, do)]['images'][f], gathered[di], ec, mo, mi, 1, Q,
                                            st.lr[(di, do)]['Kp'], S[f], accumulate=False, alg_P=P)
                        ops.fold_basis(S, bpairs[(di, do)][e0 * P * Q * Fq:(e0 + ec) * P * Q * Fq], ec, mo, P, Q, Fq, out,
                                       accumulate=accumulate)
                        del S
                    elif how == 'combined':
                        ops.pairwise_lr(st.U[pi, e0:e0 + ec], st.lr[(di, do)]['images'][0], workspace, ec, mo, mi, Fq, P,
                                        st.lr[(di, do)]['Kp'], out, accumulate=accumulate)
                    elif how == 'tc':
                        ops.pairwise_tc(st.g[pi, e0:e0 + ec], conv.w3_image(di, do), workspace, ec, mo, mi, Fq, P, out,
                                        accumulate=accumulate)
                    else:
                        lin = conv.kernel_unary[f'({di},{do})'].rp.net['6']
                        ops.pairwise_simt(st.g[pi, e0:e0 + ec], lin.weight, lin.bias, workspace, ec, mo, mi, Fq, P, out,
                                          accumulate=accumulate)
                accumulate = True
    return workspace


def _conv_results(st, inp, edge_info):
    """The outputs of one convolution as the reference returns them: pooled over the neighbours and with the self-interaction
    added where the ConvSE3 asks for them; AlignedKV for degrees kept in the edge frame."""
    conv = st.conv
    idx, nmask, _ = edge_info
    b, n, k = idx.shape
    if st.pooled is not None:
        return {str(do): st.pooled[do].view(b, n, mo, to_order(do)) for do, mo in conv.fiber_out}
    outputs = {}
    for do, mo in conv.fiber_out:
        if do in st.aligned_out:
            outputs[str(do)] = AlignedKV(st.aligned_out[do].view(b, n, k, to_order(do), mo), do)
        else:
            o = st.outs[do].view(b, n, k, mo, to_order(do))
            outputs[str(do)] = ops.pool(o, nmask) if conv.pool else o
    if conv.self_interaction:
        outputs = residual_add(outputs, conv.self_interact(inp) if st.self_out is None else st.self_out)
    return outputs


class FeedForwardSE3(nn.Module):
    """reference S:347-365"""

    def __init__(self, fiber, mult=4):
        super().__init__()
        hidden = Fiber([(d, c * mult) for d, c in fiber])
        self.project_in = LinearSE3(fiber, hidden)
        self.nonlin = NormSE3(hidden)
        self.project_out = LinearSE3(hidden, fiber)

    def forward(self, x, residual=None):
        return self.project_out(self.nonlin(self.project_in(x)), residual=residual)


class FeedForwardBlockSE3(nn.Module):
    """reference S:367-383"""

    def __init__(self, fiber, norm_gated_scale=False):
        super().__init__()
        self.prenorm = NormSE3(fiber, gated_scale=norm_gated_scale)
        self.feedforward = FeedForwardSE3(fiber)

    def forward(self, x):
        return self.feedforward(self.prenorm(x), residual=x)          # residual added in the epilogue of project_out


class AttentionSE3(nn.Module):
    """AttentionSE3 (reference S:387-519) and, with one_headed=True, OneHeadedKVAttentionSE3 (S:522-654)."""

    def __init__(self, fiber, dim_head=64, heads=8, attend_self=False, edge_dim=None, fourier_encode_dist=False,
                 rel_dist_num_fourier_features=4, use_null_kv=False, splits=4, global_feats_dim=None, linear_proj_keys=False,
                 tie_key_values=False, one_headed=False):
        super().__init__()
        hidden_dim = dim_head * heads
        self.fiber = fiber
        hidden_fiber = Fiber([(d, hidden_dim) for d, _ in fiber])
        kv_fiber = Fiber([(d, dim_head) for d, _ in fiber]) if one_headed else hidden_fiber
        project_out = not (heads == 1 and len(fiber.dims) == 1 and dim_head == fiber.dims[0])
        self.scale = dim_head ** -0.5
        self.heads, self.dim_head, self.one_headed = heads, dim_head, one_headed
        self.linear_proj_keys = linear_proj_keys
        conv_kw = dict(edge_dim=default(edge_dim, 0), pool=False, self_interaction=False, fourier_encode_dist=fourier_encode_dist,
                       num_fourier_features=rel_dist_num_fourier_features, splits=splits)
        self.to_q = LinearSE3(fiber, hidden_fiber)
        self.to_v = ConvSE3(fiber, kv_fiber, **conv_kw)
        assert not (linear_proj_keys and tie_key_values), 'you cannot do linear projection of keys and have shared key / values turned on at the same time'
        if linear_proj_keys:
            self.to_k = LinearSE3(fiber, kv_fiber)
        elif not tie_key_values:
            self.to_k = ConvSE3(fiber, kv_fiber, **conv_kw)
        else:
            self.to_k = None
        self.to_out = LinearSE3(hidden_fiber, fiber) if project_out else nn.Identity()
        self.use_null_kv = use_null_kv
        if use_null_kv:
            self.null_keys = nn.ParameterDict()
            self.null_values = nn.ParameterDict()
            for degree in fiber.degrees:
                shape = (dim_head, to_order(degree)) if one_headed else (heads, dim_head, to_order(degree))
                self.null_keys[str(degree)] = nn.Parameter(torch.zeros(*shape))
                self.null_values[str(degree)] = nn.Parameter(torch.zeros(*shape))
        self.attend_self = attend_self
        if attend_self:
            self.to_self_k = LinearSE3(fiber, kv_fiber)
            self.to_self_v = LinearSE3(fiber, kv_fiber)
        self.accept_global_feats = exists(global_feats_dim)
        if self.accept_global_feats:
            gin = Fiber.create(1, global_feats_dim)
            gout = Fiber.create(1, kv_fiber[0])
            self.to_global_k = LinearSE3(gin, gout)
            self.to_global_v = LinearSE3(gin, gout)

    def forward(self, features, edge_info, rel_dist, basis, global_feats=None, pos_emb=None, mask=None, residual=None):
        forward_only_guard('AttentionSE3', [self], list(features.values()))
        idx = edge_info[0]
        flat, plan, geom = split_basis(basis)
        fuse = self.fuse_rotation(geom)
        queries, kv, k_emb = self.node_level(features, global_feats, pos_emb)
        decisions = [conv_decide(conv, idx.numel(), rel_dist, geom) for conv in self.edge_convs()]
        attn_bytes = 0 if k_emb is None else 4 * self.to_v.fiber_out[0] * (4 + self.linear_proj_keys) + 4 * k_emb.shape[-1]
        outputs = over_node_chunks((flat, plan, geom), decisions, features, idx,
                                   lambda c, cbasis, sx: self._attend(c, features, queries, kv, k_emb, edge_info, rel_dist, cbasis,
                                                                      decisions, fuse, sx),
                                   keep_aligned=fuse, attn_bytes=attn_bytes)
        return self.project_out(outputs, residual)

    def fuse_rotation(self, geom):
        """The rotate-back of the values is fused into the attention kernel."""
        return geom is not None and not switches.current().no_attn_rotate and ops.attn_aligned_supported(self.dim_head)

    def edge_convs(self):
        """The convolutions that make keys and values on the edges, keys first."""
        return [self.to_v] if self.linear_proj_keys or self.to_k is None else [self.to_k, self.to_v]

    def project_out(self, outputs, residual):
        if isinstance(self.to_out, LinearSE3):
            return self.to_out(outputs, residual=residual)             # residual added in the epilogue of to_out
        return outputs if residual is None else residual_add(outputs, residual)

    def node_level(self, features, global_feats, pos_emb, node_keys=None):
        """Node-level work of the nodes of `features`: queries, (node keys, self keys, self values, global keys, global values)
        and the key rotary embedding; node_keys (linear_proj_keys) default to to_k of the features."""
        queries = self.to_q(features)
        if self.linear_proj_keys and node_keys is None:
            node_keys = self.to_k(features)
        self_keys = self_values = global_keys = global_values = None
        if self.attend_self:
            self_keys, self_values = self.to_self_k(features), self.to_self_v(features)
        if exists(global_feats):
            global_keys, global_values = self.to_global_k(global_feats), self.to_global_v(global_feats)
        k_emb = None
        if exists(pos_emb):
            # rotary embeddings on the type-0 queries / keys / values (reference S:488-494, 623-629; rotary.py:15-24): cheap
            # elementwise glue in torch around the attention kernel.  The key embedding has 1 + k positions, self first.
            assert self.attend_self, 'rotary embeddings need attend_self = True (the key positions include the node itself, as in the reference)'
            q_emb, k_emb = pos_emb                                     # [b, n, rot], [b, n, 1 + k, rot]
            b_, n_ = q_emb.shape[:2]
            Dh, hk = self.dim_head, (1 if self.one_headed else self.heads)
            queries = dict(queries)
            queries['0'] = apply_rotary_pos_emb(queries['0'].view(b_, n_, self.heads, Dh, 1), q_emb[:, :, None, :, None]).reshape(b_, n_, -1, 1)
            self_emb = k_emb[:, :, 0, None, :, None]
            self_keys, self_values = dict(self_keys), dict(self_values)
            self_keys['0'] = apply_rotary_pos_emb(self_keys['0'].view(b_, n_, hk, Dh, 1), self_emb).reshape(b_, n_, -1, 1)
            self_values['0'] = apply_rotary_pos_emb(self_values['0'].view(b_, n_, hk, Dh, 1), self_emb).reshape(b_, n_, -1, 1)
        return queries, (node_keys, self_keys, self_values, global_keys, global_values), k_emb

    def _attend(self, c, features, queries, kv, k_emb, edge_info, rel_dist, basis, decisions, fuse, sx):
        """The edge work of node chunk c (over_node_chunks): keys / values of its edges (the convolutions of the whole graph's
        decisions, keys first), then attention of its queries -> {degree: [b', n', H*Dh, 2d+1]}.  basis: the chunk's; sx: its
        rows of the whole graph's edge scales, None for the whole graph."""
        node_keys, self_keys, self_values, global_keys, global_values = kv
        edge_info = c.edge_info(edge_info)
        idx, nmask, _ = edge_info
        _, _, geom = basis
        outs = conv_forward([d.conv for d in decisions], c.src(features), edge_info, c.rows(rel_dist), basis, keep_aligned=fuse,
                            decisions=decisions, sx=sx)
        keys, values, k_idx = outs[0], outs[-1], None          # tie_key_values: one convolution, keys = values
        if self.linear_proj_keys:
            keys, k_idx = c.src(node_keys), idx                 # node level; the attention kernel gathers through idx
        if k_emb is not None:
            b_, n_, kk = idx.shape
            Dh, hk = self.dim_head, (1 if self.one_headed else self.heads)
            if k_idx is not None:                                      # linear_proj_keys: keys live on the nodes; rotary is per edge
                keys = dict(keys)
                keys['0'] = node_keys['0'][c.b0:c.b1][torch.arange(b_, device=idx.device)[:, None, None], idx]
            nb_emb = c.rows(k_emb)[:, :, 1:, None, :, None]
            new_k = apply_rotary_pos_emb(keys['0'].view(b_, n_, kk, hk, Dh, 1), nb_emb).reshape(b_, n_, kk, -1, 1)
            new_v = new_k if values is keys else apply_rotary_pos_emb(values['0'].view(b_, n_, kk, hk, Dh, 1), nb_emb).reshape(b_, n_, kk, -1, 1)
            keys, values = dict(keys), dict(values)
            keys['0'], values['0'] = new_k, new_v
        outputs = {}
        for degree in features.keys():
            kw = {}
            if self.attend_self:
                kw.update(self_k=c.rows(self_keys[degree]), self_v=c.rows(self_values[degree]))
            if self.use_null_kv:
                kw.update(null_k=self.null_keys[degree].reshape(-1, to_order(int(degree))),
                          null_v=self.null_values[degree].reshape(-1, to_order(int(degree))))
            if global_keys is not None and degree == '0':
                kw.update(global_k=global_keys[degree][c.b0:c.b1], global_v=global_values[degree][c.b0:c.b1])
            kd, vd = keys[degree], values[degree]
            if isinstance(vd, AlignedKV) or isinstance(kd, AlignedKV):
                if isinstance(kd, AlignedKV) and not isinstance(vd, AlignedKV):
                    kd = geom.to_global(kd)           # (keys and values come from the same dispatch: not reached in practice)
                if isinstance(vd, AlignedKV):
                    k_al = isinstance(kd, AlignedKV)
                    kw.update(D=geom.frames().D[int(degree)], k_aligned=k_al)
                    kd, vd = (kd.t if k_al else kd), vd.t
            outputs[degree] = ops.attention(c.rows(queries[degree]), kd, vd, heads=self.heads, dim_head=self.dim_head,
                                            scale=self.scale, nmask=nmask, k_idx=(None if k_emb is not None and degree == '0' else k_idx),
                                            kv_heads=1 if self.one_headed else self.heads, **kw)
        return outputs


class SinusoidalEmbeddings(nn.Module):
    """reference rotary.py:5-13"""

    def __init__(self, dim):
        super().__init__()
        self.register_buffer('inv_freq', 1. / (10000 ** (torch.arange(0, dim, 2).float() / dim)))

    def forward(self, t):
        freqs = t[..., None].float() * self.inv_freq
        return freqs.repeat_interleave(2, dim=-1)                      # '... d -> ... (d r)', r = 2


def rotate_half(x):
    """reference rotary.py:15-18 on [..., d, m]: pairs (x1, x2) of consecutive channels -> cat(-x2, x1) along d (NOT re-interleaved)."""
    return torch.cat((-x[..., 1::2, :], x[..., 0::2, :]), dim=-2)


def apply_rotary_pos_emb(t, freqs):
    """reference rotary.py:20-24: t [..., d, m], freqs [..., rot, 1] (rot <= d leading channels are rotated)."""
    rot = freqs.shape[-2]
    tr, tp = t[..., :rot, :], t[..., rot:, :]
    return torch.cat((tr * freqs.cos() + rotate_half(tr) * freqs.sin(), tp), dim=-2)


class OneHeadedKVAttentionSE3(AttentionSE3):
    def __init__(self, fiber, **kwargs):
        super().__init__(fiber, one_headed=True, **kwargs)


class AttentionBlockSE3(nn.Module):
    """reference S:656-683"""

    def __init__(self, fiber, dim_head=24, heads=8, attend_self=False, edge_dim=None, use_null_kv=False, fourier_encode_dist=False,
                 rel_dist_num_fourier_features=4, splits=4, global_feats_dim=False, linear_proj_keys=False, tie_key_values=False,
                 attention_klass=AttentionSE3, norm_gated_scale=False):
        super().__init__()
        self.attn = attention_klass(fiber, heads=heads, dim_head=dim_head, attend_self=attend_self, edge_dim=edge_dim,
                                    use_null_kv=use_null_kv, rel_dist_num_fourier_features=rel_dist_num_fourier_features,
                                    fourier_encode_dist=fourier_encode_dist, splits=splits, global_feats_dim=global_feats_dim,
                                    linear_proj_keys=linear_proj_keys, tie_key_values=tie_key_values)
        self.prenorm = NormSE3(fiber, gated_scale=norm_gated_scale)

    def forward(self, features, edge_info, rel_dist, basis, global_feats=None, pos_emb=None, mask=None):
        return self.attn(self.prenorm(features), edge_info, rel_dist, basis, global_feats, pos_emb, mask, residual=features)


class SequentialSequence(nn.Module):
    """reference reversible.py:189-198"""

    def __init__(self, blocks):
        super().__init__()
        self.blocks = blocks

    def forward(self, x, **kwargs):
        for attn, ff in self.blocks:
            x = attn(x, **kwargs)
            x = ff(x)
        return x


def masked_mean_nodes(t, mask):
    """reference utils.py:72-80 over the node axis (return_pooled, S:1365-1367)."""
    m = mask[(..., *((None,) * (t.dim() - mask.dim())))]
    tot = mask.sum(dim=1)
    tot = tot[(..., *((None,) * (t.dim() - 1 - tot.dim())))]
    mean = t.masked_fill(~m, 0.).sum(dim=1) / tot.clamp(min=1.)
    return mean.masked_fill(tot == 0, 0.)


class SE3Transformer(nn.Module):
    """Drop-in for se3_transformer_pytorch.SE3Transformer (reference S:936-1375), inference on H100.

    Not carried over (raise NotImplementedError): reversible, use_egnn -- they are outside the hot path named by BASELINE.json
    (SURVEY.md section 2, "OUT OF SCOPE")."""

    def __init__(self, *, dim, heads=8, dim_head=24, depth=2, input_degrees=1, num_degrees=None, output_degrees=1,
                 valid_radius=1e5, reduce_dim_out=False, num_tokens=None, num_positions=None, num_edge_tokens=None, edge_dim=None,
                 reversible=False, attend_self=True, use_null_kv=False, differentiable_coors=False, fourier_encode_dist=False,
                 rel_dist_num_fourier_features=4, num_neighbors=float('inf'), attend_sparse_neighbors=False, num_adj_degrees=None,
                 adj_dim=0, max_sparse_neighbors=float('inf'), dim_in=None, dim_out=None, norm_out=False, num_conv_layers=0,
                 causal=False, splits=4, global_feats_dim=None, linear_proj_keys=False, one_headed_key_values=False,
                 tie_key_values=False, rotary_position=False, rotary_rel_dist=False, norm_gated_scale=False, use_egnn=False,
                 egnn_hidden_dim=32, egnn_weights_clamp_value=None, egnn_feedforward=False, hidden_fiber_dict=None,
                 out_fiber_dict=None):
        super().__init__()
        for flag, name in ((reversible, 'reversible'), (use_egnn, 'use_egnn')):
            if flag:
                raise NotImplementedError(f'{name}=True is outside the H100 hot path of this package')
        if differentiable_coors:
            raise NotImplementedError('differentiable_coors=True needs the backward pass; this package is forward only (SURVEY.md 8f row 4)')
        dim_in = default(dim_in, dim)
        self.dim_in = dim_in if isinstance(dim_in, tuple) else (dim_in,) * input_degrees
        self.dim = dim
        self.token_emb = nn.Embedding(num_tokens, dim) if exists(num_tokens) else None
        self.rotary_rel_dist, self.rotary_position = rotary_rel_dist, rotary_position      # reference S:998-1004
        self.rotary_pos_emb = None
        if rotary_position or rotary_rel_dist:
            self.rotary_pos_emb = SinusoidalEmbeddings(dim_head // (int(rotary_position) + int(rotary_rel_dist)))
        self.num_positions = num_positions
        self.pos_emb = nn.Embedding(num_positions, dim) if exists(num_positions) else None
        assert not (exists(num_edge_tokens) and not exists(edge_dim)), 'edge dimension (edge_dim) must be supplied if SE3 transformer is to have edge tokens'
        self.edge_emb = nn.Embedding(num_edge_tokens, edge_dim) if exists(num_edge_tokens) else None
        self.has_edges = exists(edge_dim) and edge_dim > 0
        self.input_degrees = input_degrees
        assert not (exists(num_adj_degrees) and num_adj_degrees < 1), 'make sure adjacent degrees is greater than 1'
        assert exists(num_degrees) or exists(hidden_fiber_dict), 'either num_degrees or hidden_fiber_dict must be specified'
        self.num_degrees = num_degrees if exists(num_degrees) else (max(hidden_fiber_dict.keys()) + 1)
        self.output_degrees = output_degrees
        self.differentiable_coors = differentiable_coors
        self.valid_radius = valid_radius
        self.num_neighbors = num_neighbors
        self.attend_sparse_neighbors = attend_sparse_neighbors
        self.max_sparse_neighbors = max_sparse_neighbors
        self.num_adj_degrees = num_adj_degrees
        self.adj_emb = nn.Embedding(num_adj_degrees + 1, adj_dim) if exists(num_adj_degrees) and adj_dim > 0 else None
        edge_dim = (edge_dim if self.has_edges else 0) + (adj_dim if exists(self.adj_emb) else 0)
        dim_out = default(dim_out, dim)
        fiber_in = Fiber.create(input_degrees, dim_in)
        fiber_hidden = Fiber(hidden_fiber_dict) if exists(hidden_fiber_dict) else Fiber.create(num_degrees, dim)
        if exists(out_fiber_dict):
            fiber_out = Fiber(out_fiber_dict)
            self.output_degrees = max(out_fiber_dict.keys()) + 1
        elif exists(output_degrees):
            fiber_out = Fiber.create(output_degrees, dim_out)
        else:
            fiber_out = None
        conv_kwargs = dict(edge_dim=edge_dim, fourier_encode_dist=fourier_encode_dist, num_fourier_features=rel_dist_num_fourier_features,
                           splits=splits)
        assert not (causal and not attend_self), 'attending to self must be turned on if in autoregressive mode (for the first token)'
        self.causal = causal
        self.conv_in = ConvSE3(fiber_in, fiber_hidden, **conv_kwargs)
        self.convs = nn.ModuleList([])
        for _ in range(num_conv_layers):
            self.convs.append(nn.ModuleList([ConvSE3(fiber_hidden, fiber_hidden, **conv_kwargs),
                                             NormSE3(fiber_hidden, gated_scale=norm_gated_scale)]))
        self.accept_global_feats = exists(global_feats_dim)
        self.attend_self = attend_self
        klass = OneHeadedKVAttentionSE3 if one_headed_key_values else AttentionSE3
        layers = nn.ModuleList([])
        for _ in range(depth):
            layers.append(nn.ModuleList([
                AttentionBlockSE3(fiber_hidden, heads=heads, dim_head=dim_head, attend_self=attend_self, edge_dim=edge_dim,
                                  fourier_encode_dist=fourier_encode_dist, rel_dist_num_fourier_features=rel_dist_num_fourier_features,
                                  use_null_kv=use_null_kv, splits=splits, global_feats_dim=global_feats_dim,
                                  linear_proj_keys=linear_proj_keys, attention_klass=klass, tie_key_values=tie_key_values,
                                  norm_gated_scale=norm_gated_scale),
                FeedForwardBlockSE3(fiber_hidden, norm_gated_scale=norm_gated_scale)]))
        self.net = SequentialSequence(layers)
        self.conv_out = ConvSE3(fiber_hidden, fiber_out, **conv_kwargs) if exists(fiber_out) else None
        self.norm = NormSE3(fiber_out, gated_scale=norm_gated_scale, nonlin=nn.Identity()) if norm_out and exists(fiber_out) else nn.Identity()
        final_fiber = default(fiber_out, fiber_hidden)
        self.linear_out = LinearSE3(final_fiber, Fiber([(d, 1) for d, _ in final_fiber])) if reduce_dim_out else None

    # ---- weights ----------------------------------------------------------------------------------------
    def conv_modules(self):
        return [m for m in self.modules() if isinstance(m, ConvSE3)]

    def pack_weights(self, free_master=False, max_distance=None):
        """Pre-build the tensor-core weight images of every ConvSE3 (otherwise done lazily on the first forward); see
        ConvSE3.pack_weights."""
        for m in self.conv_modules():
            m.pack_weights(free_master=free_master, max_distance=max_distance)
        return self

    def graphed(self, feats, coors, mask=None, **fwd_kwargs):
        """Capture one forward for these (static) input shapes in a CUDA graph and return a replayable callable
        (see GraphedForward).  Small point clouds are launch bound (~100 kernels of a few microseconds each); replaying a
        graph removes the per-launch host cost.  Not available with attend_sparse_neighbors / neighbor_mask (their
        host-side `.item()` synchronisations, reference S:1208, 1253, cannot be captured), nor with sparse pair inputs."""
        if any(_is_sparse(v) for v in fwd_kwargs.values()):
            raise ValueError('graphed: sparse pair inputs are not supported (their number of entries is not static); pass dense '
                             'tensors or call forward')
        return GraphedForward(self, feats, coors, mask, **fwd_kwargs)

    def causal_decoder(self, batch_size=1):
        """An empty CausalDecoder of this causal model for batch_size clouds: generation one node (or a few) at a time, each step
        doing the edge work of its new nodes only."""
        return CausalDecoder(self, batch_size)

    def packed_decoder(self, page_size=None, max_nodes=None, prefix_cache=False):
        """An empty PackedCausalDecoder of this causal model: clouds of different lengths decoded together, each opened, extended,
        truncated, forked and closed on its own, every step carrying the new nodes of any subset of them.  With an integer
        page_size >= 1, a PagedCausalDecoder instead, the same decoder with its cache in pages of page_size nodes: memory follows
        the nodes decoded and forks share their prefix; max_nodes (pages for that many nodes, reserved at the first step) caps
        its pool, which otherwise doubles when full.  prefix_cache=True (paged only) shares the full pages of equal prompts
        between clouds opened separately (DESIGN.md 10.4)."""
        if not isinstance(prefix_cache, bool):
            raise ValueError(f'packed_decoder: prefix_cache must be a bool, got {prefix_cache!r}')
        if page_size is None:
            if max_nodes is not None:
                raise ValueError('packed_decoder: max_nodes caps the pages of a paged cache; give a page_size too')
            if prefix_cache:
                raise ValueError('packed_decoder: the prefix cache shares pages of a paged cache; give a page_size too')
            return PackedCausalDecoder(self)
        return PagedCausalDecoder(self, page_size, max_nodes, prefix_cache)

    # ---- forward ----------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, feats, coors, mask=None, adj_mat=None, edges=None, return_type=None, return_pooled=False,
                neighbor_mask=None, global_feats=None):
        """adj_mat, edges and neighbor_mask may each also be a torch.sparse_coo tensor (see _check_sparse_pairs); the result is
        then bit-identical to the same call with its to_dense(), and no intermediate is [n, n]."""
        self._check_sparse_pairs(coors, adj_mat, edges, neighbor_mask)
        kw = dict(mask=mask, adj_mat=adj_mat, edges=edges, return_type=return_type, return_pooled=return_pooled,
                  neighbor_mask=neighbor_mask, global_feats=global_feats)
        return self._checked(lambda: self._forward_once(feats, coors, **kw))

    @torch.no_grad()
    def forward_packed(self, feats, coors, seqlens, adj_mat=None, edges=None, neighbor_mask=None, return_type=None,
                       return_pooled=False):
        """Clouds of different sizes in one forward, concatenated along the node axis instead of padded (no reference
        counterpart; DESIGN.md section 7).  For every cloud c this returns what forward() returns for that cloud alone (batch 1,
        no mask, its own pair inputs), concatenated along the node axis: each cloud keeps its own neighbour count
        k_c = min(min(num_neighbors, n_c - 1) + min(max_sparse_neighbors, bonded_c), n_c - 1), and positions, rotary positions
        and causal order count from the cloud's first node.  No edge of one cloud reaches another, and none is spent on padding.

        feats: [T, dim_in] float, [T] long tokens (num_tokens) or {'d': [T, C_d, 2d+1]}; coors [T, 3];
        seqlens: B node counts summing to T (1-D int tensor or sequence of ints), each in [2, 4097].
        adj_mat, neighbor_mask: lists of B bool [n_c, n_c]; edges: list of B [n_c, n_c] long tokens or [n_c, n_c, edge_dim] float.
        Returns {'d': [T, C, 2d+1]} ('0': [T, C]; reduce_dim_out drops C), or one of them with return_type; return_pooled gives
        the per-cloud mean over nodes, [B, ...].  Models built with global_feats_dim are not supported."""
        seqlens = self._check_packed(feats, coors, seqlens, adj_mat, edges, neighbor_mask)
        return self._checked(lambda: self._forward_packed_once(feats, coors, seqlens, adj_mat, edges, neighbor_mask, return_type,
                                                               return_pooled))

    def _checked(self, once):
        """Run one forward (once() -> (out, deferred low-rank checks)) and the run-time check of its low-rank plans; on a plan
        miss the affected ConvSE3 move to the direct kernels and the forward runs again."""
        out, checks = once()
        if torch.cuda.is_current_stream_capturing():
            self._graph_checks = checks               # static tensors of the graph: GraphedForward reads them after each replay
            return out
        bad = check_lowrank_stats(checks)             # the one host synchronisation of the low-rank plans, once per forward
        if bad:
            self.handle_plan_miss(bad)
            out, checks = once()
            assert not check_lowrank_stats(checks)
        return out

    @staticmethod
    def handle_plan_miss(bad):
        """The radial trunk outputs of a forward left the cached low-rank subspace of these ConvSE3 (distances beyond the plan's
        range): with released masters there is nothing to fall back to; otherwise they run on the direct kernels from now on."""
        if any(conv.free_master for conv in bad):
            raise LowRankPlanMiss('low-rank radial plan does not cover this input; pack_weights(max_distance=...) was given too small a distance')
        import warnings
        warnings.warn(f'{len(bad)} ConvSE3 left their low-rank radial plan (residual above {ConvSE3.LR_RUNTIME_TOL:g}): evaluating them with '
                      'the direct K = 128 kernels')
        for conv in bad:
            conv._lr_blocked = True

    def _forward_once(self, feats, coors, mask=None, adj_mat=None, edges=None, return_type=None, return_pooled=False,
                      neighbor_mask=None, global_feats=None):
        assert not (self.accept_global_feats ^ exists(global_feats)), 'you cannot pass in global features unless you init the class correctly'
        _mask = mask
        out_dtype = self._compute_dtype(coors)
        if self.output_degrees == 1:
            return_type = 0
        feats = self._embed_tokens(feats)
        assert not (self.attend_sparse_neighbors and not exists(adj_mat)), 'adjacency matrix (adjacency_mat) or edges (edges) must be passed in'
        assert not (self.has_edges and not exists(edges)), 'edge embedding (num_edge_tokens & edge_dim) must be supplied if one were to train on edge types'
        if torch.is_tensor(feats):
            feats = {'0': feats[..., None]}
        if torch.is_tensor(global_feats):
            global_feats = {'0': global_feats[..., None]}
        if exists(global_feats):
            global_feats = {k: v.float() for k, v in global_feats.items()}
        if exists(edges) and edges.is_floating_point() and not edges.is_sparse:      # sparse: after coalescing, as to_dense()
            edges = edges.float()
        b, n = feats['0'].shape[:2]
        device = feats['0'].device
        feats = self._check_features(feats, coors)
        valid_radius = self._valid_radius()
        if exists(edges) and exists(self.edge_emb) and edges.dim() == 2:   # [b, n] tokens: the reference broadcasts them over rows
            assert b == 1, 'edges of shape [b, n] only broadcast for batch size 1 (as in the reference)'
            edges = edges.unsqueeze(1).expand(b, n, n)
        graph = self._sparse_graph if any(_is_sparse(t) for t in (adj_mat, edges, neighbor_mask)) else self._dense_graph
        idx, nmask, rel_pos, rel_dist, e = graph(coors, mask, adj_mat, edges, neighbor_mask, b, n, valid_radius)

        pos_emb = None
        if exists(self.rotary_pos_emb):
            pos = torch.arange(n, device=device)
            pos_emb = self._rotary(pos.view(1, n).expand(b, n), torch.cat((pos.view(1, n, 1).expand(b, n, 1), idx), dim=2), n, rel_dist)
        pool = None
        if return_pooled:
            pool = lambda v: masked_mean_nodes(v, _mask) if exists(_mask) else v.mean(dim=1)
        return self._trunk(feats, (idx, nmask, e), rel_pos, rel_dist, pos_emb, global_feats, _mask, pool, out_dtype, return_type)

    # ---- pieces shared by forward and forward_packed -------------------------------------------------------
    def _compute_dtype(self, coors):
        """float64 models / inputs (reference tests/test_equivariance.py:228-258 runs under a float64 default dtype): the kernels
        compute in float32; parameters are converted once, inputs are cast, results are returned in the caller's dtype."""
        if any(p.dtype == torch.float64 for p in self.parameters()):
            import warnings
            warnings.warn('se3_transformer_pytorch_b200 computes in float32: converting the float64 parameters of this model to float32')
            self.float()
        return coors.dtype if coors.dtype == torch.float64 else None

    def _embed_tokens(self, feats, positions=None):
        """Token and absolute-position embeddings (reference S:1149-1160) of feats [b, n, ...]; positions [n] (default 0 .. n-1)."""
        if exists(self.token_emb):
            feats = self.token_emb(feats)
        if exists(self.pos_emb):
            if positions is None:
                assert feats.shape[1] <= self.num_positions, 'feature sequence length must be less than the number of positions given at init'
                positions = torch.arange(feats.shape[1], device=feats.device)
            feats = feats + self.pos_emb(positions).unsqueeze(0)
        return feats

    def _check_features(self, feats, coors):
        if not coors.is_cuda:
            raise RuntimeError('se3_transformer_pytorch_b200 runs on CUDA (sm_90a) only; move the model and inputs to the GPU')
        d = feats['0'].shape[2]
        assert d == self.dim_in[0], f'feature dimension {d} must be equal to dimension given at init {self.dim_in[0]}'
        assert set(map(int, feats.keys())) == set(range(self.input_degrees)), f'input must have {self.input_degrees} degree'
        return {k: v.float().contiguous() for k, v in feats.items()}

    def _bonded(self, adj_mat, b, n, device):
        """N-hop adjacency (reference S:1177-1191) and the bonded neighbours (S:1198-1217) of clouds of n nodes: returns
        (adj_indices [b, n, n] hop counts or None, sparse_mask [b, n, n] or None, num_sparse)."""
        max_sparse = self.max_sparse_neighbors
        adj_indices = None
        if exists(self.num_adj_degrees):                       # N-hop adjacency, reference S:1177-1191
            if adj_mat.dim() == 2:
                adj_mat = adj_mat.unsqueeze(0).expand(b, -1, -1).clone()
            adj_indices = adj_mat.clone().long()
            for ind in range(self.num_adj_degrees - 1):
                degree = ind + 2
                nxt = (adj_mat.float() @ adj_mat.float()) > 0
                nxt_mask = (nxt.float() - adj_mat.float()).bool()
                adj_indices = adj_indices.masked_fill(nxt_mask, degree)
                adj_mat = nxt.clone()

        sparse_mask = None
        num_sparse = 0
        if self.attend_sparse_neighbors:                       # reference S:1198-1217
            assert exists(adj_mat), 'adjacency matrix must be passed in (keyword argument adj_mat)'
            if adj_mat.dim() == 2:
                adj_mat = adj_mat.unsqueeze(0).expand(b, -1, -1)
            eye = torch.eye(n, dtype=torch.bool, device=device)
            adj_vals = adj_mat.float().masked_fill(eye.unsqueeze(0), 0.)
            adj_max = int(adj_vals.sum(dim=-1).max().item())
            if max_sparse < adj_max:
                adj_vals = adj_vals + torch.empty_like(adj_vals).uniform_(-0.01, 0.01).masked_fill(eye.unsqueeze(0), 0.)
                adj_vals = adj_vals.masked_fill(eye.unsqueeze(0), -1.)
            num_sparse = int(min(max_sparse, adj_max))
            if num_sparse > 0:
                vals, inds = adj_vals.topk(num_sparse, dim=-1)
                sparse_mask = torch.zeros_like(adj_vals).scatter_(-1, inds, vals) > 0.5
            else:
                sparse_mask = torch.zeros_like(adj_vals, dtype=torch.bool)

        return adj_indices, sparse_mask, num_sparse

    def _valid_radius(self):
        """The search radius: none at all when only bonded neighbours are attended to (num_neighbors == 0)."""
        assert self.attend_sparse_neighbors or self.num_neighbors > 0, 'you must either attend to sparsely bonded neighbors, or set number of locally attended neighbors to be greater than 0'
        return 0 if self.num_neighbors == 0 else self.valid_radius

    def _num_neighbors(self, n, num_sparse):
        """Neighbour slots per node: the local neighbours plus the bonded ones, at most n - 1 (reference S:1220-1226)."""
        total = int(int(min(self.num_neighbors, n - 1)) + num_sparse)
        assert total > 0, 'you must be fetching at least 1 neighbor'
        return int(min(total, n - 1))

    def _edge_features(self, edge_values, hop_values):
        """Edge features on the neighbour list (reference S:1231-1239, 1293-1294) from the pair values each graph builder looked
        up on it: edge tokens embedded or continuous edges as float, then the embedded hop counts concatenated; None if neither."""
        e = None
        if edge_values is not None:
            e = self.edge_emb(edge_values) if exists(self.edge_emb) else edge_values.float()
        if hop_values is not None:
            a = self.adj_emb(hop_values)
            e = torch.cat((e, a), dim=-1) if exists(e) else a
        return e

    def _dense_graph(self, coors, mask, adj_mat, edges, neighbor_mask, b, n, valid_radius):
        """The neighbour graph and edge features of _forward_once with dense pair inputs: the search reads the byte masks, and
        edge values and hop counts are gathered on the neighbour list (gather first, embed after).  Returns idx, nmask,
        rel_pos, rel_dist, e."""
        adj_indices, sparse_mask, num_sparse = self._bonded(adj_mat, b, n, coors.device)
        if exists(neighbor_mask):
            eye = torch.eye(n, dtype=torch.bool, device=neighbor_mask.device)
            self._report_neighbor_mask(neighbor_mask.masked_fill(eye.unsqueeze(0), False).sum(dim=-1))
        idx, nmask, rel_pos, rel_dist = ops.knn(coors.float(), self._num_neighbors(n, num_sparse), valid_radius, node_mask=mask,
                                                neighbor_mask=neighbor_mask, sparse_adj=sparse_mask, causal=self.causal)
        edge_values = None
        if exists(edges):
            edge_values = edges.gather(2, idx) if exists(self.edge_emb) else ops.gather_pairs(edges.float(), idx)
        hops = adj_indices.gather(2, idx) if exists(self.adj_emb) else None
        return idx, nmask, rel_pos, rel_dist, self._edge_features(edge_values, hops)

    # ---- sparse pair inputs --------------------------------------------------------------------------------
    def _check_sparse_pairs(self, coors, adj_mat, edges, neighbor_mask):
        """The sparse pair inputs forward takes, checked before any device work (missing entries mean: not bonded, not
        allowed, token 0 / a zero feature vector):
          adj_mat        torch.sparse_coo [n, n] (shared by the batch) or [b, n, n], any real dtype;
          neighbor_mask  torch.sparse_coo [n, n], [1, n, n] or [b, n, n], any real dtype;
          edges          torch.sparse_coo [b, n, n] integer tokens (num_edge_tokens), or [b, n, n, edge_dim] with 3 sparse
                         dims and 1 dense dim (continuous edges)."""
        named = (('adj_mat', adj_mat), ('edges', edges), ('neighbor_mask', neighbor_mask))
        if not any(_is_sparse(t) for _, t in named):
            return
        if not torch.is_tensor(coors) or coors.dim() != 3:
            raise ValueError(f'coors must be [b, n, 3], got {tuple(coors.shape) if torch.is_tensor(coors) else type(coors).__name__}')
        b, n = coors.shape[:2]
        for name, t in named:
            if not _is_sparse(t):
                continue
            if t.layout != torch.sparse_coo:
                raise ValueError(f'{name}: the sparse layout {t.layout} is not supported; pass a torch.sparse_coo tensor '
                                 f'({name}.to_sparse_coo())')
            if t.dtype.is_complex:
                raise ValueError(f'{name}: complex values are not supported, got {t.dtype}')
            shape = tuple(t.shape)
            if name == 'edges':
                if t.dim() == 2:
                    raise ValueError('edges: a 2-D sparse tensor is not accepted (it would be ambiguous with the [b, n] token '
                                     f'form); pass [b, n, n] = {(b, n, n)}')
                if exists(self.edge_emb):
                    if shape != (b, n, n) or t.dense_dim() != 0:
                        raise ValueError(f'edges: sparse edge tokens must be [b, n, n] = {(b, n, n)} with no dense dims, got '
                                         f'{shape} with {t.dense_dim()} dense dims')
                    if t.dtype.is_floating_point or t.dtype == torch.bool:
                        raise ValueError(f'edges: sparse edge tokens must have an integer dtype, got {t.dtype}')
                elif t.dim() != 4 or shape[:3] != (b, n, n) or t.sparse_dim() != 3:
                    raise ValueError(f'edges: sparse continuous edges must be [b, n, n, edge_dim] with b, n = {(b, n)}, 3 sparse '
                                     f'dims and 1 dense dim, got {shape} with {t.sparse_dim()} sparse dims')
                continue
            allowed = [(n, n), (b, n, n)] + ([(1, n, n)] if name == 'neighbor_mask' else [])
            if shape not in allowed or t.dense_dim() != 0:
                raise ValueError(f'{name}: a sparse {name} must be one of {sorted(set(allowed))} with no dense dims, got {shape} '
                                 f'with {t.dense_dim()} dense dims')

    def _bonded_sparse(self, adj_mat, b, n):
        """_bonded for a torch.sparse_coo adj_mat ([n, n] or [b, n, n]) in O(nnz) memory, on the block-diagonal [R, R] matrix
        of its clouds (R = n for a shared [n, n]).  Returns (hop counts as PairRows or None, bonded neighbours as PairRows or
        None, num_sparse): the densified PairRows equal _bonded's adj_indices and sparse_mask, except that a random
        sub-sample (max_sparse_neighbors below a row's bonded count) has the same distribution, not the same draw."""
        a = ops.coo_to_rows(adj_mat, n)
        R = a.ptr.numel() - 1
        rows = torch.repeat_interleave(torch.arange(R, device=a.ptr.device), a.ptr.diff())
        cols = a.cols.long() + (rows // n) * n                                             # global column of the block
        keys, vals = rows * R + cols, a.values.float()                                     # M_1 = A, sorted by key
        hop_keys = hop_vals = None
        if exists(self.num_adj_degrees):
            hop_keys, hop_vals = keys, a.values.long()
            for degree in range(2, self.num_adj_degrees + 1):
                m = torch.sparse_coo_tensor(torch.stack((keys // R, keys % R)), vals, (R, R), is_coalesced=True)
                sq = torch.sparse.mm(m, m).coalesce()
                nxt = sq.indices()[:, sq.values() > 0]
                nxt_keys = nxt[0] * R + nxt[1]                                            # M_d = (M_{d-1} @ M_{d-1}) > 0
                # the reference's XOR: pairs where M_d (1 or absent) differs from M_{d-1} (its value or absent) take this degree
                pos = torch.searchsorted(keys, nxt_keys).clamp(max=max(keys.numel() - 1, 0))
                prev = torch.where(keys[pos] == nxt_keys, vals[pos], 0.) if keys.numel() else torch.zeros_like(nxt_keys, dtype=torch.float)
                flip = torch.cat((nxt_keys[prev != 1.], keys[(vals != 0.) & ~torch.isin(keys, nxt_keys)]))
                keep = ~torch.isin(hop_keys, flip)
                hop_keys, order = torch.cat((hop_keys[keep], flip)).sort()
                hop_vals = torch.cat((hop_vals[keep], torch.full_like(flip, degree)))[order]
                keys, vals = nxt_keys, torch.ones(nxt_keys.numel(), device=keys.device)
        hops = None
        if hop_keys is not None:
            hop_rows = hop_keys // R
            hops = ops.pair_rows(hop_rows, hop_keys % R - (hop_rows // n) * n, hop_vals, R, R == n)

        bonded, num_sparse = None, 0
        if self.attend_sparse_neighbors:                       # reference S:1198-1217 on the entries of M_D
            rows, cols = keys // R, keys % R
            off = rows != cols
            rows, cols, vals = rows[off], cols[off], vals[off]
            row_sums = torch.zeros(R, device=vals.device).index_add_(0, rows, vals)
            adj_max = int(row_sums.max().item())
            subsample = self.max_sparse_neighbors < adj_max
            num_sparse = int(min(self.max_sparse_neighbors, adj_max))
            if subsample and R == n and b > 1:                 # every cloud draws its own subset of the shared adjacency
                shift = (torch.arange(b, device=rows.device) * n).repeat_interleave(rows.numel())
                rows, cols, vals = rows.repeat(b) + shift, cols.repeat(b) + shift, vals.repeat(b)
                R = b * n
            score = vals + torch.empty_like(vals).uniform_(-0.01, 0.01) if subsample else vals
            # the top num_sparse scores of every row (ties: lower column first), of which those above 0.5 are bonded
            order = torch.argsort(-score, stable=True)
            order = order[torch.argsort(rows[order], stable=True)]
            ptr = ops.pair_rows(rows, cols, vals, R, False).ptr
            rank = torch.arange(order.numel(), device=rows.device) - ptr[rows[order]]
            pick = order[(rank < num_sparse) & (score[order] > 0.5)].sort().values
            brows = rows[pick]
            bonded = ops.pair_rows(brows, cols[pick] - (brows // n) * n, torch.ones_like(brows, dtype=torch.bool), R, R == n)
        return hops, bonded, num_sparse

    def _sparse_graph(self, coors, mask, adj_mat, edges, neighbor_mask, b, n, valid_radius):
        """The neighbour graph and edge features of _forward_once when at least one pair input is torch.sparse_coo (the dense
        ones are converted): the search reads sorted column lists (ops.PairRows), and edge tokens, edge features and hop counts
        are looked up in them (ops.pair_lookup).  Memory is O(nnz + n k).  Returns idx, nmask, rel_pos, rel_dist, e."""
        hops, bonded, num_sparse = None, None, 0
        if exists(self.num_adj_degrees) or self.attend_sparse_neighbors:
            assert exists(adj_mat), 'adjacency matrix must be passed in (keyword argument adj_mat)'
            hops, bonded, num_sparse = self._bonded_sparse(adj_mat if adj_mat.is_sparse else adj_mat.to_sparse(), b, n)
        total = self._num_neighbors(n, num_sparse)
        nbr = None
        if exists(neighbor_mask):
            nbr = ops.coo_to_rows(neighbor_mask if neighbor_mask.is_sparse else neighbor_mask.to_sparse(), n)
            rows = torch.repeat_interleave(torch.arange(nbr.ptr.numel() - 1, device=nbr.ptr.device), nbr.ptr.diff())
            v = nbr.values
            off, dt = nbr.cols.long() != rows % n, v.sum().dtype                           # dt: the dtype of the dense row sums
            self._report_neighbor_mask(torch.zeros(nbr.ptr.numel() - 1, dtype=dt, device=v.device).index_add_(0, rows[off], v[off].to(dt)))
            allowed = v if v.dtype == torch.bool else v.to(torch.uint8) != 0              # the byte the dense search reads
            nbr = ops.pair_rows(rows[allowed], nbr.cols[allowed], v[allowed], nbr.ptr.numel() - 1, nbr.shared)
        idx, nmask, rel_pos, rel_dist = ops.knn(coors.float(), total, valid_radius, node_mask=mask, neighbor_mask=nbr,
                                                sparse_adj=bonded, causal=self.causal)

        def lookup(rows):
            """rows.values on the neighbour list, zero where a pair is absent"""
            v = rows.values
            return torch.cat((v, v.new_zeros((1, *v.shape[1:]))))[ops.pair_lookup(rows, idx)]

        edge_values = lookup(ops.coo_to_rows(edges if edges.is_sparse else edges.to_sparse(3), n)) if exists(edges) else None
        hop_values = lookup(hops) if exists(self.adj_emb) else None
        return idx, nmask, rel_pos, rel_dist, self._edge_features(edge_values, hop_values)

    def _report_neighbor_mask(self, row_counts):
        """Reference S:1253: row_counts [...] are the row sums of neighbor_mask without its diagonal."""
        max_nb = int(row_counts.max().item())
        if max_nb > self.num_neighbors:
            print(f'neighbor_mask shows maximum number of neighbors as {max_nb} but specified number of neighbors is {self.num_neighbors}')

    def _rotary(self, q_pos, k_pos, n_pos, rel_dist):
        """Rotary embeddings of the type-0 queries and keys (reference S:1298-1325): q_pos [b, n] and k_pos [b, n, 1 + k] (self
        first) are node positions inside their cloud, all below n_pos; rel_dist [b, n, k]."""
        q_parts, k_parts = [], []
        if self.rotary_position:
            seq_emb = self.rotary_pos_emb(torch.arange(n_pos, device=q_pos.device))                # [n_pos, d]
            k_parts.append(seq_emb[k_pos])                                                          # [b, n, 1 + k, d]
            q_parts.append(seq_emb[q_pos])
        if self.rotary_rel_dist:
            k_parts.append(self.rotary_pos_emb(F.pad(rel_dist, (1, 0), value=0.) * 1e2))
            q_parts.append(self.rotary_pos_emb(torch.zeros(q_pos.shape, device=q_pos.device)))
        return torch.cat(q_parts, dim=-1), torch.cat(k_parts, dim=-1)

    def _trunk(self, feats, edge_info, rel_pos, rel_dist, pos_emb, global_feats, mask, reduce, out_dtype, return_type):
        """Everything after the graph (reference S:1240-1375): conv_in, pre-convs, attention blocks, conv_out, norm, linear_out
        and the output format.  reduce (or None) maps every output [b, n, ...] to what is returned (pooling, unbatching).
        Returns (output, the deferred run-time checks of the low-rank plans)."""
        # every ConvSE3 and attention block runs its edge work over node chunks under the edge budget (DESIGN.md 4.7); the flat
        # basis is built by the Geometry of a chunk (or of the whole graph) only when an R-first convolution reads it
        geom = Geometry(rel_pos, self.num_degrees - 1, deferred=[], edge_budget=edge_budget_bytes(switches.current(), rel_pos.device))
        basis = (None, None, geom)
        x = self.conv_in(feats, edge_info, rel_dist=rel_dist, basis=basis)
        for conv, nonlin in self.convs:
            x = nonlin(x)
            x = conv(x, edge_info, rel_dist=rel_dist, basis=basis)
        x = self.net(x, edge_info=edge_info, rel_dist=rel_dist, basis=basis, global_feats=global_feats, pos_emb=pos_emb, mask=mask)
        if exists(self.conv_out):
            x = self.conv_out(x, edge_info, rel_dist=rel_dist, basis=basis)
        return self._output(x, reduce, out_dtype, return_type), geom.deferred

    def _output(self, x, reduce, out_dtype, return_type):
        """The output format after conv_out: norm, linear_out, reduce (or None), type-0 squeeze, dtype and return_type."""
        x = self.norm(x)
        if exists(self.linear_out):
            x = self.linear_out(x)
            x = {k: v.squeeze(dim=2) for k, v in x.items()}
        if exists(reduce):
            x = {k: reduce(v) for k, v in x.items()}
        if '0' in x:
            x['0'] = x['0'].squeeze(dim=-1)
        if exists(out_dtype):
            x = {k: v.to(out_dtype) for k, v in x.items()}
        if exists(return_type):
            return x[str(return_type)]
        return x

    # ---- packed batches ------------------------------------------------------------------------------------
    def _check_packed(self, feats, coors, seqlens, adj_mat, edges, neighbor_mask):
        """Everything forward_packed takes from the caller, checked before any device work; returns seqlens as a list of ints."""
        if self.accept_global_feats:
            raise NotImplementedError('forward_packed: models built with global_feats_dim are not supported (the attention kernel '
                                      'indexes the global keys by batch row, and a packed batch is one row)')
        if torch.is_tensor(seqlens):
            if seqlens.dim() != 1 or seqlens.is_floating_point() or seqlens.is_complex() or seqlens.dtype == torch.bool:
                raise ValueError(f'forward_packed: seqlens must be a 1-D integer tensor, got {seqlens.dtype} of shape {tuple(seqlens.shape)}')
            seqlens = seqlens.tolist()
        try:
            seqlens = [operator.index(n) for n in seqlens]
        except TypeError:
            raise ValueError('forward_packed: seqlens must be a 1-D integer tensor or a sequence of ints') from None
        if not seqlens:
            raise ValueError('forward_packed: seqlens is empty')
        B, T = len(seqlens), sum(seqlens)
        for t in (feats.values() if isinstance(feats, dict) else [feats]):
            if not torch.is_tensor(t) or t.dim() < 1 or t.shape[0] != T:
                raise ValueError(f'forward_packed: the features must have sum(seqlens) = {T} rows, got '
                                 f'{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
        if not torch.is_tensor(coors) or tuple(coors.shape) != (T, 3):
            raise ValueError(f'forward_packed: coors must be [sum(seqlens), 3] = {(T, 3)}, got '
                             f'{tuple(coors.shape) if torch.is_tensor(coors) else type(coors).__name__}')
        bad = [n for n in seqlens if not 2 <= n <= ops.MAX_CLOUD]
        if bad:
            raise ValueError(f'forward_packed: every cloud needs 2 .. {ops.MAX_CLOUD} nodes, got {bad[:8]}')
        for name, per_cloud in (('adj_mat', adj_mat), ('edges', edges), ('neighbor_mask', neighbor_mask)):
            if per_cloud is None:
                continue
            if not isinstance(per_cloud, (list, tuple)) or len(per_cloud) != B:
                raise ValueError(f'forward_packed: {name} must be a list of {B} per-cloud tensors, got '
                                 f'{len(per_cloud) if isinstance(per_cloud, (list, tuple)) else type(per_cloud).__name__}')
            dims = 3 if name == 'edges' and not exists(self.edge_emb) else 2
            for c, (t, n) in enumerate(zip(per_cloud, seqlens)):
                if _is_sparse(t):
                    raise ValueError(f'forward_packed: {name}[{c}] is a sparse tensor; forward_packed takes dense per-cloud '
                                     f'tensors (its clouds have at most {ops.MAX_CLOUD} nodes), or use forward for sparse pair inputs')
                if not torch.is_tensor(t) or t.dim() != dims or tuple(t.shape[:2]) != (n, n):
                    want = f'[{n}, {n}, edge_dim]' if dims == 3 else f'[{n}, {n}]'
                    raise ValueError(f'forward_packed: {name}[{c}] must be {want} for a cloud of {n} nodes, got '
                                     f'{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
        assert not (self.attend_sparse_neighbors and not exists(adj_mat)), 'adjacency matrix (adjacency_mat) or edges (edges) must be passed in'
        assert not (self.has_edges and not exists(edges)), 'edge embedding (num_edge_tokens & edge_dim) must be supplied if one were to train on edge types'
        if exists(self.pos_emb):
            assert max(seqlens) <= self.num_positions, 'feature sequence length must be less than the number of positions given at init'
        return seqlens

    def _forward_packed_once(self, feats, coors, seqlens, adj_mat, edges, neighbor_mask, return_type, return_pooled):
        out_dtype = self._compute_dtype(coors)
        if self.output_degrees == 1:
            return_type = 0
        T, dev = sum(seqlens), coors.device
        lens = torch.tensor(seqlens)
        node_len = torch.repeat_interleave(lens, lens)                                  # n_c of every node
        node_start = torch.repeat_interleave(lens.cumsum(0) - lens, lens)               # start_c of every node
        local_pos = torch.arange(T) - node_start                                        # i_local
        pair_row = torch.repeat_interleave(torch.tensor(ops.pair_offsets(seqlens)), lens) + local_pos * node_len - node_start
        node_start, local_pos = node_start.to(dev), local_pos.to(dev)

        if isinstance(feats, dict):
            feats = {k: v.unsqueeze(0) for k, v in feats.items()}
        else:
            feats = self._embed_tokens(feats.unsqueeze(0), local_pos)
            feats = {'0': feats[..., None]}
        feats = self._check_features(feats, coors)
        valid_radius = self._valid_radius()

        # per cloud, exactly as forward() on that cloud alone: bonded neighbours, hop counts and the neighbour count k_c
        ks, sparse, hops = [], [], []
        for c, n in enumerate(seqlens):
            adj_indices, sparse_mask, num_sparse = self._bonded(adj_mat[c].to(dev) if exists(adj_mat) else None, 1, n, dev)
            ks.append(self._num_neighbors(n, num_sparse))
            if exists(sparse_mask):
                sparse.append(sparse_mask.reshape(-1))
            if exists(adj_indices):
                hops.append(adj_indices.reshape(-1))
            if exists(neighbor_mask):
                eye = torch.eye(n, dtype=torch.bool, device=dev)
                self._report_neighbor_mask(neighbor_mask[c].to(dev).masked_fill(eye, False).sum(dim=-1))
        nbr = torch.cat([m.to(dev).reshape(-1) for m in neighbor_mask]) if exists(neighbor_mask) else None
        idx, nmask, rel_pos, rel_dist = ops.knn(coors.float(), ks, valid_radius, neighbor_mask=nbr,
                                                sparse_adj=torch.cat(sparse) if sparse else None, causal=self.causal, seqlens=seqlens)

        # edge values: pair (i, j) of cloud c sits at pair_off[c] + i_local n_c + j_local of the flattened per-cloud inputs
        flat = pair_row.to(dev)[:, None] + idx if exists(edges) or exists(self.adj_emb) else None      # [T, K]
        edge_values = None
        if exists(edges):
            edge_values = torch.cat([t.to(dev).reshape(n * n, *t.shape[2:]) for t, n in zip(edges, seqlens)])[flat]
        e = self._edge_features(edge_values, torch.cat(hops)[flat] if exists(self.adj_emb) else None)

        idx, nmask, rel_pos, rel_dist = idx.unsqueeze(0), nmask.unsqueeze(0), rel_pos.unsqueeze(0), rel_dist.unsqueeze(0)
        pos_emb = None
        if exists(self.rotary_pos_emb):
            k_pos = torch.cat((local_pos.view(1, T, 1), idx - node_start.view(1, T, 1)), dim=2)
            pos_emb = self._rotary(local_pos.view(1, T), k_pos, max(seqlens), rel_dist)
        if return_pooled:
            reduce = lambda v: torch.stack([s.mean(dim=0) for s in v[0].split(seqlens)])
        else:
            reduce = lambda v: v[0]
        edge_info = (idx, nmask, None if e is None else e.unsqueeze(0))
        return self._trunk(feats, edge_info, rel_pos, rel_dist, pos_emb, None, None, reduce, out_dtype, return_type)


class GraphedForward:
    """CUDA-graph replay of SE3Transformer.forward for fixed shapes.  Inputs are copied into static device buffers
    (host tensors are accepted: the copy is then the H2D transfer); the returned tensors are the graph's static outputs
    and are overwritten by the next call.  A replay runs the kernels the switches (switches.py) selected at capture; changing a
    switch needs a new capture."""

    def __init__(self, model, feats, coors, mask=None, warmup=2, **fwd_kwargs):
        assert not model.attend_sparse_neighbors and fwd_kwargs.get('neighbor_mask') is None, \
            'graph capture needs a synchronisation-free forward'
        dev = next(model.parameters()).device
        self.model, self.kw = model, fwd_kwargs
        clone = lambda t: t.to(dev).clone()
        self.feats = {k: clone(v) for k, v in feats.items()} if isinstance(feats, dict) else clone(feats)
        self.coors = clone(coors)
        self.mask = None if mask is None else clone(mask)
        self.static_kw = {k: (clone(v) if torch.is_tensor(v) else v) for k, v in fwd_kwargs.items()}
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):                    # builds weight images / tables outside the capture
                model(self.feats, self.coors, self.mask, **self.static_kw)
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = model(self.feats, self.coors, self.mask, **self.static_kw)
        self.checks = model._graph_checks

    def __call__(self, feats, coors, mask=None, **tensor_kwargs):
        if isinstance(feats, dict):
            for k, v in feats.items():
                self.feats[k].copy_(v, non_blocking=True)
        else:
            self.feats.copy_(feats, non_blocking=True)
        self.coors.copy_(coors, non_blocking=True)
        if (mask is None) != (self.mask is None):
            raise ValueError('GraphedForward: `mask` must be given exactly when the graph was captured with one')
        if mask is not None:
            self.mask.copy_(mask, non_blocking=True)
        for k, v in tensor_kwargs.items():                # edges / adj_mat / global_feats captured as static buffers
            if not torch.is_tensor(self.static_kw.get(k)):
                raise ValueError(f'GraphedForward: {k} was not a tensor argument of the captured forward')
            self.static_kw[k].copy_(v, non_blocking=True)
        self.graph.replay()
        # the run-time check of the low-rank plans, read once per replay (the tensors are static outputs of the graph)
        bad = check_lowrank_stats(self.checks)
        if bad:
            raise LowRankPlanMiss('captured forward: the low-rank radial plan does not cover this input (distances beyond the range '
                                  'seen when the graph was captured); build a new graph or pack_weights(max_distance=...) for a larger range')
        return self.out


FLT_MAX = 3.4028234663852886e38


class _StepRows:
    """The node chunk of a decoding step, in the batch-1 view with global indices that forward_packed uses: its rows are
    the step's new nodes (row-level tensors are passed as they are) and its neighbours are gathered from the decoder's cache,
    a [1, rows * capacity, ...] tensor of which src() gives the view the kernels expect (NodeChunk.src)."""
    b0, b1, whole = 0, 1, False

    def __init__(self, rows):
        self.n_rows = rows

    def rows(self, t):
        return t

    def edge_info(self, edge_info):
        return edge_info

    def src(self, t):
        if isinstance(t, dict):
            return {key: self.src(v) for key, v in t.items()}
        return t[:, :self.n_rows]


def _refuse_undecodable(model, api):
    """The models whose outputs cannot be decoded from a cache of earlier rows, refused with the reason (both decoders)."""
    if not model.causal:
        raise ValueError(f'{api}: the model is not causal (causal=False): the outputs of earlier nodes would change as '
                         'nodes arrive, so they cannot be cached')
    if model.attend_sparse_neighbors or exists(model.num_adj_degrees):
        raise NotImplementedError(f'{api}: attend_sparse_neighbors and num_adj_degrees are not supported: the number of '
                                  'bonded neighbours and the hop counts depend on the whole adjacency, including future rows')
    if model.accept_global_feats:
        raise NotImplementedError(f'{api}: models built with global_feats_dim are not supported (the attention kernel '
                                  'indexes the global keys by batch row, and a decoding step is one row)')
    if not model.valid_radius < FLT_MAX:
        raise ValueError(f'{api}: valid_radius = {model.valid_radius} >= FLT_MAX: the FLT_MAX keys of later nodes would '
                         'count as valid neighbours, so even forward() is not causal; give a finite radius below FLT_MAX')


class _DecoderStages:
    """What CausalDecoder and PackedCausalDecoder share: the per-stage cache and the walk of a step through the stages once its
    graph is built.

    Node i of a causal model depends only on nodes j <= i: the neighbour search gives every later column the key FLT_MAX, so
    later nodes only fill masked slots, which get zero weight in the attention softmax and in the pooled means; everything else
    is per node.  A decoder therefore keeps, per cloud and per stage, the node features that later nodes gather as neighbours
    (the embedded input of conv_in, the input of each pre-convolution, prenorm(x) of every attention block and its node keys
    with linear_proj_keys, the input of conv_out), with their node maxima (the production route's edge scales), in tensors
    [rows, cap, ...] whose row r holds one cloud.  A step searches the neighbours of the new rows only, runs every convolution
    and attention block over the new nodes' edges and the node-level work over the new rows, and stores the new rows in the
    cache.  A subclass builds the step's graph and says where its new rows go (_store)."""

    row_bytes = 12                                # cache bytes per node besides the stages: the coordinates

    def __init__(self, model, api):
        _refuse_undecodable(model, api)
        self.model = model
        self.cap = 0
        self.coors = None                         # [rows, cap, 3] fp32
        self.stages = {}                          # name -> (feats {d: [rows, cap, C, 2d+1]}, nodemax [rows, cap])

    def cache_bytes_per_node(self):
        """Bytes the cache holds per node of a cloud (features, node maxima, coordinates and, with a node mask, the mask)."""
        per = self.row_bytes
        for feats, nodemax in self.stages.values():
            per += sum(t[0, 0].numel() * 4 for t in feats.values()) + 4
        return per

    def _store(self, cache, rows, step):
        """Write the step's new rows [R, ...] into their places in cache [rows, cap, ...]."""
        raise NotImplementedError

    def _append(self, name, x, step):
        """Store the new rows x {d: [1, R, C, 2d+1]} of stage `name`; returns the stage's cache in the batch-1 view,
        {d: [1, rows cap, C, 2d+1]}, and its node maxima [rows cap]."""
        if name not in self.stages:
            shape = tuple(self.coors.shape[:2])
            self.stages[name] = ({d: t.new_empty(shape + tuple(t.shape[2:])) for d, t in x.items()},
                                 torch.empty(shape, dtype=torch.float32, device=self.coors.device))
        feats, nodemax = self.stages[name]
        for d, t in x.items():
            self._store(feats[d], t[0], step)
        self._store(nodemax, ops.node_absmax(x).view(-1), step)
        return {d: t.view((1, -1) + tuple(t.shape[2:])) for d, t in feats.items()}, nodemax.view(-1)

    def _conv(self, conv, name, x, step):
        """conv over the step's edges, its neighbours gathered from the cache of stage `name`, to which x is appended first."""
        src, nodemax = self._append(name, x, step)
        edge_info, rel_dist, geom, rows = step['edge_info'], step['rel_dist'], step['geom'], step['rows']
        d = conv_decide(conv, edge_info[0].numel(), rel_dist, geom)
        sx = self._edge_scale([d], nodemax, edge_info[0])
        self_out = conv.self_interact(x) if conv.self_interaction else None
        return conv_forward([conv], rows.src(src), edge_info, rel_dist, (None, None, geom), decisions=[d], self_out=self_out, sx=sx)[0]

    def _edge_scale(self, decisions, nodemax, idx):
        """chunk_edge_scale from the cached node maxima."""
        if not any(d.route == 'production' for d in decisions):
            return None
        return ops.edge_scale(None, idx, max(di for di, _ in decisions[0].conv.fiber_in), nodemax=nodemax).view(idx.shape)

    def _attend(self, i, block, x, step, pos_emb):
        attn = block.attn
        features = block.prenorm(x)
        src, nodemax = self._append(('attn', i), features, step)
        node_keys = None
        if attn.linear_proj_keys:
            node_keys = self._append(('keys', i), attn.to_k(features), step)[0]
        edge_info, rel_dist, geom, rows = step['edge_info'], step['rel_dist'], step['geom'], step['rows']
        queries, kv, k_emb = attn.node_level(features, None, pos_emb, node_keys=node_keys)
        decisions = [conv_decide(conv, edge_info[0].numel(), rel_dist, geom) for conv in attn.edge_convs()]
        sx = self._edge_scale(decisions, nodemax, edge_info[0])
        outputs = attn._attend(rows, src, queries, kv, k_emb, edge_info, rel_dist, (None, None, geom), decisions,
                               attn.fuse_rotation(geom), sx)
        return attn.project_out(outputs, x)

    def _walk(self, feats, step, pos_emb, reduce, out_dtype, return_type):
        """Every stage of the trunk over the step's R new rows (feats {d: [1, R, C, 2d+1]}; step: the graph in the batch-1 view,
        rows, edge_info, rel_dist and geom, and what _store needs): (outputs, deferred checks of the low-rank plans)."""
        model = self.model
        x = self._conv(model.conv_in, 'in', feats, step)
        for i, (conv, nonlin) in enumerate(model.convs):
            x = self._conv(conv, ('conv', i), nonlin(x), step)
        for i, (attn_block, ff) in enumerate(model.net.blocks):
            x = ff(self._attend(i, attn_block, x, step, pos_emb))
        if exists(model.conv_out):
            x = self._conv(model.conv_out, 'out', x, step)
        return self._output(x, reduce, out_dtype, return_type, step), step['geom'].deferred

    def _output(self, x, reduce, out_dtype, return_type, step):
        """The step's outputs from the trunk's last features (SE3Transformer._output)."""
        return self.model._output(x, reduce, out_dtype, return_type)


class CausalDecoder(_DecoderStages):
    """Generation with a causal SE3Transformer, node by node (SE3Transformer.causal_decoder); see _DecoderStages for what is
    cached and why it is exact.  Lockstep batches: the cache row of cloud c is c, and every call adds the same number of nodes
    to each of the batch_size clouds.

    extend(feats, coors, ...) returns rows [n_prev, n_cur) of what forward returns for all nodes so far, with the [b, n, n] pair
    inputs stacked from the rows given (anything above the diagonal).  The first call (the prefill) needs at least 2 nodes, as a
    forward does."""

    row_bytes = 13                                # coordinates and node mask

    def __init__(self, model, batch_size=1):
        super().__init__(model, 'causal_decoder')
        if operator.index(batch_size) < 1:
            raise ValueError(f'causal_decoder: batch_size must be >= 1, got {batch_size}')
        self.b = int(batch_size)
        self.n = 0
        self.mask = None                          # [b, cap] bool

    def __len__(self):
        return self.n

    # ---- checks --------------------------------------------------------------------------------------------
    def _check(self, feats, coors, mask, edges, neighbor_mask, return_pooled):
        """Everything extend takes from the caller, checked before any device work; returns m."""
        model, b = self.model, self.b
        if return_pooled:
            raise ValueError('extend: return_pooled is not supported: the mean over nodes changes with every node that arrives')
        for name, t in (('edges', edges), ('neighbor_mask', neighbor_mask), ('mask', mask), ('coors', coors)):
            if _is_sparse(t):
                raise ValueError(f'extend: {name} is a sparse tensor; decoding takes dense rows (sparse pair inputs are not supported)')
        if not torch.is_tensor(coors) or coors.dim() != 3 or coors.shape[0] != b or coors.shape[2] != 3 or coors.shape[1] < 1:
            raise ValueError(f'extend: coors must be [batch_size, m, 3] with batch_size = {b}, m >= 1, got '
                             f'{tuple(coors.shape) if torch.is_tensor(coors) else type(coors).__name__}')
        m = coors.shape[1]
        n_cur = self.n + m
        if n_cur < 2:
            raise ValueError('extend: the first call (the prefill) needs at least 2 nodes per cloud, as a forward does')
        for t in (feats.values() if isinstance(feats, dict) else [feats]):
            if not torch.is_tensor(t) or t.dim() < 2 or tuple(t.shape[:2]) != (b, m):
                raise ValueError(f'extend: the features must be [batch_size, m, ...] = {(b, m)} like coors, got '
                                 f'{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
            if _is_sparse(t):
                raise ValueError('extend: sparse features are not supported')
        if mask is not None and (not torch.is_tensor(mask) or tuple(mask.shape) != (b, m)):
            raise ValueError(f'extend: mask must be [batch_size, m] = {(b, m)}, got {tuple(mask.shape) if torch.is_tensor(mask) else type(mask).__name__}')
        if neighbor_mask is not None and (not torch.is_tensor(neighbor_mask) or tuple(neighbor_mask.shape) != (b, m, n_cur)):
            raise ValueError(f'extend: neighbor_mask must be the new rows [batch_size, m, n_cur] = {(b, m, n_cur)}, got '
                             f'{tuple(neighbor_mask.shape) if torch.is_tensor(neighbor_mask) else type(neighbor_mask).__name__}')
        if model.has_edges and edges is None:
            raise ValueError('extend: the model has edge features (edge_dim): pass edges for the new rows')
        if edges is not None:
            if not model.has_edges:
                raise ValueError('extend: edges given, but the model was built without edge_dim')
            dims = 3 if exists(model.edge_emb) else 4
            if not torch.is_tensor(edges) or edges.dim() != dims or tuple(edges.shape[:3]) != (b, m, n_cur):
                shape = '[batch_size, m, n_cur]' if exists(model.edge_emb) else '[batch_size, m, n_cur, edge_dim]'
                raise ValueError(f'extend: edges must hold the pair values of every new node to every node so far, {shape} with '
                                 f'batch_size, m, n_cur = {(b, m, n_cur)}, got {tuple(edges.shape) if torch.is_tensor(edges) else type(edges).__name__}')
        if exists(model.pos_emb) and n_cur > model.num_positions:
            raise ValueError(f'extend: node {n_cur - 1} is past num_positions = {model.num_positions}')
        return m

    # ---- one step ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def extend(self, feats, coors, mask=None, edges=None, neighbor_mask=None, return_type=None, return_pooled=False):
        """Append m >= 1 nodes to each cloud and return their outputs, shaped like forward's for [batch_size, m] nodes.
        feats [b, m, dim_in] float, [b, m] tokens or {'d': [b, m, C, 2d+1]}; coors [b, m, 3]; mask [b, m]; edges [b, m, n_cur]
        tokens or [b, m, n_cur, edge_dim]; neighbor_mask [b, m, n_cur] (n_cur = len(self) + m)."""
        m = self._check(feats, coors, mask, edges, neighbor_mask, return_pooled)
        out = self.model._checked(lambda: self._step(feats, coors, mask, edges, neighbor_mask, return_type, m))
        self.n += m
        return out

    def _grow(self, n_cur, dev):
        """Capacity for n_cur nodes per cloud: doubled when full, so a step never copies the whole prefix."""
        if n_cur <= self.cap:
            return
        cap = max(n_cur, 2 * self.cap, 16)

        def grown(t):
            new = t.new_empty((self.b, cap) + tuple(t.shape[2:]))
            new[:, :self.n] = t[:, :self.n]
            return new
        if self.coors is None:
            self.coors = torch.empty((self.b, 0, 3), dtype=torch.float32, device=dev)
            self.mask = torch.ones((self.b, 0), dtype=torch.bool, device=dev)
        self.coors, self.mask = grown(self.coors), grown(self.mask)
        self.stages = {name: ({d: grown(t) for d, t in feats.items()}, grown(nodemax)) for name, (feats, nodemax) in self.stages.items()}
        self.cap = cap

    def _step(self, feats, coors, mask, edges, neighbor_mask, return_type, m):
        """One extend (idempotent until self.n moves, so that a low-rank plan miss can run it again): (outputs, deferred checks)."""
        model, b = self.model, self.b
        n0, n1 = self.n, self.n + m
        out_dtype = model._compute_dtype(coors)
        if model.output_degrees == 1:
            return_type = 0
        dev = coors.device
        positions = torch.arange(n0, n1, device=dev)
        feats = model._embed_tokens(feats, positions)
        if torch.is_tensor(feats):
            feats = {'0': feats[..., None]}
        if exists(edges) and edges.is_floating_point():
            edges = edges.float()
        feats = model._check_features(feats, coors)
        self._grow(n1, dev)
        self.coors[:, n0:n1] = coors.float()
        self.mask[:, n0:n1] = True if mask is None else mask.to(dev, torch.bool)
        k = model._num_neighbors(n1, 0)
        idx, nmask, rel_pos, rel_dist = ops.knn_rows(self.coors, n1, n0, m, k, model._valid_radius(), node_mask=self.mask,
                                                     neighbor_mask=None if neighbor_mask is None else neighbor_mask.to(dev),
                                                     causal=True)
        edge_values = None
        if exists(edges):
            edges = edges.to(dev)
            edge_values = edges.gather(2, idx) if exists(model.edge_emb) else \
                edges.gather(2, idx[..., None].expand(-1, -1, -1, edges.shape[-1]))
        e = model._edge_features(edge_values, None)
        pos_emb = None
        if exists(model.rotary_pos_emb):
            q_pos = positions.view(1, m).expand(b, m)
            pos_emb = model._rotary(q_pos.reshape(1, b * m), torch.cat((q_pos[..., None], idx), dim=2).view(1, b * m, 1 + k), n1,
                                    rel_dist.view(1, b * m, k))
        # the batch-1 view: new row (c, i) is row c m + i, cached node (c, j) is node c cap + j
        gidx = (idx + (torch.arange(b, device=dev) * self.cap).view(b, 1, 1)).view(1, b * m, k)
        flat = lambda t: None if t is None else t.reshape((1, b * m) + tuple(t.shape[2:]))
        geom = Geometry(flat(rel_pos), model.num_degrees - 1, deferred=[])
        step = dict(n0=n0, m=m, rows=_StepRows(b * m), edge_info=(gidx, flat(nmask), flat(e)), rel_dist=flat(rel_dist), geom=geom)
        return self._walk({d: flat(t) for d, t in feats.items()}, step, pos_emb, lambda v: v.view((b, m) + tuple(v.shape[2:])),
                          out_dtype, return_type)

    def _store(self, cache, rows, step):
        """New row (c, i) goes to node n0 + i of cache row c."""
        n0, m = step['n0'], step['m']
        cache[:, n0:n0 + m] = rows.view((self.b, m) + tuple(rows.shape[1:]))


class PackedCausalDecoder(_DecoderStages):
    """Generation with a causal SE3Transformer for clouds of different lengths that join, leave, rewind and fork on their own
    (SE3Transformer.packed_decoder); see _DecoderStages for what is cached and why it is exact.  Inputs and outputs follow
    forward_packed: the nodes of a step are concatenated along one axis, with no batch padding and no node mask.

    For every cloud, the rows returned across its extend calls are the rows of model(feats_c[None], coors_c[None], ...) over that
    cloud's nodes so far (batch 1, no mask), whatever the other clouds of the same steps do, however its nodes were split into
    calls, and across truncate, fork and the reuse of a closed cloud's cache row.  Each cloud has its own neighbour count
    k_c = min(num_neighbors, n_cur_c - 1) in a step of K = max k_c slots (slots r >= k_c are masked), and positions and rotary
    positions count from the cloud's first node.

    The cache is [S, cap, ...] per stage: cloud c lives in row slot_c, and its node j at column j.  S doubles when more clouds
    are open than there are rows and cap doubles when a cloud outgrows it; a row costs cap nodes whatever its cloud's length (no
    paged cache).  Columns at or past a cloud's length are never read, so truncate only moves the length and close only frees
    the row.  A step without pair inputs launches no device work per cloud; edges and neighbor_mask are concatenated from one
    tensor per listed cloud."""

    def __init__(self, model):
        super().__init__(model, 'packed_decoder')
        self.S = 0                                # cache rows allocated on the device
        self._next_id = 0
        self._slot, self._len = {}, {}            # open cloud id -> cache row, number of nodes

    # ---- lifecycle -----------------------------------------------------------------------------------------
    def open(self, count=1):
        """count new empty clouds; returns their ids, increasing integers that are never reused."""
        if operator.index(count) < 1:
            raise ValueError(f'open: count must be >= 1, got {count}')
        ids = []
        for _ in range(int(count)):
            used = set(self._slot.values())
            slot = next(s for s in range(len(used) + 1) if s not in used)
            ids.append(self._next_id)
            self._slot[self._next_id], self._len[self._next_id] = slot, 0
            self._next_id += 1
        return ids

    def close(self, cloud):
        """Forget a cloud; its cache row is free for the next cloud that opens."""
        self._known(cloud, 'close')
        del self._slot[cloud], self._len[cloud]

    def truncate(self, cloud, n):
        """Rewind a cloud to its first n nodes (0 <= n <= length).  Exact: cached rows of nodes < n do not depend on later nodes."""
        self._known(cloud, 'truncate')
        n = operator.index(n)
        if not 0 <= n <= self._len[cloud]:
            raise ValueError(f'truncate: n must be in [0, {self._len[cloud]}] for cloud {cloud}, got {n}')
        self._len[cloud] = n

    @torch.no_grad()
    def fork(self, cloud):
        """A new cloud whose nodes so far are a copy of `cloud`'s (beam search, parallel sampling); returns its id."""
        self._known(cloud, 'fork')
        n, src = self._len[cloud], self._slot[cloud]
        new = self.open()[0]
        if n:
            dst = self._slot[new]
            self._grow(dst + 1, n, self.coors.device)
            for t in [self.coors] + [t for feats, nodemax in self.stages.values() for t in (*feats.values(), nodemax)]:
                t[dst, :n] = t[src, :n]
            self._len[new] = n
        return new

    def length(self, cloud):
        self._known(cloud, 'length')
        return self._len[cloud]

    def open_ids(self):
        return sorted(self._len)

    def _known(self, cloud, api):
        try:
            if operator.index(cloud) in self._len:
                return
        except TypeError:
            pass
        raise ValueError(f'{api}: {cloud!r} is not an open cloud of this decoder (open: {self.open_ids()[:16]})')

    # ---- checks --------------------------------------------------------------------------------------------
    def _check(self, ids, seqlens, feats, coors, edges, neighbor_mask, return_pooled):
        """Everything extend takes from the caller, checked before any device work; returns (ids, seqlens) as lists of ints."""
        model = self.model
        if return_pooled:
            raise ValueError('extend: return_pooled is not supported: the mean over nodes changes with every node that arrives')
        try:
            ids, seqlens = [operator.index(c) for c in ids], [operator.index(m) for m in seqlens]
        except TypeError:
            raise ValueError('extend: ids and seqlens must be sequences of ints') from None
        if not ids or len(set(ids)) != len(ids):
            raise ValueError(f'extend: ids must be distinct open clouds, at least one, got {ids[:16]}')
        for c in ids:
            self._known(c, 'extend')
        if len(seqlens) != len(ids) or min(seqlens) < 1:
            raise ValueError(f'extend: seqlens must hold one count >= 1 per listed cloud ({len(ids)}), got {seqlens[:16]}')
        M = sum(seqlens)
        n_cur = [self._len[c] + m for c, m in zip(ids, seqlens)]
        short = [c for c, n in zip(ids, n_cur) if n < 2]
        if short:
            raise ValueError(f'extend: clouds {short[:16]} would have fewer than 2 nodes; the first call of a cloud needs at least '
                             '2 nodes, as a forward does')
        if _is_sparse(coors) or not torch.is_tensor(coors) or tuple(coors.shape) != (M, 3):
            raise ValueError(f'extend: coors must be a dense [sum(seqlens), 3] = {(M, 3)} tensor, got '
                             f'{tuple(coors.shape) if torch.is_tensor(coors) else type(coors).__name__}')
        for t in (feats.values() if isinstance(feats, dict) else [feats]):
            if not torch.is_tensor(t) or t.dim() < 1 or t.shape[0] != M or _is_sparse(t):
                raise ValueError(f'extend: the features must be dense with sum(seqlens) = {M} rows, got '
                                 f'{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
        if model.has_edges and edges is None:
            raise ValueError('extend: the model has edge features (edge_dim): pass edges for the new rows of every listed cloud')
        if edges is not None and not model.has_edges:
            raise ValueError('extend: edges given, but the model was built without edge_dim')
        for name, per_cloud in (('edges', edges), ('neighbor_mask', neighbor_mask)):
            if per_cloud is None:
                continue
            if not isinstance(per_cloud, (list, tuple)) or len(per_cloud) != len(ids):
                raise ValueError(f'extend: {name} must be a list of {len(ids)} per-cloud tensors, got '
                                 f'{len(per_cloud) if isinstance(per_cloud, (list, tuple)) else type(per_cloud).__name__}')
            dims = 3 if name == 'edges' and not exists(model.edge_emb) else 2
            for c, t, m, n in zip(ids, per_cloud, seqlens, n_cur):
                if _is_sparse(t):
                    raise ValueError(f'extend: {name} of cloud {c} is a sparse tensor; decoding takes dense rows')
                if not torch.is_tensor(t) or t.dim() != dims or tuple(t.shape[:2]) != (m, n):
                    want = f'[m, n_cur, edge_dim] = [{m}, {n}, edge_dim]' if dims == 3 else f'[m, n_cur] = [{m}, {n}]'
                    raise ValueError(f'extend: {name} of cloud {c} must hold its new rows against all of its nodes so far, {want}, '
                                     f'got {tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
        if exists(model.pos_emb) and max(n_cur) > model.num_positions:
            raise ValueError(f'extend: node {max(n_cur) - 1} is past num_positions = {model.num_positions}')
        return ids, seqlens

    # ---- one step ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def extend(self, ids, seqlens, feats, coors, edges=None, neighbor_mask=None, return_type=None, return_pooled=False):
        """Append seqlens[i] >= 1 nodes to each listed cloud ids[i] and return their outputs; clouds not listed do not move.
        feats [M, dim_in] float, [M] tokens or {'d': [M, C, 2d+1]}; coors [M, 3]; M = sum(seqlens), rows in ids order.
        edges: one [m_c, n_cur_c] token or [m_c, n_cur_c, edge_dim] float tensor per listed cloud; neighbor_mask: one bool
        [m_c, n_cur_c] per listed cloud (the new rows against all of the cloud's nodes so far).  Returns what forward_packed
        returns for those M rows: {'d': [M, C, 2d+1]} ('0': [M, C]), or one degree with return_type."""
        ids, seqlens = self._check(ids, seqlens, feats, coors, edges, neighbor_mask, return_pooled)
        self._reserve(ids, seqlens, coors)
        out = self._run(ids, seqlens, feats, coors, edges, neighbor_mask, return_type)
        for c, m in zip(ids, seqlens):
            self._len[c] += m
        return out

    def _run(self, ids, seqlens, feats, coors, edges, neighbor_mask, return_type):
        """The step's outputs, once its cache room is reserved: its body and the check of its low-rank plans."""
        return self.model._checked(lambda: self._step(ids, seqlens, feats, coors, edges, neighbor_mask, return_type))

    def _reserve(self, ids, seqlens, coors):
        """Room in the cache for the step, made once before its body (which a low-rank plan miss runs again).  The rows of this
        cache grow inside the body (_search), which is idempotent."""

    def _grow(self, rows, n_cur, dev):
        """Room for cache rows [0, rows) of n_cur nodes: each axis doubled when full, so a step never copies the whole prefix."""
        S = self.S if rows <= self.S else max(rows, 2 * self.S)
        cap = self.cap if n_cur <= self.cap else max(n_cur, 2 * self.cap, 16)
        if self.coors is not None and (S, cap) == (self.S, self.cap):
            return
        keep = min(self.cap, max(self._len.values(), default=0))

        def grown(t):
            new = t.new_empty((S, cap) + tuple(t.shape[2:]))
            new[:self.S, :keep] = t[:, :keep]
            return new
        if self.coors is None:
            self.coors = torch.empty((0, 0, 3), dtype=torch.float32, device=dev)
        self.coors = grown(self.coors)
        self.stages = {name: ({d: grown(t) for d, t in feats.items()}, grown(nodemax)) for name, (feats, nodemax) in self.stages.items()}
        self.S, self.cap = S, cap

    def _step(self, ids, seqlens, feats, coors, edges, neighbor_mask, return_type):
        """One extend (idempotent until the lengths move, so that a low-rank plan miss can run it again): (outputs, deferred
        checks)."""
        model = self.model
        B, M = len(ids), sum(seqlens)
        n_prev = [self._len[c] for c in ids]
        n_cur = [p + m for p, m in zip(n_prev, seqlens)]
        out_dtype = model._compute_dtype(coors)
        if model.output_degrees == 1:
            return_type = 0
        dev = coors.device
        # per new row: its position in its cloud, where it goes (_where) and where its pair row starts in the concatenated inputs
        lens = torch.tensor(seqlens)
        first = torch.repeat_interleave(lens.cumsum(0) - lens, lens)
        local = torch.arange(M) - first
        pair_off = torch.tensor([0] + [m * n for m, n in zip(seqlens, n_cur)][:-1]).cumsum(0)
        pos = local + torch.repeat_interleave(torch.tensor(n_prev), lens)
        rows = torch.stack((pos, self._where(ids, lens, pos),
                            torch.repeat_interleave(pair_off, lens) + local * torch.repeat_interleave(torch.tensor(n_cur), lens)))
        pos, where, pair_row = rows.to(dev)
        if isinstance(feats, dict):
            feats = {d: v.unsqueeze(0) for d, v in feats.items()}
        else:
            feats = model._embed_tokens(feats.unsqueeze(0), pos)
            feats = {'0': feats[..., None]}
        feats = model._check_features(feats, coors)
        ks = [model._num_neighbors(n, 0) for n in n_cur]
        dest, idx, local_idx, nmask, rel_pos, rel_dist = self._search(
            ids, n_prev, seqlens, ks, pos, where, coors, None if neighbor_mask is None else [t.to(dev) for t in neighbor_mask])
        K = idx.shape[1]
        edge_values = None
        if exists(edges):
            edge_values = torch.cat([(t if exists(model.edge_emb) else t.float()).to(dev).reshape((-1,) + tuple(t.shape[2:]))
                                     for t in edges])[pair_row[:, None] + local_idx]
        e = model._edge_features(edge_values, None)
        pos_emb = None
        if exists(model.rotary_pos_emb):
            pos_emb = model._rotary(pos.view(1, M), torch.cat((pos[:, None], local_idx), dim=1).view(1, M, 1 + K), max(n_cur),
                                    rel_dist.view(1, M, K))
        geom = Geometry(rel_pos[None], model.num_degrees - 1, deferred=[])
        step = dict(dest=dest, rows=_StepRows(M), edge_info=(idx[None], nmask[None], None if e is None else e[None]),
                    rel_dist=rel_dist[None], geom=geom)
        return self._walk(feats, step, pos_emb, lambda v: v[0], out_dtype, return_type)

    def _where(self, ids, lens, pos):
        """What _search needs to place each new row (pos: its node in its cloud), host int64 [M]: its cloud's cache row."""
        return torch.repeat_interleave(torch.tensor([self._slot[c] for c in ids]), lens)

    def _search(self, ids, n_prev, seqlens, ks, pos, where, coors, neighbor_mask):
        """Store the step's coordinates and search its new rows' neighbours: (dest [M], the new rows' positions in the flat cache;
        idx [M, K], the neighbours' positions there; their columns in their clouds [M, K]; mask, rel_pos, rel_dist)."""
        slots = [self._slot[c] for c in ids]
        self._grow(max(slots) + 1, max(p + m for p, m in zip(n_prev, seqlens)), coors.device)
        base = where * self.cap                                             # the batch-1 view: node j of row s is s cap + j
        dest = base + pos
        self.coors.view(-1, 3).index_copy_(0, dest, coors.float())
        idx, nmask, rel_pos, rel_dist = ops.knn_rows_packed(self.coors, slots, n_prev, seqlens, ks, self.model._valid_radius(),
                                                            causal=True, neighbor_mask=neighbor_mask)
        return dest, idx, idx - base[:, None], nmask, rel_pos, rel_dist

    def _store(self, cache, rows, step):
        """New row t goes to flat position dest[t] of the cache (node n_prev_c + r of cache row slot_c)."""
        cache.view((-1,) + tuple(cache.shape[2:])).index_copy_(0, step['dest'], rows)


class DecoderCacheFull(RuntimeError):
    """A step of a PagedCausalDecoder with max_nodes needs more pages than its pool has free.  Raised before any device work,
    with the decoder unchanged: close, truncate or pre-empt clouds and send the step again."""


class StepPages(NamedTuple):
    """What a step needs from PageTables.plan: the pool size after it, the copy-on-write pages (cloud, index in its table, rows
    to copy), the fresh pages each listed cloud appends and, with a prefix cache, the cached pages each cloud in its first call
    attaches ((cloud, pages), ...)."""
    reserved: int
    cow: list
    fresh: list
    hits: tuple = ()


class PageTables:
    """The page bookkeeping of a PagedCausalDecoder, on the host (it holds no tensors): each cloud's block table, the ids of the
    pages that hold its nodes [0, P), [P, 2P), ...; one reference count per page; and a free list.  The pool has `reserved`
    pages on the device; a page that no table references is free, and allocations take freed pages first (the most recent
    first).  A cloud of n nodes has at least ceil(n / P) pages: more only after a step failed once its pages were taken.

    With cache=True it also keeps the prefix cache (DESIGN.md 10.4): page key -> page, least recently used first.  The cache holds
    one reference on each page it registers; a page only the cache holds is evictable (n_evictable counts them).  An allocation
    takes a free page, else evicts the least recently used evictable page; only then does the pool grow (or a capped pool refuse
    the step).  A page that a copy on write of the same commit copies from is never evicted by it.  A hit counts as a use once
    its step succeeds (use).  rollback restores tables, counts and entries, except the entries the commit evicted: their pages may
    already hold the failed step's rows, so they stay out of the cache and their pages are free."""

    def __init__(self, page_size, max_pages=None, cache=False):
        self.P, self.max_pages = page_size, max_pages
        self.reserved = 0
        self.refs = []                            # page id -> number of tables (and the cache) that hold it
        self.free = []                            # unreferenced page ids, taken from the end
        self.tables = {}                          # cloud -> page ids
        self.cached = collections.OrderedDict() if cache else None      # page key -> page id, least recently used first
        self.page_key = {}                        # cached page id -> its key
        self.n_evictable = 0                      # cached pages that only the cache holds
        self._victims = None                      # during a commit: its candidates for eviction, least recently used first

    def pages_in_use(self):
        return self.reserved - len(self.free) - self.n_evictable

    def pages_cached(self):
        return 0 if self.cached is None else len(self.cached)

    def _ref(self, p, delta):
        """Add delta to page p's count, keeping n_evictable in step."""
        r = self.refs[p]
        self.refs[p] = r + delta
        if p in self.page_key:
            self.n_evictable += (r + delta == 1) - (r == 1)

    def open(self, cloud):
        self.tables[cloud] = []

    def close(self, cloud):
        self._drop(self.tables.pop(cloud))

    def truncate(self, cloud, n):
        """Drop the cloud's pages past its first n nodes."""
        table = self.tables[cloud]
        keep = -(-n // self.P)
        self._drop(table[keep:])
        del table[keep:]

    def fork(self, cloud, new, n):
        """new shares the pages of cloud's first n nodes."""
        table = self.tables[cloud][:-(-n // self.P)]
        for p in table:
            self._ref(p, 1)
        self.tables[new] = list(table)

    def _drop(self, pages):
        for p in pages:
            self._ref(p, -1)
            if not self.refs[p]:
                self.free.append(p)

    # ---- the prefix cache ------------------------------------------------------------------------------------------
    def lookup(self, keys):
        """The cached pages of keys[0], keys[1], ... up to the first miss (nothing changes)."""
        pages = []
        for key in keys:
            p = self.cached.get(key) if self.cached else None
            if p is None:
                break
            pages.append(p)
        return pages

    def use(self, pages):
        """Mark the entries of these cached pages as the most recently used (a hit, once its step has succeeded)."""
        for p in pages:
            if p in self.page_key:
                self.cached.move_to_end(self.page_key[p])

    def register(self, key, page):
        """Cache `page` (a full page of a prompt) under `key`, with one reference; a key already registered keeps its entry."""
        if key in self.cached or page in self.page_key:
            return
        self.refs[page] += 1
        self.cached[key] = page
        self.page_key[page] = key
        self.n_evictable += self.refs[page] == 1

    def clear(self):
        """Drop every entry and the cache's references."""
        if self.cached:
            pages = list(self.cached.values())
            self.cached.clear()
            self.page_key.clear()
            self.n_evictable = 0
            self._drop(pages)

    def _evict(self, keep):
        """Take the least recently used evictable page (none in keep) out of the cache; returns it, unreferenced and not on the
        free list.  The candidates are listed once per commit: within a commit no page becomes evictable except the ones in keep."""
        if self._victims is None:
            self._victims = collections.deque(p for p in self.cached.values() if self.refs[p] == 1)
        while True:
            p = self._victims.popleft()
            if p in self.page_key and self.refs[p] == 1 and p not in keep:
                break
        del self.cached[self.page_key.pop(p)]
        self.n_evictable -= 1
        self.refs[p] = 0
        return p

    # ---- steps -------------------------------------------------------------------------------------------------------
    def plan(self, ids, n_prev, seqlens, hits=()):
        """The pages a step that appends seqlens[i] nodes to cloud ids[i] of n_prev[i] nodes needs (StepPages), without changing
        anything.  A step writes nodes >= n_prev only, so the one page of a cloud that it may write while another cloud holds it
        is the page of node n_prev, when n_prev is not a page boundary: that page is copied on write, its first n_prev % P rows.
        Clouds are planned in order, so of siblings that write one shared page in the same step the last writes it in place.
        hits: (cloud, cached pages) of clouds in their first call, which attach those pages (n_prev = len(pages) P).  Raises
        DecoderCacheFull if a capped pool has too few free and evictable pages."""
        P = self.P
        attach = dict(hits)
        refs, cow, fresh = {}, [], []
        for c, p, m in zip(ids, n_prev, seqlens):
            table = attach.get(c, self.tables[c])
            if p % P:
                page = table[p // P]
                r = refs.get(page, self.refs[page])
                if r > 1:
                    cow.append((c, p // P, p % P))
                    refs[page] = r - 1
            fresh.append(max(0, -(-(p + m) // P) - len(table)))
        need = len(cow) + sum(fresh)
        hit_pages = {p for _, pages in hits for p in pages}
        spare = len(self.free) + self.n_evictable - sum(self.refs[p] == 1 for p in hit_pages)
        hits = tuple((c, tuple(pages)) for c, pages in hits)
        if self.max_pages is not None:
            if need > spare + self.max_pages - self.reserved:
                raise DecoderCacheFull(f'extend: the step needs {need} free pages of {P} nodes and the pool has '
                                       f'{spare + self.max_pages - self.reserved} of {self.max_pages} (max_nodes); close, '
                                       'truncate or pre-empt clouds and retry')
            return StepPages(self.max_pages, cow, fresh, hits)
        short = need - spare
        return StepPages(self.reserved if short <= 0 else max(2 * self.reserved, self.reserved + short), cow, fresh, hits)

    def commit(self, plan, ids):
        """Take the planned pages: attach the cached pages of plan.hits, grow the pool to plan.reserved, give each copy-on-write
        cloud a fresh page in place of the shared one and append fresh pages.  Returns the copies [(old page, new page, rows)]
        that the caller makes on the device."""
        self._victims = None
        keep = set()                              # pages copied from: they must keep their rows until the copies are made
        for c, pages in plan.hits:
            self.tables[c] = list(pages)
            for p in pages:
                self._ref(p, 1)
        if plan.reserved > self.reserved:
            # every evictable page goes before the pool grows: the new pages come after the free and the evicted ones
            evicted = [self._evict(keep) for _ in range(self.n_evictable)]
            self.free[:0] = list(range(plan.reserved - 1, self.reserved - 1, -1)) + evicted[::-1]
            self.refs += [0] * (plan.reserved - self.reserved)
            self.reserved = plan.reserved
        copies = []
        for c, at, rows in plan.cow:
            old = self.tables[c][at]
            keep.add(old)
            new = self._take(keep)
            self.tables[c][at] = new
            self._ref(old, -1)                    # still held by the cloud it was shared with (or the cache)
            copies.append((old, new, rows))
        for c, f in zip(ids, plan.fresh):
            self.tables[c] += [self._take(keep) for _ in range(f)]
        self._victims = None
        return copies

    def rollback(self, plan, ids, copies):
        """Undo commit(plan, ids), which returned copies, when it did not grow the pool: tables, counts and the free list are as
        they were before it, and so are the cache's entries except those it evicted, which stay evicted with their pages free
        (the failed step may have written them).  Pages go back to the free list in the reverse order of their taking."""
        for c, f in reversed(list(zip(ids, plan.fresh))):
            for _ in range(f):
                p = self.tables[c].pop()
                self.refs[p] = 0
                self.free.append(p)
        for (c, at, _), (old, new, _) in reversed(list(zip(plan.cow, copies))):
            self.tables[c][at] = old
            self._ref(old, 1)
            self.refs[new] = 0
            self.free.append(new)
        for c, pages in reversed(plan.hits):
            for p in pages:
                self._ref(p, -1)
            self.tables[c] = []

    def _take(self, keep=()):
        p = self.free.pop() if self.free else self._evict(keep)
        self.refs[p] = 1
        return p


PREFIX_SEEDS = (0x243F6A8885A308D3, 0x13198A2E03707344)         # se3_prefix_keys_fwd's lane seeds
PREFIX_GOLD = 0x9E3779B97F4A7C15
_U64 = (1 << 64) - 1


def _mix64(z):
    """splitmix64's finalizer on uint64 numpy arrays (wrapping)."""
    z = z ^ (z >> np.uint64(30))
    z = z * np.uint64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> np.uint64(27))
    z = z * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def prefix_page_keys(digests, P):
    """The prefix-cache keys of the full pages of a prompt from its node digests (uint64 [n, 2], se3_prefix_keys_fwd): per
    lane l, page q's digest is mix64(sum over its rows r of mix64(d[qP + r, l] + (r + 1) G)) and its key
    key_q = mix64(key_{q-1} ^ digest_q) from key_{-1} = the lane seed, so a key names every node of the prefix up to its page.
    Returns [(q, key lane 0, key lane 1)] for q < n // P, as Python ints."""
    d = np.asarray(digests, dtype=np.uint64)
    pages = d.shape[0] // P
    if not pages:
        return []
    with np.errstate(over='ignore'):
        r = (np.arange(1, P + 1, dtype=np.uint64) * np.uint64(PREFIX_GOLD))[None, :, None]
        page = _mix64(_mix64(d[:pages * P].reshape(pages, P, 2) + r).sum(axis=1, dtype=np.uint64))
        keys, k = [], np.array(PREFIX_SEEDS, dtype=np.uint64)
        for q in range(pages):
            k = _mix64(k ^ page[q])
            keys.append((q, int(k[0]), int(k[1])))
    return keys


DECODE_GRAPH_ROWS = 64        # most rows of a paged decoding step that is replayed from a CUDA graph


def decode_graph_bucket(max_nodes, n_prev, seqlens, ks):
    """The CUDA-graph bucket (M rounded up to a power of two, K) of a step of a PagedCausalDecoder built with max_nodes that
    appends seqlens[c] nodes to clouds of n_prev[c] nodes with k_c = ks[c] neighbours, or None if the step runs eagerly: a
    decoder without max_nodes (its pool moves when it grows), a cloud in its first call (a prompt), more than DECODE_GRAPH_ROWS
    rows or clouds with different k_c."""
    M = sum(seqlens)
    if max_nodes is None or min(n_prev) == 0 or M > DECODE_GRAPH_ROWS or len(set(ks)) != 1:
        return None
    return 1 << (M - 1).bit_length(), ks[0]


class _DecodeGraph:
    """One captured step of a PagedCausalDecoder for a bucket of rows (M_bucket) and neighbours (K), and the static buffers it
    reads: the descriptor (pinned on the host, and its device copy), the features, coordinates and pair inputs of M_bucket rows
    (pair inputs concatenated per cloud, room for M_bucket rows of n_pos columns), and the outputs and deferred low-rank
    checks it writes."""

    def __init__(self, rows, K, n_pos, page_ids, feats, coors, edges, neighbor_mask):
        dev = coors.device
        self.rows, self.K, self.room = rows, K, page_ids
        self.out_dtype = coors.dtype if coors.dtype == torch.float64 else None       # as SE3Transformer._compute_dtype
        words = ops.decode_desc_words(rows, page_ids)
        self.host_desc = torch.zeros(words, dtype=torch.int32).pin_memory()
        self.desc = torch.zeros(words, dtype=torch.int32, device=dev)
        static = lambda t: torch.zeros((rows,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        self.feats = {d: static(v) for d, v in feats.items()} if isinstance(feats, dict) else static(feats)
        self.coors = torch.zeros((rows, 3), dtype=torch.float32, device=dev)
        self.edges = self.nbr = None
        if edges is not None:
            e = edges[0]
            dtype = e.dtype if not e.is_floating_point() else torch.float32
            self.edges = torch.zeros((rows * n_pos,) + tuple(e.shape[2:]), dtype=dtype, device=dev)
        if neighbor_mask is not None:
            self.nbr = torch.zeros(rows * n_pos, dtype=torch.uint8, device=dev)
        self.copied = torch.cuda.Event()          # recorded after each replay: its descriptor copy is done
        self.graph = self.out = self.checks = None


class PagedCausalDecoder(PackedCausalDecoder):
    """PackedCausalDecoder with its cache in pages of page_size nodes (SE3Transformer.packed_decoder(page_size=...)): the same
    open, extend, truncate, fork, close, length and open_ids, with the same results, refusals and messages, while memory
    follows the nodes decoded and forked clouds share their prefix.

    Every stage is [pages, P, C, 2d+1], with node maxima [pages, P] and coordinates [pages, P, 3], and each cloud has a block
    table on the host (PageTables): node j of cloud c is row j % P of page table_c[j // P].  The neighbour search reads
    coordinates through the tables and returns pool rows, which every later kernel reads in the flat [1, pages P, ...] view,
    as it reads cache rows of the packed decoder; rows are therefore bit for bit the packed decoder's.  fork shares every page
    of the parent and does no device work; truncate and close drop references, and a page nobody references is reused.  A
    step writes nodes >= n_prev only, so before it runs, a page it would write while another cloud holds it is copied
    (PageTables.plan).  The pool doubles when it runs out of pages, or, with max_nodes, is fixed at ceil(max_nodes / P) pages
    and a step that does not fit raises DecoderCacheFull before any device work, leaving the decoder unchanged."""

    def __init__(self, model, page_size, max_nodes=None, prefix_cache=False):
        _DecoderStages.__init__(self, model, 'packed_decoder')
        if isinstance(page_size, bool) or not isinstance(page_size, numbers.Integral) or page_size < 1:
            raise ValueError(f'packed_decoder: page_size must be None or an integer >= 1, got {page_size!r}')
        if max_nodes is not None and (isinstance(max_nodes, bool) or not isinstance(max_nodes, numbers.Integral) or max_nodes < 1):
            raise ValueError(f'packed_decoder: max_nodes must be None or an integer >= 1, got {max_nodes!r}')
        if not isinstance(prefix_cache, bool):
            raise ValueError(f'packed_decoder: prefix_cache must be a bool, got {prefix_cache!r}')
        self.page_size = int(page_size)
        self.max_nodes = None if max_nodes is None else int(max_nodes)
        self.prefix_cache = prefix_cache
        self._book = PageTables(self.page_size, None if max_nodes is None else -(-self.max_nodes // self.page_size), prefix_cache)
        # the prefix cache (DESIGN.md 10.4): every eager step's outputs per pool row, the state its entries were computed under,
        # and how many nodes of each cloud came from it
        self._out = None                          # {d: [pages, P, ...]} float32, before the dtype cast and return_type
        self._out_rows = None                     # the rows of the running step that _out keeps (its prompts of a page or more)
        self._cache_sw = self._cache_plans = None
        self._prefix = {}
        self._next_id = 0
        self._len = {}                            # open cloud id -> number of nodes
        # CUDA-graph steps (max_nodes only, DESIGN.md 10.3): padding rows store into scratch pages after the pool's
        self._scratch_pages = 0 if max_nodes is None else -(-DECODE_GRAPH_ROWS // self.page_size)
        self._graphs = {}                         # (M_bucket, K, input kind) -> _DecodeGraph
        self._graph_pool = None                   # the memory pool the graphs share (they never run at the same time)
        self._graph_sw = self._graph_plans = None     # the switches and low-rank plans the graphs were captured with
        self._commit = None                       # the last step's page plan, ids and copies (PageTables.rollback)
        self.graph_replays = 0                    # steps replayed from a graph
        self.graph_capture_s = {}                 # (M_bucket, K) -> seconds its last capture took (with its warm-up step)

    def pages_in_use(self):
        """Distinct pages that open clouds reference."""
        return self._book.pages_in_use()

    def pages_reserved(self):
        """Pages allocated on the device."""
        return self._book.reserved

    def pages_cached(self):
        """Pages the prefix cache holds, whether or not a cloud also references them."""
        return self._book.pages_cached()

    def clear_prefix_cache(self):
        """Drop every prefix-cache entry; pages that no cloud references become free."""
        self._book.clear()

    def prefix_nodes(self, cloud):
        """How many of the cloud's nodes came from the prefix cache (its first nodes)."""
        self._known(cloud, 'prefix_nodes')
        return min(self._prefix.get(cloud, 0), self._len[cloud])

    # ---- lifecycle -----------------------------------------------------------------------------------------
    def open(self, count=1):
        """count new empty clouds; returns their ids, increasing integers that are never reused."""
        if operator.index(count) < 1:
            raise ValueError(f'open: count must be >= 1, got {count}')
        ids = list(range(self._next_id, self._next_id + int(count)))
        for c in ids:
            self._len[c] = 0
            self._book.open(c)
        self._next_id += int(count)
        return ids

    def close(self, cloud):
        """Forget a cloud; the pages only it held are free for the next allocation."""
        self._known(cloud, 'close')
        del self._len[cloud]
        self._prefix.pop(cloud, None)
        self._book.close(cloud)

    def truncate(self, cloud, n):
        """Rewind a cloud to its first n nodes (0 <= n <= length) and drop its pages past them."""
        super().truncate(cloud, n)
        self._book.truncate(cloud, self._len[cloud])
        if cloud in self._prefix:
            self._prefix[cloud] = min(self._prefix[cloud], self._len[cloud])

    def fork(self, cloud):
        """A new cloud whose nodes so far are `cloud`'s, sharing its pages (no device work, nothing allocated); returns its id."""
        self._known(cloud, 'fork')
        new = self.open()[0]
        self._len[new] = self._len[cloud]
        self._book.fork(cloud, new, self._len[cloud])
        if cloud in self._prefix:
            self._prefix[new] = self._prefix[cloud]
        return new

    # ---- the prefix cache (DESIGN.md 10.4) -----------------------------------------------------------------------------
    @torch.no_grad()
    def extend(self, ids, seqlens, feats, coors, edges=None, neighbor_mask=None, return_type=None, return_pooled=False):
        if not self.prefix_cache:
            return super().extend(ids, seqlens, feats, coors, edges, neighbor_mask, return_type, return_pooled)
        ids, seqlens = self._check(ids, seqlens, feats, coors, edges, neighbor_mask, return_pooled)
        prompts = [i for i, c in enumerate(ids) if self._len[c] == 0]
        self._commit = None
        if not prompts:                           # a decode step: no lookup, nothing to register
            out = self._attempt(lambda: (self._reserve(ids, seqlens, coors),
                                         self._run(ids, seqlens, feats, coors, edges, neighbor_mask, return_type))[1], {})
            for c, m in zip(ids, seqlens):
                self._len[c] += m
            return out
        ops._require_cuda(coors)                  # the lookup runs on the device
        sw = switches.current()
        if self._book.cached and not self._cache_current(sw):
            self._book.clear()                    # its rows were computed under other switches or plans
        starts = [0]
        for m in seqlens:
            starts.append(starts[-1] + m)
        keys, hits = self._lookup(ids, seqlens, starts, prompts, feats, coors, edges, neighbor_mask)
        P = self.page_size
        H = {c: len(pages) * P for c, pages in hits.items()}
        sub = [(i, c) for i, c in enumerate(ids) if seqlens[i] > H.get(c, 0)]
        sub_ids, sub_lens = [c for _, c in sub], [seqlens[i] - H.get(c, 0) for i, c in sub]
        args = (feats, coors, edges, neighbor_mask)
        if hits:                                  # the rest of the step: rows from n_prev = hP of each hit prompt
            keep = torch.tensor([r for i, c in sub for r in range(starts[i] + H.get(c, 0), starts[i + 1])], dtype=torch.int64)
            rows = lambda t: t[keep.to(t.device)]
            per_cloud = lambda ts: None if ts is None else [ts[i][H.get(c, 0):] for i, c in sub]
            args = ({d: rows(v) for d, v in feats.items()} if isinstance(feats, dict) else rows(feats), rows(coors),
                    per_cloud(edges), per_cloud(neighbor_mask))
        for c, h in H.items():
            self._len[c] = h
        kept, at = [], 0                          # the step rows of the prompts whose full pages may be registered
        for (i, _), m in zip(sub, sub_lens):
            if i in keys:
                kept += range(at, at + m)
            at += m
        self._out_rows = torch.tensor(kept, dtype=torch.int64).to(coors.device) if kept else None
        try:
            out = self._attempt(lambda: (self._reserve(sub_ids, sub_lens, coors, tuple(hits.items())),
                                         PackedCausalDecoder._run(self, sub_ids, sub_lens, *args, return_type) if sub_ids else None)[1],
                                H)
        finally:
            self._out_rows = None
        for c, m in zip(sub_ids, sub_lens):
            self._len[c] += m
        for i in prompts:
            self._prefix[ids[i]] = H.get(ids[i], 0)
        for pages in hits.values():
            self._book.use(pages)
        self._register(sw, ids, keys, hits)
        if not hits:
            return out
        return self._assemble(ids, seqlens, starts, hits, sub, out, coors, return_type)

    def _attempt(self, step, hits):
        """Run step(); if it raises, undo its page commit (the cache's entries too) and the lengths of the hit clouds."""
        try:
            return step()
        except BaseException:
            if self._commit is not None:
                self._rollback()
            for c in hits:
                self._len[c] = 0
            raise

    def _rollback(self):
        self._book.rollback(*self._commit)
        self._commit = None

    def _cache_current(self, sw):
        return sw == self._cache_sw and self._same_plans(self._plan_state(sw), self._cache_plans)

    def _lookup(self, ids, seqlens, starts, prompts, feats, coors, edges, neighbor_mask):
        """The page keys of every prompt of at least one page ({step index: [key of page 0, 1, ...]}), and the verified cached
        pages each prompt attaches ({cloud: pages}): its keys looked up from page 0 to the first miss, then its stored coordinates
        and conv_in rows compared bit for bit with the prompt's (one device comparison), stopping at the first page that differs."""
        model, P, dev = self.model, self.page_size, coors.device
        long = [i for i in prompts if seqlens[i] >= P]
        if not long:
            return {}, {}
        lens = [seqlens[i] for i in long]
        rows = torch.cat([torch.arange(starts[i], starts[i + 1]) for i in long])
        # the conv_in input of the prompt rows, as _step builds it (positions count from 0 in a first call)
        if isinstance(feats, dict):
            x = {d: v[rows.to(v.device)].unsqueeze(0) for d, v in feats.items()}
        else:
            pos = torch.cat([torch.arange(m) for m in lens]).to(dev)
            x = {'0': model._embed_tokens(feats[rows.to(feats.device)].unsqueeze(0), pos)[..., None]}
        x = {d: v[0] for d, v in model._check_features(x, coors).items()}
        R = rows.shape[0]
        width = torch.cat([x[d].reshape(R, -1) for d in sorted(x, key=int)], dim=1)
        xyz = coors[rows.to(dev)].float().contiguous()
        pair = lambda ts, f: None if ts is None else [f(ts[i].to(dev)) for i in long]
        e = pair(edges, lambda t: t.float() if t.is_floating_point() else t.long())
        digests = ops.prefix_keys(width, xyz, lens, edges=e, neighbor_mask=pair(neighbor_mask, lambda t: t))
        digests = digests.cpu().numpy().view(np.uint64)                # the one read-back of the keys
        first = torch.tensor([0] + lens[:-1]).cumsum(0).tolist()          # each prompt's first row among the R
        keys = {i: prefix_page_keys(digests[f:f + m], P) for i, f, m in zip(long, first, lens)}
        cand = {i: (f, self._book.lookup(keys[i])) for i, f in zip(long, first)}
        cand = {i: c for i, c in cand.items() if c[1]}
        if not cand:
            return keys, {}
        pages = torch.tensor([p for _, pg in cand.values() for p in pg]).to(dev)
        at = torch.tensor([f + r for f, pg in cand.values() for r in range(len(pg) * P)]).to(dev)
        n = pages.shape[0]
        same = lambda stored, new: (stored.reshape(n, -1).view(torch.int32) == new.reshape(n, -1).view(torch.int32)).all(1)
        ok = same(self.coors[pages], xyz[at])
        for d, t in self.stages['in'][0].items():
            ok &= same(t[pages], x[d][at])
        ok = ok.cpu().tolist()
        hits, j = {}, 0
        for i, (_, pg) in cand.items():
            good = ok[j:j + len(pg)]
            j += len(pg)
            h = good.index(False) if False in good else len(good)
            if h:
                hits[ids[i]] = pg[:h]
        return keys, hits

    def _register(self, sw, ids, keys, hits):
        """After a step that carried prompts: each prompt's full pages that the step wrote go into the cache under their keys,
        tagged with the switches and plans they were computed under (entries of other ones are dropped first)."""
        if not keys:
            return
        state = self._plan_state(sw)
        if self._book.cached and not (sw == self._cache_sw and self._same_plans(state, self._cache_plans)):
            self._book.clear()
        self._cache_sw, self._cache_plans = sw, state
        for i, page_keys in keys.items():
            table = self._book.tables[ids[i]]
            for q in range(len(hits.get(ids[i], ())), len(page_keys)):
                self._book.register(page_keys[q], table[q])

    def _assemble(self, ids, seqlens, starts, hits, sub, out, coors, return_type):
        """The step's rows in ids order: the hit prompts' first hP rows from the cached outputs, the others from the step."""
        P, dev = self.page_size, coors.device
        out_dtype = self.model._compute_dtype(coors)
        rt = 0 if self.model.output_degrees == 1 else return_type
        where = {c: i for i, c in enumerate(ids)}
        hit_at = torch.tensor([starts[where[c]] + r for c, pg in hits.items() for r in range(len(pg) * P)]).to(dev)
        pool = torch.tensor([p * P + r for pg in hits.values() for p in pg for r in range(P)]).to(dev)
        H = {c: len(pg) * P for c, pg in hits.items()}
        sub_at = torch.tensor([r for i, c in sub for r in range(starts[i] + H.get(c, 0), starts[i + 1])], dtype=torch.int64).to(dev)
        M = starts[-1]

        def place(d, part):
            v = self._out[d]
            cached = v.view((-1,) + tuple(v.shape[2:]))[pool]
            if exists(out_dtype):
                cached = cached.to(out_dtype)
            res = cached.new_empty((M,) + tuple(cached.shape[1:]))
            res.index_copy_(0, hit_at, cached)
            if part is not None:
                res.index_copy_(0, sub_at, part)
            return res
        if exists(rt):
            return place(str(rt), out)
        return {d: place(d, None if out is None else out[d]) for d in self._out}

    def _output(self, x, reduce, out_dtype, return_type, step):
        """With the prefix cache, a step that carries prompts of a page or more (always eager) also keeps their rows of every
        degree, in float32 before the dtype cast and return_type, at their pool rows: a later hit on their pages returns them."""
        rows = self._out_rows
        if rows is None:
            return super()._output(x, reduce, out_dtype, return_type, step)
        x = self.model._output(x, reduce, None, None)
        if self._out is None:
            self._out = {d: v.new_empty((self.coors.shape[0], self.page_size) + tuple(v.shape[1:])) for d, v in x.items()}
        dest = step['dest'][rows]
        for d, v in x.items():
            self._out[d].view((-1,) + tuple(v.shape[1:])).index_copy_(0, dest, v[rows])
        if exists(out_dtype):
            x = {k: v.to(out_dtype) for k, v in x.items()}
        return x[str(return_type)] if exists(return_type) else x

    # ---- one step ------------------------------------------------------------------------------------------
    def _reserve(self, ids, seqlens, coors, hits=()):
        """Every page of the step, and its copies on write, before its body: the body must stay idempotent.  hits: the cached
        pages that clouds in their first call attach (prefix cache)."""
        plan = self._book.plan(ids, [self._len[c] for c in ids], seqlens, hits)
        ops._require_cuda(coors)
        self._grow(plan.reserved, coors.device)
        copies = self._book.commit(plan, ids)
        self._commit = (plan, ids, copies)
        if copies:
            P = self.page_size
            rows = torch.tensor([[old * P + r for old, _, n in copies for r in range(n)],
                                 [new * P + r for _, new, n in copies for r in range(n)]]).to(coors.device)
            for t in self._tensors():
                flat = t.view((-1,) + tuple(t.shape[2:]))
                flat.index_copy_(0, rows[1], flat.index_select(0, rows[0]))

    def _tensors(self):
        return [self.coors] + [t for feats, nodemax in self.stages.values() for t in (*feats.values(), nodemax)] + \
            list((self._out or {}).values())

    def _grow(self, pages, dev):
        """A pool of `pages` pages, the old pool copied to its first pages (page ids do not change).  A fixed pool has scratch
        pages after them, which no cloud owns: the padding rows of graph steps store there."""
        if self.coors is not None and pages + self._scratch_pages <= self.coors.shape[0]:
            return
        pages += self._scratch_pages

        def grown(t):
            new = t.new_empty((pages,) + tuple(t.shape[1:]))
            new[:t.shape[0]] = t
            return new
        if self.coors is None:
            self.coors = torch.empty((0, self.page_size, 3), dtype=torch.float32, device=dev)
        self.coors = grown(self.coors)
        self.stages = {name: ({d: grown(t) for d, t in feats.items()}, grown(nodemax)) for name, (feats, nodemax) in self.stages.items()}
        if self._out is not None:
            self._out = {d: grown(t) for d, t in self._out.items()}

    def _where(self, ids, lens, pos):
        """Each new row's pool row, table_c[pos // P] P + pos % P."""
        P, tables = self.page_size, [self._book.tables[c] for c in ids]
        start = torch.tensor([0] + [len(t) for t in tables][:-1]).cumsum(0)
        flat = torch.tensor([p for t in tables for p in t], dtype=torch.int64)
        return flat[torch.repeat_interleave(start, lens) + pos // P] * P + pos % P

    def _search(self, ids, n_prev, seqlens, ks, pos, where, coors, neighbor_mask):
        self.coors.view(-1, 3).index_copy_(0, where, coors.float())
        idx, col, nmask, rel_pos, rel_dist = ops.knn_rows_paged(self.coors, [self._book.tables[c] for c in ids], n_prev, seqlens,
                                                                ks, self.model._valid_radius(), causal=True,
                                                                neighbor_mask=neighbor_mask)
        return where, idx, col, nmask, rel_pos, rel_dist

    # ---- steps replayed from CUDA graphs (DESIGN.md 10.3) -----------------------------------------------------------------
    def drop_graphs(self):
        """Forget every captured step and the memory they share; the next eligible step of each bucket captures again."""
        self._graphs.clear()
        self._graph_pool = self._graph_sw = self._graph_plans = None

    def _plan_state(self, sw):
        """What the captured steps read of every ConvSE3's decisions: its weight pack, low-rank plan and whether it left it.
        Holding it keeps the plan's tensors, which the graphs read, alive."""
        state = []
        for conv in self.model.conv_modules():
            pk = conv.packed(sw)
            state.append((pk, pk['lr'], conv._lr_blocked))
        return state

    @staticmethod
    def _same_plans(a, b):
        return all(x[0] is y[0] and x[1] is y[1] and x[2] == y[2] for x, y in zip(a, b))

    def _desc_room(self, need, rows):
        """Page ids a bucket's descriptor has room for: the step's need rounded up to a power of two (at least 1024), at most
        rows * max_pages (each listed cloud reads at most max_pages).  A later step that needs more captures the bucket again."""
        return min(max(1024, 1 << (need - 1).bit_length()), rows * self._book.max_pages)

    def _graph_key(self, ids, seqlens, feats, coors, edges, neighbor_mask, return_type, sw):
        """(M_bucket, K, the kind of inputs) of a step to replay from a graph, or None if it runs eagerly."""
        if sw.no_decode_graphs or not self.stages:
            return None
        n_prev = [self._len[c] for c in ids]
        bucket = decode_graph_bucket(self.max_nodes, n_prev, seqlens, [self.model._num_neighbors(p + m, 0) for p, m in zip(n_prev, seqlens)])
        if bucket is None:
            return None
        rows, K = bucket
        if ops.lowrank_enabled(rows * K, sw) != ops.lowrank_enabled(sum(seqlens) * K, sw):
            return None                           # the capture decides the route for rows * K edges, the step has fewer
        kind = (tuple((d, tuple(v.shape[1:]), v.dtype) for d, v in sorted(feats.items())) if isinstance(feats, dict) else
                (tuple(feats.shape[1:]), feats.dtype))
        pairs = None if edges is None else (tuple(edges[0].shape[2:]), edges[0].is_floating_point())
        return rows, K, kind, coors.dtype, pairs, neighbor_mask is not None, return_type

    def _run(self, ids, seqlens, feats, coors, edges, neighbor_mask, return_type):
        sw = switches.current()
        key = self._graph_key(ids, seqlens, feats, coors, edges, neighbor_mask, return_type, sw)
        if key is None:
            return super()._run(ids, seqlens, feats, coors, edges, neighbor_mask, return_type)
        if self._graphs and (sw != self._graph_sw or not self._same_plans(self._plan_state(sw), self._graph_plans)):
            self.drop_graphs()                    # a switch or a low-rank plan changed since the capture
        P = self.page_size
        need = sum(-(-(self._len[c] + m) // P) for c, m in zip(ids, seqlens))
        g = self._graphs.get(key)
        if g is not None and need > g.room:       # the descriptor outgrew its room: capture the bucket again with more
            del self._graphs[key]
            if not self._graphs:
                self.drop_graphs()
            g = None
        fresh = g is None
        if fresh:
            g = _DecodeGraph(key[0], key[1], self._n_pos(), self._desc_room(need, key[0]), feats, coors, edges, neighbor_mask)
        elif not g.copied.query():
            g.copied.synchronize()                # the previous replay still reads the pinned descriptor (no checks waited)
        M = self._fill(g, ids, seqlens, feats, coors, edges, neighbor_mask)
        if fresh:
            self._capture(g, key, return_type, sw)
        g.graph.replay()
        g.copied.record()
        self.graph_replays += 1
        bad = check_lowrank_stats(g.checks)       # the one host synchronisation of a replayed step
        if bad:
            self.drop_graphs()
            if any(conv.free_master for conv in bad):
                self._rollback()
                raise LowRankPlanMiss('low-rank radial plan does not cover this input; pack_weights(max_distance=...) was given too '
                                      'small a distance')
            return super()._run(ids, seqlens, feats, coors, edges, neighbor_mask, return_type)
        if isinstance(g.out, dict):
            return {d: v[:M].clone() for d, v in g.out.items()}
        return g.out[:M].clone()

    def _n_pos(self):
        """A bound on every cloud's length: the nodes of the pool's pages."""
        return self._book.max_pages * self.page_size

    def _fill(self, g, ids, seqlens, feats, coors, edges, neighbor_mask):
        """The step's descriptor and inputs into g's static buffers (no host synchronisation); returns its rows M."""
        P = self.page_size
        n_prev = [self._len[c] for c in ids]
        n_cur = [p + m for p, m in zip(n_prev, seqlens)]
        tables = [self._book.tables[c][:-(-n // P)] for c, n in zip(ids, n_cur)]
        M = ops.fill_decode_desc(g.host_desc, g.rows, n_prev, seqlens, [g.K] * len(ids), tables)
        if isinstance(feats, dict):
            for d, v in feats.items():
                g.feats[d][:M].copy_(v, non_blocking=True)
        else:
            g.feats[:M].copy_(feats, non_blocking=True)
        g.coors[:M].copy_(coors, non_blocking=True)
        for buf, per_cloud in ((g.edges, edges), (g.nbr, neighbor_mask)):
            if per_cloud is not None:
                flat = torch.cat([t.reshape((-1,) + tuple(t.shape[2:])) for t in per_cloud])
                buf[:flat.shape[0]].copy_(flat, non_blocking=True)
        return M

    def _capture(self, g, key, return_type, sw):
        """Warm up g's step outside the capture (weight images, plans and library state are built there), then capture it."""
        import time
        t0 = time.perf_counter()
        dev = g.coors.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            self._graph_body(g, return_type)
        torch.cuda.current_stream(dev).wait_stream(side)
        plans = self._plan_state(sw)
        if self._graphs and not self._same_plans(plans, self._graph_plans):
            self.drop_graphs()                    # the warm-up rebuilt a low-rank plan that the other graphs read
        if self._graph_pool is None:
            self._graph_pool = torch.cuda.graph_pool_handle()
        g.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g.graph, pool=self._graph_pool):
            g.out, g.checks = self._graph_body(g, return_type)
        self._graphs[key] = g
        self._graph_sw, self._graph_plans = sw, plans
        self.graph_capture_s[key[:2]] = time.perf_counter() - t0

    def _graph_body(self, g, return_type):
        """_step over g's static buffers, every per-row tensor built on the device from the descriptor: (outputs, deferred
        checks).  Rows M .. M_bucket pad the step: they repeat row M - 1's search and store into the scratch pages."""
        model, rows, K, n_pos = self.model, g.rows, g.K, self._n_pos()
        out_dtype = g.out_dtype
        if model.output_degrees == 1:
            return_type = 0
        g.desc.copy_(g.host_desc, non_blocking=True)
        desc = g.desc.view(torch.int64)
        pos, where, pair_row, _ = ops.decode_plan(desc, rows, rows, self.page_size, n_pos)
        if isinstance(g.feats, dict):
            feats = {d: v.unsqueeze(0) for d, v in g.feats.items()}
        else:
            feats = model._embed_tokens(g.feats.unsqueeze(0), pos)
            feats = {'0': feats[..., None]}
        feats = model._check_features(feats, g.coors)
        self.coors.view(-1, 3).index_copy_(0, where, g.coors)
        idx, col, nmask, rel_pos, rel_dist = ops.knn_rows_paged_bucket(self.coors, desc, rows, rows, n_pos, K, model._valid_radius(),
                                                                       causal=True, neighbor_mask=g.nbr)
        e = model._edge_features(None if g.edges is None else g.edges[pair_row[:, None] + col], None)
        pos_emb = None
        if exists(model.rotary_pos_emb):
            pos_emb = model._rotary(pos.view(1, rows), torch.cat((pos[:, None], col), dim=1).view(1, rows, 1 + K), n_pos,
                                    rel_dist.view(1, rows, K))
        geom = Geometry(rel_pos[None], model.num_degrees - 1, deferred=[])
        step = dict(dest=where, rows=_StepRows(rows), edge_info=(idx[None], nmask[None], None if e is None else e[None]),
                    rel_dist=rel_dist[None], geom=geom)
        out, checks = self._walk(feats, step, pos_emb, lambda v: v[0], out_dtype, return_type)
        # An eager step rebuilds a plan that its ConvSE3 can still rebuild (masters kept) once the step's largest distance
        # exceeds the plan's range D (ConvSE3.lowrank_plan).  The replay keeps the captured plan, so such a step counts as a
        # plan miss: the graphs are dropped and the step runs eagerly.  Padding rows repeat row M - 1, so the maximum over the
        # bucket is the step's; it is compared in float64, as lowrank_plan compares float(rel_dist.max()) with D.
        d_max, seen = None, set()
        for conv, _, _ in list(checks):
            if conv.free_master or id(conv) in seen:
                continue
            seen.add(id(conv))
            if d_max is None:
                d_max = rel_dist.max().double()
            beyond = torch.where(d_max > conv._packed['lr']['D'], 1e30, 0.0).float()
            checks.append((conv, torch.stack((beyond, torch.ones_like(beyond))).view(1, 2),
                           torch.ones(1, dtype=torch.bool, device=beyond.device)))
        return out, checks
