"""Shared helpers for the parity tests (no reference import; fixtures only)."""
import json
import os
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

MODEL_CASES = ['cfg1', 'deg4', 'af2', 'edges_sparse', 'ragged', 'tc_deg2', 'tc_deg4', 'allnbr', 'causal', 'tiekv',
               'linkeys', 'nullkv', 'noself', 'global', 'onehead', 'preconv_normout', 'tokens_pos', 'adjdeg', 'nbrmask',
               'contedges', 'rotary_both', 'rotary_pos_onehead', 'rotary_dist_linkeys', 'rotary_tiekv']

# BASELINE.json configs[2] at full size, configs[3] at batch 2 (the reference needs ~8 GB of host RAM per cloud there)
BIG_CASES = ['cfg3', 'cfg4_b2']


# widths the one-GEMM production kernel takes (every fiber a multiple of 128 channels, DESIGN.md 4.5)
Z_CASES = ['z128', 'z256_deg4']

# num_degrees 5 and 6, the top of the documented range (tests/golden/gen_golden.py DEG_CASES)
DEG_CASES = ['deg6', 'tc_deg5', 'z128_deg6']


def load_case(name):
    z = dict(np.load(os.path.join(GOLDEN, f'model_{name}.npz')))
    # the largest fixtures are split into model_<name>.part<i>.npz files (each stored file stays under 1 MB)
    for part in sorted(f for f in os.listdir(GOLDEN) if f.startswith(f'model_{name}.part')):
        z.update(np.load(os.path.join(GOLDEN, part)))
    cfg = json.loads(str(z.pop('config')))
    ctor = cfg['ctor']
    if isinstance(ctor.get('dim_in'), list):
        ctor['dim_in'] = tuple(ctor['dim_in'])
    return z, cfg


def state_keys(name):
    with open(os.path.join(GOLDEN, 'state_keys.json')) as f:
        keys = json.load(f)
    if name in keys:
        return keys[name]
    return json.loads(str(load_case(name)[0]['state_keys']))      # (DEG_CASES: stored in the fixture)


def det_params(name, seed=11):
    from detfill import det_tensor
    return {k: det_tensor(k, tuple(s), seed).astype(np.float32) for k, s in state_keys(name).items()
            if not k.endswith('inv_freq')}


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def case_inputs(z):
    inp = {k[3:]: v for k, v in z.items() if k.startswith('in/')}
    if 'feats' in inp:
        feats = inp['feats']
    else:
        feats = {'0': inp['feats/0'], '1': inp['feats/1']}
    extra = {k: inp[k] for k in ('adj_mat', 'edges', 'neighbor_mask', 'global_feats') if k in inp}
    return feats, inp['coors'], inp['mask'], extra


def case_outputs(z):
    if 'out' in z:
        return z['out']
    return {k[4:]: v for k, v in z.items() if k.startswith('out/')}


def assert_graph_equal(idx, mask, dist, ref_idx, ref_mask, ref_dist, atol=1e-5):
    """Neighbour lists agree as sets of valid (unmasked) neighbours with the same distances."""
    assert idx.shape == ref_idx.shape
    big = np.iinfo(np.int64).max
    a = np.where(mask, idx, big)
    b = np.where(ref_mask, ref_idx, big)
    oa = np.argsort(a, -1, kind='stable')
    ob = np.argsort(b, -1, kind='stable')
    assert np.array_equal(np.take_along_axis(a, oa, -1), np.take_along_axis(b, ob, -1))
    da = np.where(mask, dist, 0.0)
    db = np.where(ref_mask, ref_dist, 0.0)
    assert np.allclose(np.take_along_axis(da, oa, -1), np.take_along_axis(db, ob, -1), atol=atol)


# ---- layout decoders for the kernel-side images (DESIGN.md "data layout") ----
def decode_operand_image(img_u8):
    """uint8 [..., 65536] UMMA operand image -> (hi, lo) float32 [..., 128, 128] (rows, k)."""
    import torch
    img = img_u8.reshape(-1, 65536).cpu().numpy()
    as16 = img.view(np.uint16).reshape(img.shape[0], 2, 2, 128, 64)        # [tile][hi/lo][khalf][row][16B chunk * 8 + j]
    r = np.arange(128)[:, None]
    kk = np.arange(64)[None, :]
    phys = ((kk >> 3) ^ (r & 7)) * 8 + (kk & 7)                            # physical element index inside the 128-byte row
    out = np.empty((img.shape[0], 2, 128, 128), dtype=np.float32)
    for part in range(2):
        for kh in range(2):
            sub = np.take_along_axis(as16[:, part, kh], np.broadcast_to(phys, (img.shape[0], 128, 64)), axis=2)
            out[:, part, :, kh * 64:(kh + 1) * 64] = (sub.astype(np.uint32) << 16).view(np.float32)
    return out[:, 0], out[:, 1]


def decode_T(T, n_tiles, Ci, F, P, padded=False):
    """tile layout [tile][ifb][4][PH][128][4] -> [n_tiles*128, Ci*F, P] (padded: [n_tiles*128, 4*ifb, 4*PH], the padding slots
    of the layout included)."""
    nifb = (Ci * F + 3) // 4
    ph = (P + 3) // 4
    t = T[: n_tiles * nifb * 4 * ph * 128 * 4].reshape(n_tiles, nifb * 4, ph, 128, 4)
    t = t.transpose(0, 3, 1, 2, 4).reshape(n_tiles * 128, nifb * 4, ph * 4)
    return t if padded else t[:, : Ci * F, :P]


# ---- the production GEMM (csrc/zgemm.cu) on random operands, and its float64 restatement ----
def x_tile_layout(xp):
    """x' [E, Ci, ncomp] -> zgemm's X layout [tiles][Ci][ncomp][128] (zero rows past E)."""
    import torch
    E, Ci, nc = xp.shape
    tiles = (E + 127) // 128
    buf = torch.zeros(tiles * 128, Ci, nc, dtype=torch.float32, device=xp.device)
    buf[:E] = xp
    return buf.reshape(tiles, 128, Ci, nc).permute(0, 2, 3, 1).contiguous().reshape(-1)


def zgemm_reference(mode, segs, Co):
    """float64: segs = [(U [E,Kp], Fp [Co*Ci*F, Kp], x' [E,Ci,ncomp], cplus, cminus)] -> out [E, mode, Co]."""
    import torch
    outs = None
    mode = min(mode, 2)                                              # mode 3 computes what mode 2 computes (Gauss form)
    for U, Fp, xp, cp, cm in segs:
        E, Ci = xp.shape[0], xp.shape[1]
        Fv = Fp.double().reshape(Co, Ci, mode, -1)
        Ud = U.double()[:, :Fv.shape[-1]]
        w = torch.einsum('ek,oifk->eoif', Ud, Fv)                     # the radial weights of this segment
        xd = xp.double()
        if mode == 1:
            o = torch.einsum('eoi,ei->eo', w[..., 0], xd[:, :, cp])[:, None]
        else:
            a, b = w[..., 0], w[..., 1]
            op = torch.einsum('eoi,ei->eo', a, xd[:, :, cp]) - torch.einsum('eoi,ei->eo', b, xd[:, :, cm])
            om = torch.einsum('eoi,ei->eo', b, xd[:, :, cp]) + torch.einsum('eoi,ei->eo', a, xd[:, :, cm])
            o = torch.stack([op, om], dim=1)
        outs = o if outs is None else outs + o
    return outs


def zgemm_problem(mode, Co, E, seg_shapes, seed=0, x_scale=1.0, positive=False, device='cuda'):
    """Random operands of one zgemm launch.  seg_shapes: [(Ci, ncomp, cplus, cminus, Kp)].  Returns (segs in the form ops.zgemm
    takes, weight image, per-edge scales sx, float64 reference [E, planes, Co])."""
    import torch
    from se3_transformer_pytorch_b200 import ops
    g = torch.Generator(device=device).manual_seed(seed)
    rnd = (lambda *s: torch.rand(*s, generator=g, device=device) + 0.1) if positive else (lambda *s: torch.randn(*s, generator=g, device=device))
    segs_ref, segs_k, parts = [], [], []
    for Ci, nc, cp, cm, Kp in seg_shapes:
        U = torch.zeros(E, 64, device=device)
        U[:, :Kp] = rnd(E, Kp)
        U[:, Kp - 1] = 1.0                                             # the bias slot
        Fp = rnd(Co * Ci * min(mode, 2), Kp) / (Ci * Kp) ** 0.5
        xp = rnd(E, Ci, nc) * x_scale
        segs_ref.append((U, Fp, xp, cp, cm))
        X = x_tile_layout(xp)
        for kc in range(Kp // 16):
            segs_k.append((U[:, 16 * kc:], X, Ci, nc, cp, cm))
        parts.append((Fp.contiguous(), Ci))
    img, S = ops.zgemm_image(parts, Co, mode)
    # per-edge power-of-two scales as the model makes them (from the row maximum), exercising the scale / unscale path
    rowmax = torch.stack([s[2].abs().amax(dim=(1, 2)) for s in segs_ref]).amax(0)
    sx = torch.exp2(torch.floor(9 - torch.log2(rowmax.clamp(min=1e-30)))).float()
    return segs_k, img, sx, zgemm_reference(mode, segs_ref, Co)


def run_zgemm(mode, Co, E, seg_shapes, flush=0, seed=0, x_scale=1.0, positive=False):
    """One zgemm launch on zgemm_problem's operands.  Returns (gpu out [E, planes, Co], float64 reference)."""
    import torch
    from se3_transformer_pytorch_b200 import ops
    segs, img, sx, ref = zgemm_problem(mode, Co, E, seg_shapes, seed, x_scale, positive)
    planes = min(mode, 2)
    out = torch.full((E, planes, Co), 7.0, device=sx.device)
    ops.zgemm(segs, img, sx, E, Co, mode, out, planes * Co, [0, Co], flush_stages=flush)
    torch.cuda.synchronize()
    return out, ref


def zgemm_split_units(segs, Co, mode, flush_stages=0):
    """The split units of a zgemm launch (its largest k_split)."""
    from se3_transformer_pytorch_b200 import ops
    arr = (ops.ZSeg * len(segs))(*[ops.ZSeg(U.data_ptr(), X.data_ptr(), Ci, nc, cp, cm) for U, X, Ci, nc, cp, cm in segs])
    return ops.lib().se3_zgemm_split_units(arr, len(segs), Co, mode, flush_stages)


def attention_reference(q, kd, vd, nmask, H, Dh, kvh, scale):
    """float64 attention of one degree: q [b,n,H*Dh,M]; kd, vd [b,n,J,kvh*Dh,M] with the prefix keys (global, null, self)
    first and the K neighbours last; nmask [b,n,K] or None -> [b,n,H*Dh,M]."""
    b, n, J, _, M = kd.shape
    qh = q.reshape(b, n, H, Dh, M).astype(np.float64)
    kh = np.broadcast_to(kd.reshape(b, n, J, kvh, Dh, M), (b, n, J, H, Dh, M)) if kvh == 1 else kd.reshape(b, n, J, H, Dh, M)
    vh = np.broadcast_to(vd.reshape(b, n, J, kvh, Dh, M), (b, n, J, H, Dh, M)) if kvh == 1 else vd.reshape(b, n, J, H, Dh, M)
    sim = np.einsum('bihdm,bijhdm->bihj', qh, kh.astype(np.float64)) * scale
    if nmask is not None:
        mk = np.concatenate([np.ones((b, n, J - nmask.shape[-1]), dtype=bool), nmask], -1)[:, :, None]
        sim = np.where(mk, sim, -np.finfo(np.float32).max)
    sim = sim - sim.max(-1, keepdims=True)
    a = np.exp(sim); a /= a.sum(-1, keepdims=True)
    return np.einsum('bihj,bijhdm->bihdm', a, vh.astype(np.float64)).reshape(b, n, H * Dh, M)
